// vamb_b200 VAE kernels, fp32 CUDA-core path (sm_90a).
//
// One optimiser step of vamb/encode.py (VAE.trainepoch :401-419) = 15 stream-ordered launches:
//   batch_rows  | fwd x (2L+2) | loss | bwd x (2L+2) (wgrad + dgrad tiles in ONE grid) | dadapt
// with every element-wise stage fused into the operand loads / epilogues of the GEMM tiles:
//   * BatchNorm is never materialised: producers write P = dropout(leakyrelu(xW^T+b)) plus
//     per-row-tile column sums; the LAST block to finish (ticket) folds them into the per-feature
//     affine (a, c) and the running statistics; consumers apply P*a + c while loading.
//   * the BatchNorm / dropout / LeakyReLU backward is applied while loading dH as a GEMM operand;
//     its two batch reductions (sum dH, sum dH*Phat) are column sums of the dgrad epilogue.
//   * bias gradients come out of the wgrad GEMM through a virtual all-ones input column.
// All reductions are two-stage with a fixed order (no floating-point atomics): same inputs ->
// same bits.  The fp32 CUDA-core kernels below are the exact-fp32 path; the tensor-core kernels (wgmma, 3xTF32,
// vk_tc.cuh) replace the GEMM core for large batches.
//
// Reference lines (RasmussenLab/vamb): encode.py:259-273 _encode, :276-286 reparameterize,
// :288-304 _decode, :316-357 calc_loss, :442-484 encode; dadaptation==3.2 DAdaptAdam.step.
#include <stdlib.h>

#include "vk_common.cuh"
#include "vk_tc.cuh"

// ------------------------------------------------------------------ small device helpers
__device__ __forceinline__ void philox4x32(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                           uint32_t k1, uint32_t (&out)[4]) {
#pragma unroll
    for (int r = 0; r < 7; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

__device__ __forceinline__ float u32_to_unit(uint32_t x) {  // (0, 1]
    return ((float)(x >> 8) + 1.0f) * (1.0f / 16777216.0f);
}

// Feistel permutation of [0, n) by cycle walking over [0, 2^(2*half_bits)).
__device__ __forceinline__ uint64_t feistel_perm(uint64_t i, uint64_t n, int half_bits, uint64_t key) {
    const uint32_t mask = (1u << half_bits) - 1u;
    uint64_t x = i;
    do {
        uint32_t l = (uint32_t)(x >> half_bits) & mask, r = (uint32_t)x & mask;
#pragma unroll
        for (int round = 0; round < 4; ++round) {
            uint32_t f = (r ^ (uint32_t)(key >> (16 * round))) * 0x9E3779B1u;
            f ^= f >> 15; f *= 0x85EBCA6Bu; f ^= f >> 13;
            const uint32_t nl = r, nr = (l ^ f) & mask;
            l = nl; r = nr;
        }
        x = ((uint64_t)l << half_bits) | r;
    } while (x >= n);
    return x;
}

__device__ __forceinline__ uint64_t mix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// Fixed-shape tree sum of one double per thread of a 256-thread block (xor butterfly inside each warp,
// then the 8 warp sums in order): same bits every run, ~50x shorter than a serial fold.  Result valid in
// thread 0.  `s8` = 8 doubles of shared memory.
__device__ __forceinline__ double block_sum256(double v, double *s8) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) s8[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < 8; ++w) t += s8[w];
    return t;
}

// ------------------------------------------------------------------ batch rows + mean weight
// mode 0: rows from inject->batch_idx; 1: epoch permutation; 2: contiguous [row0, row0+B)
// "last block done": returns true in every thread of the block that finishes last.
// One fencing thread per block: after the block barrier, thread 0's device-scope fence is cumulative over what the
// block wrote before the barrier (release), and its second fence orders the last block's reads after the ticket
// (acquire) -- the pattern of cutlass/semaphore.h.  A MEMBAR by every thread of every block cost microseconds per launch.
__device__ __forceinline__ bool last_block_done(int32_t *ticket, int total) {
    __shared__ int s_last;
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const int t = atomicAdd(ticket, 1);
        s_last = (t == total - 1);
        if (s_last) {
            *ticket = 0;  // self-reset for the next launch
            __threadfence();
        }
    }
    __syncthreads();
    return s_last != 0;
}

// Dataset row of batch position b.  mode 0: host-injected indices; 1: epoch permutation (Feistel network keyed by
// seed / epoch, position = step within the epoch * B + b); 2: contiguous [row0, row0 + B).
__device__ __forceinline__ int64_t batch_row_index(int mode, int b, int B, const int64_t *batch_idx, const vk_vae_ctl *ctl,
                                                   int64_t n_rows, int64_t row0, int steps_per_epoch) {
    if (mode == 0) return batch_idx[b];
    if (mode == 1) {
        int half_bits = 1;
        while ((1ull << (2 * half_bits)) < (uint64_t)n_rows) ++half_bits;
        const uint64_t key = mix64(ctl->seed ^ (0x5851F42D4C957F2Dull * (uint64_t)(ctl->epoch + 1)));
        int64_t t = ctl->step - ctl->epoch_step0;
        if (steps_per_epoch > 0) t %= steps_per_epoch;
        return (int64_t)feistel_perm((uint64_t)(t * (int64_t)B + b), (uint64_t)n_rows, half_bits, key);
    }
    return row0 + b;
}

// One thread per batch row (grid = ceil(B / 256) blocks); the batch-mean weight is folded by the last
// block from per-block partial sums in block order (fixed order -> reproducible).
__global__ void __launch_bounds__(256)
batch_rows_kernel(int64_t *batch_rows, const int64_t *batch_idx, const float *weights, vk_vae_ctl *ctl, int B,
                  int64_t n_rows, int mode, int64_t row0, int steps_per_epoch, double *part, int ticket_id) {
    const int tk = tk_begin(1);
    pdl_entry();
    __shared__ double s_w[16];
    const int tid = threadIdx.x;
    const int b = blockIdx.x * 256 + tid;
    double acc = 0.0;
    if (b < B) {
        const int64_t r = batch_row_index(mode, b, B, batch_idx, ctl, n_rows, row0, steps_per_epoch);
        batch_rows[b] = r;
        acc = (double)weights[r];
    }
    const double t = block_sum256(acc, s_w);
    if (tid == 0) part[blockIdx.x] = t;
    tk_end(tk);
    if (!last_block_done(&ctl->tickets[ticket_id], gridDim.x)) return;
    if (tid == 0) {
        double tot = 0.0;
        for (unsigned i = 0; i < gridDim.x; ++i) tot += __ldcg(part + i);
        ctl->wbar = tot / (double)B;
    }
    tk_end(tk);
}

// ------------------------------------------------------------------ operand loaders
// at(r, c): element (row r, column c) of the logical [rows, cols] operand, 0 outside.
// ld4(r, c4): elements (r, 4*c4 .. 4*c4+3) -- one 16-byte load per array when the row is 16-byte
// aligned and fully inside, else four at() calls (used by the tensor-core path, vk_tc.cuh).
__device__ __forceinline__ bool vec_ok(const void *p, int ld) {
    return ((ld & 3) == 0) && ((reinterpret_cast<uintptr_t>(p) & 15) == 0);
}
__device__ __forceinline__ float4 ldg4(const float *q) { return __ldg(reinterpret_cast<const float4 *>(q)); }

struct LdPlain {
    const float *p; int ld, rows, cols;
    __device__ __forceinline__ float at(int r, int c) const {
        return (r < rows && c < cols) ? __ldg(p + (int64_t)r * ld + c) : 0.0f;
    }
    __device__ __forceinline__ float4 ld4(int r, int c4) const {
        const int c = c4 << 2;
        if (r < rows && c + 3 < cols && vec_ok(p, ld)) return ldg4(p + (int64_t)r * ld + c);
        return make_float4(at(r, c), at(r, c + 1), at(r, c + 2), at(r, c + 3));
    }
};
struct LdAffine {  // BatchNorm applied on load: P * a + c
    const float *p; const float *a; const float *sh; int ld, rows, cols;
    __device__ __forceinline__ float at(int r, int c) const {
        if (r >= rows || c >= cols) return 0.0f;
        return __fmaf_rn(__ldg(p + (int64_t)r * ld + c), __ldg(a + c), __ldg(sh + c));
    }
    __device__ __forceinline__ float4 ld4(int r, int c4) const {
        const int c = c4 << 2;
        if (r < rows && c + 3 < cols && vec_ok(p, ld)) {
            const float4 v = ldg4(p + (int64_t)r * ld + c), s4 = ldg4(a + c), h4 = ldg4(sh + c);
            return make_float4(__fmaf_rn(v.x, s4.x, h4.x), __fmaf_rn(v.y, s4.y, h4.y), __fmaf_rn(v.z, s4.z, h4.z),
                               __fmaf_rn(v.w, s4.w, h4.w));
        }
        return make_float4(at(r, c), at(r, c + 1), at(r, c + 2), at(r, c + 3));
    }
};
struct LdData {  // gathered dataset rows
    const float *data; const int64_t *rows_idx; int ld, rows, cols;
    __device__ __forceinline__ float at(int r, int c) const {
        return (r < rows && c < cols) ? __ldg(data + rows_idx[r] * (int64_t)ld + c) : 0.0f;
    }
    __device__ __forceinline__ float4 ld4(int r, int c4) const {
        const int c = c4 << 2;
        if (r < rows && c + 3 < cols && vec_ok(data, ld)) return ldg4(data + rows_idx[r] * (int64_t)ld + c);
        return make_float4(at(r, c), at(r, c + 1), at(r, c + 2), at(r, c + 3));
    }
};
struct LdDY {  // dL/dY of a hidden block from dL/dBN(P): BatchNorm, dropout and LeakyReLU backward
    const float *dh; const float *p; const float *g; const float *mean; const float *rstd;
    const float *m1; const float *m2; int ld, rows, cols; float inv_keep, slope; int has_dropout;
    __device__ __forceinline__ float one(float pv, float dhv, float gv, float mu, float rs, float a1, float a2) const {
        if (has_dropout && pv == 0.0f) return 0.0f;  // dropped unit
        const float ph = (pv - mu) * rs;
        float v = gv * rs * (dhv - a1 - ph * a2);
        v *= inv_keep;
        return pv > 0.0f ? v : v * slope;
    }
    __device__ __forceinline__ float at(int r, int c) const {
        if (r >= rows || c >= cols) return 0.0f;
        const int64_t o = (int64_t)r * ld + c;
        return one(__ldg(p + o), __ldg(dh + o), __ldg(g + c), __ldg(mean + c), __ldg(rstd + c), __ldg(m1 + c),
                   __ldg(m2 + c));
    }
    __device__ __forceinline__ float4 ld4(int r, int c4) const {
        const int c = c4 << 2;
        if (r < rows && c + 3 < cols && vec_ok(p, ld) && vec_ok(dh, ld)) {
            const int64_t o = (int64_t)r * ld + c;
            const float4 pv = ldg4(p + o), dv = ldg4(dh + o), gv = ldg4(g + c), mu = ldg4(mean + c),
                         rs = ldg4(rstd + c), a1 = ldg4(m1 + c), a2 = ldg4(m2 + c);
            return make_float4(one(pv.x, dv.x, gv.x, mu.x, rs.x, a1.x, a2.x), one(pv.y, dv.y, gv.y, mu.y, rs.y, a1.y, a2.y),
                               one(pv.z, dv.z, gv.z, mu.z, rs.z, a1.z, a2.z), one(pv.w, dv.w, gv.w, mu.w, rs.w, a1.w, a2.w));
        }
        return make_float4(at(r, c), at(r, c + 1), at(r, c + 2), at(r, c + 3));
    }
};
// generic input activation of a layer (data / BN(P) / z) with an optional all-ones extra column
struct LdInput {
    int in_kind; LdData d; LdAffine a; LdPlain z; int ones_col;  // ones_col < 0: none
    __device__ __forceinline__ int nrows() const { return in_kind == VK_IN_DATA ? d.rows : in_kind == VK_IN_BN ? a.rows : z.rows; }
    __device__ __forceinline__ float at(int r, int c) const {
        if (c == ones_col) return r < nrows() ? 1.0f : 0.0f;
        if (in_kind == VK_IN_DATA) return d.at(r, c);
        if (in_kind == VK_IN_BN) return a.at(r, c);
        return z.at(r, c);
    }
    __device__ __forceinline__ float4 ld4(int r, int c4) const {
        const int c = c4 << 2;
        if (ones_col >= c && ones_col < c + 4) return make_float4(at(r, c), at(r, c + 1), at(r, c + 2), at(r, c + 3));
        if (in_kind == VK_IN_DATA) return d.ld4(r, c4);
        if (in_kind == VK_IN_BN) return a.ld4(r, c4);
        return z.ld4(r, c4);
    }
};
// generic dL/dY of a layer: hidden -> LdDY, mu / out -> plain
struct LdGradOut {
    int hidden; LdDY h; LdPlain pl;
    __device__ __forceinline__ float at(int r, int c) const { return hidden ? h.at(r, c) : pl.at(r, c); }
    __device__ __forceinline__ float4 ld4(int r, int c4) const { return hidden ? h.ld4(r, c4) : pl.ld4(r, c4); }
};
// rows [off, off + n) of another loader (split-K slices of the batch dimension)
template <class L>
struct LdRowSlice {
    L inner; int off, n;
    __device__ __forceinline__ float4 ld4(int r, int c4) const {
        return r < n ? inner.ld4(r + off, c4) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
};

// ------------------------------------------------------------------ 64x64x16 fp32 GEMM tile
constexpr int GT = 256;       // threads: 16 x 16, each a TM x TN micro-tile
constexpr int BK = 16;
constexpr int SMEM_GEMM_FLOATS = 2 * BK * (64 + 4) * 2;

// C[m, n] = sum_k A(m, k) * B(n, k).  AT: A stored [k][m] (at(k, m)); else [m][k].  Same for B.
template <int BM, int BN, bool AT, bool BT, class LA, class LB>
__device__ __forceinline__ void gemm_block(int K, int m0, int n0, const LA &la, const LB &lb,
                                           float (&acc)[BM / 16][BN / 16], float *smem) {
    constexpr int TM = BM / 16, TN = BN / 16, LDA = BM + 4, LDB = BN + 4;
    float *As = smem;
    float *Bs = smem + 2 * BK * LDA;
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    float ra[TM], rb[TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.0f;

    auto gload = [&](int k0) {
#pragma unroll
        for (int i = 0; i < TM; ++i) {
            if (!AT) { const int k = tid & 15, m = (tid >> 4) + 16 * i; ra[i] = la.at(m0 + m, k0 + k); }
            else { const int m = tid % BM, k = tid / BM + (GT / BM) * i; ra[i] = la.at(k0 + k, m0 + m); }
        }
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            if (!BT) { const int k = tid & 15, n = (tid >> 4) + 16 * j; rb[j] = lb.at(n0 + n, k0 + k); }
            else { const int n = tid % BN, k = tid / BN + (GT / BN) * j; rb[j] = lb.at(k0 + k, n0 + n); }
        }
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int i = 0; i < TM; ++i) {
            int m, k;
            if (!AT) { k = tid & 15; m = (tid >> 4) + 16 * i; }
            else { m = tid % BM; k = tid / BM + (GT / BM) * i; }
            As[(buf * BK + k) * LDA + m] = ra[i];
        }
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            int n, k;
            if (!BT) { k = tid & 15; n = (tid >> 4) + 16 * j; }
            else { n = tid % BN; k = tid / BN + (GT / BN) * j; }
            Bs[(buf * BK + k) * LDB + n] = rb[j];
        }
    };

    const int nk = (K + BK - 1) / BK;
    gload(0);
    sstore(0);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nk) gload((kt + 1) * BK);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[TM], b[TN];
            const float *ap = As + (buf * BK + k) * LDA + ty * TM;
            const float *bp = Bs + (buf * BK + k) * LDB + tx * TN;
#pragma unroll
            for (int i = 0; i < TM; ++i) a[i] = ap[i];
#pragma unroll
            for (int j = 0; j < TN; ++j) b[j] = bp[j];
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = __fmaf_rn(a[i], b[j], acc[i][j]);
        }
        if (kt + 1 < nk) sstore(buf ^ 1);
        __syncthreads();
    }
}

// column sums of a 64x64 tile held as 4x4 micro-tiles: deterministic two-stage reduction.
// v0/v1[j] = this thread's partial over its TM rows.  Writes out0/out1[col] for col < 64.
template <int TN>
__device__ __forceinline__ void tile_colsum2(const float (&v0)[TN], const float (&v1)[TN], double *s_red,
                                             double *out0, double *out1, int n0, int N) {
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    constexpr int BN = TN * 16;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
        s_red[(0 * 16 + ty) * BN + tx * TN + j] = (double)v0[j];
        s_red[(1 * 16 + ty) * BN + tx * TN + j] = (double)v1[j];
    }
    __syncthreads();
    if (tid < 2 * BN) {
        const int which = tid / BN, col = tid % BN;
        double t = 0.0;
#pragma unroll
        for (int r = 0; r < 16; ++r) t += s_red[(which * 16 + r) * BN + col];
        if (n0 + col < N) (which ? out1 : out0)[n0 + col] = t;
    }
    __syncthreads();
}

// ------------------------------------------------------------------ forward layer
struct FwdArgs {
    LdInput in;           // input activation [B, K]
    const float *W, *bias;  // [N, K], [N]
    int B, K, N, kind, training;
    float *out;           // P / MU / R  [B, N]
    // hidden
    float dropout; const uint8_t *keep; double *part;
    float *bn_a, *bn_c, *bn_mean, *bn_rstd; const float *gamma, *beta;
    float *running_mean, *running_var; int64_t *nbt;
    // mu
    float *z; const float *eps; int add_eps; int mask_bits; float *latent_out;
    vk_vae_ctl *ctl; int layer_id; float slope;
    int tile_n;           // tensor-core path: output columns per CTA (multiple of 16, <= 128)
    tc::OpRef a_op, b_op; // staged operands (layer input, W)
    // fused staging of the NEXT layer's operands from this layer's output tile (tensor-core path):
    // 0 off; 1 BatchNorm with this batch's statistics (grid barrier, then every CTA folds its own columns);
    // 2 plain copy (z) or BatchNorm with the precomputed affine bn_a / bn_c (evaluation)
    int stage; float *stage_a; int stage_a_ld; float *stage_t; int stage_t_ld;
    // B operand (W and its tf32 remainder) through TMA: 128B-swizzled tensor maps, box = 32 floats x tile_n rows
    int use_tma; VkTmap tm_b_hi, tm_b_lo;
    int cluster_rt;       // > 0: the row tiles of one column tile form a thread-block cluster of this size (cluster fold)
    int b_pow2; double inv_b, unbias;  // B is a power of two; 1 / B; B / (B - 1)
};

// Fold the per-row-tile column sums of P and P^2 into the BatchNorm affine, the saved batch statistics
// and the running statistics (torch.nn.BatchNorm1d, momentum 0.1, unbiased running variance).  Run by
// every thread of the last block to finish.
__device__ __forceinline__ void bn_forward_finalize(const FwdArgs &a, int n_rt, int nthreads) {
    for (int n = threadIdx.x; n < a.N; n += nthreads) {
        double s = 0.0, q = 0.0;
#pragma unroll 8
        for (int rt = 0; rt < n_rt; ++rt) {
            s += __ldcg(a.part + ((int64_t)rt * 2 + 0) * a.N + n);
            q += __ldcg(a.part + ((int64_t)rt * 2 + 1) * a.N + n);
        }
        const double mean = s / a.B;
        double var = q / a.B - mean * mean;
        if (var < 0.0) var = 0.0;
        const float rstd = (float)(1.0 / sqrt(var + 1e-5));
        const float fm = (float)mean;
        a.bn_mean[n] = fm;
        a.bn_rstd[n] = rstd;
        const float sc = a.gamma[n] * rstd;
        a.bn_a[n] = sc;
        a.bn_c[n] = a.beta[n] - fm * sc;
        const float unb = a.B > 1 ? (float)(var * ((double)a.B / (double)(a.B - 1))) : (float)var;
        a.running_mean[n] = 0.9f * a.running_mean[n] + 0.1f * fm;
        a.running_var[n] = 0.9f * a.running_var[n] + 0.1f * unb;
    }
    if (threadIdx.x == 0) *a.nbt += 1;
}

__global__ void __launch_bounds__(GT) fwd_layer_kernel(FwdArgs a) {
    pdl_entry();
    __shared__ __align__(16) float s_gemm[SMEM_GEMM_FLOATS];
    __shared__ double s_red[2 * 16 * 64];
    float acc[4][4];
    const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
    LdPlain w{a.W, a.K, a.N, a.K};
    gemm_block<64, 64, false, false>(a.K, m0, n0, a.in, w, acc, s_gemm);

    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const uint32_t k0 = (uint32_t)a.ctl->seed, k1 = (uint32_t)(a.ctl->seed >> 32);
    const uint32_t step_lo = (uint32_t)a.ctl->step, step_hi = (uint32_t)(a.ctl->step >> 32);
    float cs[4] = {0.f, 0.f, 0.f, 0.f}, cq[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= a.B) continue;
        uint32_t rnd[4] = {0u, 0u, 0u, 0u};
        const int nq = n0 / 4 + tx;
        if (a.kind == VK_LAYER_HIDDEN && a.training && a.dropout > 0.0f && a.keep == nullptr)
            philox4x32((uint32_t)m, (uint32_t)nq, step_lo, step_hi ^ ((uint32_t)(a.layer_id + 1) << 24), k0, k1, rnd);
        if (a.kind == VK_LAYER_MU && a.add_eps && a.eps == nullptr)
            philox4x32((uint32_t)m, (uint32_t)nq, step_lo, step_hi ^ 0x7F000000u, k0, k1, rnd);
        float nrm[4] = {0.f, 0.f, 0.f, 0.f};
        if (a.kind == VK_LAYER_MU && a.add_eps && a.eps == nullptr) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float u1 = u32_to_unit(rnd[2 * h]), u2 = u32_to_unit(rnd[2 * h + 1]);
                const float r = sqrtf(-2.0f * logf(u1));
                float sn, cn;
                sincosf(6.28318530717958647692f * u2, &sn, &cn);
                nrm[2 * h] = r * cn;
                nrm[2 * h + 1] = r * sn;
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= a.N) continue;
            const float y = acc[i][j] + __ldg(a.bias + n);
            const int64_t o = (int64_t)m * a.N + n;
            if (a.kind == VK_LAYER_HIDDEN) {
                float p = y > 0.0f ? y : y * a.slope;
                if (a.training && a.dropout > 0.0f) {
                    bool kp;
                    if (a.keep) kp = a.keep[o] != 0;
                    else kp = u32_to_unit(rnd[j]) > a.dropout;  // P(keep) = 1 - dropout
                    p = kp ? p * (1.0f / (1.0f - a.dropout)) : 0.0f;
                }
                a.out[o] = p;
                cs[j] += p;
                cq[j] = __fmaf_rn(p, p, cq[j]);
            } else if (a.kind == VK_LAYER_MU) {
                a.out[o] = y;
                if (a.add_eps) {
                    const float e = a.eps ? __ldg(a.eps + o) : nrm[j];
                    a.z[o] = y + e;
                }
                if (a.latent_out) {
                    const uint32_t bits = __float_as_uint(y) & ~((1u << a.mask_bits) - 1u);
                    a.latent_out[o] = __uint_as_float(bits);
                }
            } else {
                a.out[o] = y;
            }
        }
    }
    if (a.kind != VK_LAYER_HIDDEN || !a.training) return;

    // ---- BatchNorm batch statistics: per-row-tile column sums, folded by the last block ----
    const int n_rt = gridDim.y;
    double *p0 = a.part + ((int64_t)blockIdx.y * 2 + 0) * a.N;
    double *p1 = a.part + ((int64_t)blockIdx.y * 2 + 1) * a.N;
    tile_colsum2<4>(cs, cq, s_red, p0, p1, n0, a.N);
    if (!last_block_done(&a.ctl->tickets[a.layer_id], gridDim.x * gridDim.y)) return;
    bn_forward_finalize(a, n_rt, blockDim.x);
}

// ------------------------------------------------------------------ loss (+ dL/dR)
struct LossArgs {
    const float *R; const float *MU; const float *data; const int64_t *batch_rows;
    float *dR; int B, S, ntnf, d_in, nlatent, data_ld; float ce_w, ab_w, sse_w, kld_w;
    double *part; vk_vae_ctl *ctl; int ticket_id; int write_grad;
    // tensor-core path, fused staging: dL/dR also as the lane-major operands of the output layer's dgrad / wgrad
    float *stage_a; int stage_a_ld; float *stage_t; int stage_t_ld;
    int fold_later;  // 1: the caller launches loss_fold_kernel on a side stream
};

// Fold the per-block partial sums of one step into the running loss sums (256 threads, fixed order).
__device__ __forceinline__ void loss_fold(const LossArgs &a, unsigned n_blocks) {
    // fixed-order parallel fold of the block partials: thread t sums blocks t, t+256, ...; then a serial
    // fold of the 256 thread sums (same order every run)
    __shared__ double s_fold[4][16];
    {
        double t[4] = {0.0, 0.0, 0.0, 0.0};
        for (unsigned i = threadIdx.x; i < n_blocks; i += 256)
            for (int c = 0; c < 4; ++c) t[c] += __ldcg(a.part + (int64_t)i * 4 + c);
        for (int c = 0; c < 4; ++c) {
            const double r = block_sum256(t[c], &s_fold[c][0]);
            if (threadIdx.x == 0) s_fold[c][8] = r;
        }
    }
    if (threadIdx.x == 0) {
        const double ab = s_fold[0][8] / a.B * a.ab_w, ce = s_fold[1][8] / a.B * a.ce_w,
                     sse = s_fold[2][8] / a.B * a.sse_w, kld = s_fold[3][8] / a.B * a.kld_w;
        // loss.mean() over the [B, B] broadcast = mean_j(l_j) * mean_i(w_i)   (encode.py:349-352)
        a.ctl->loss_sums[0] += ((ce + ab + sse) + kld) * a.ctl->wbar;
        a.ctl->loss_sums[1] += ab;
        a.ctl->loss_sums[2] += ce;
        a.ctl->loss_sums[3] += sse;
        a.ctl->loss_sums[4] += kld;
        a.ctl->n_loss_steps += 1;
    }
}


constexpr int LOSS_STAGE_MAX_D = 160;  // widest reconstruction the loss kernel stages itself (else a prep launch does)

__global__ void __launch_bounds__(256) loss_kernel(LossArgs a) {
    const int tk = tk_begin(30);
    pdl_entry();
    __shared__ double s_part[8][4];
    __shared__ __align__(16) float s_g[8][LOSS_STAGE_MAX_D + 4];  // the block's eight rows of dL/dR (fused staging)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int b = blockIdx.x * 8 + warp;
    double l_ce = 0.0, l_sse = 0.0, l_ab = 0.0, l_kld = 0.0;
    if (a.stage_a)
        for (int i = threadIdx.x; i < 8 * (LOSS_STAGE_MAX_D + 4); i += 256) (&s_g[0][0])[i] = 0.0f;
    if (a.stage_a) __syncthreads();
    if (b < a.B) {
        const float *r = a.R + (int64_t)b * a.d_in;
        const float *x = a.data + a.batch_rows[b] * (int64_t)a.data_ld;
        float *g = a.dR + (int64_t)b * a.d_in;
        const float gsc = (float)(a.ctl->wbar / (double)a.B);
        // softmax over the S depth outputs (encode.py:302)
        float mx = -INFINITY;
        for (int s = lane; s < a.S; s += 32) mx = fmaxf(mx, r[s]);
        for (int o = 16; o; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        float sum = 0.0f;
        for (int s = lane; s < a.S; s += 32) sum += expf(r[s] - mx);
        for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        float ce = 0.0f, dot = 0.0f;
        for (int s = lane; s < a.S; s += 32) {
            const float p = expf(r[s] - mx) / sum;
            const float pe = p + 1e-9f;
            ce -= logf(pe) * x[s];
            dot += p * (-gsc * a.ce_w * x[s] / pe);
        }
        for (int o = 16; o; o >>= 1) {
            ce += __shfl_xor_sync(0xffffffffu, ce, o);
            dot += __shfl_xor_sync(0xffffffffu, dot, o);
        }
        if (a.write_grad)
            for (int s = lane; s < a.S; s += 32) {
                const float p = expf(r[s] - mx) / sum;
                const float gs = -gsc * a.ce_w * x[s] / (p + 1e-9f);
                g[s] = p * (gs - dot);
                if (a.stage_a) s_g[warp][s] = p * (gs - dot);
            }
        float sse = 0.0f;
        for (int t = lane; t < a.ntnf; t += 32) {
            const float df = r[a.S + t] - x[a.S + t];
            sse = __fmaf_rn(df, df, sse);
            if (a.write_grad) g[a.S + t] = gsc * a.sse_w * 2.0f * df;
            if (a.stage_a) s_g[warp][a.S + t] = gsc * a.sse_w * 2.0f * df;
        }
        for (int o = 16; o; o >>= 1) sse += __shfl_xor_sync(0xffffffffu, sse, o);
        const int ia = a.S + a.ntnf;
        const float dab = r[ia] - x[ia];
        if (lane == 0 && a.write_grad) g[ia] = gsc * a.ab_w * 2.0f * dab;
        if (lane == 0 && a.stage_a) s_g[warp][ia] = gsc * a.ab_w * 2.0f * dab;
        float kld = 0.0f;
        for (int k = lane; k < a.nlatent; k += 32) {
            const float m = a.MU[(int64_t)b * a.nlatent + k];
            kld = __fmaf_rn(m, m, kld);
        }
        for (int o = 16; o; o >>= 1) kld += __shfl_xor_sync(0xffffffffu, kld, o);
        l_ce = ce; l_sse = sse; l_ab = dab * dab; l_kld = 0.5f * kld;
    }
    if (lane == 0) { s_part[warp][0] = l_ab; s_part[warp][1] = l_ce; s_part[warp][2] = l_sse; s_part[warp][3] = l_kld; }
    __syncthreads();
    if (a.stage_a) {
        // rows b0 .. b0 + 7 (zeros beyond the batch: the grid covers the batch rounded up to a k-tile)
        const int b0 = blockIdx.x * 8, ng = (a.d_in + 3) >> 2;
        for (int q = threadIdx.x; q < ng * 8; q += 256) {
            const int g4 = q >> 3, r = q & 7;
            *reinterpret_cast<float4 *>(a.stage_a + tc::lane_major_index(b0 + r, 4 * g4, a.stage_a_ld)) =
                *reinterpret_cast<const float4 *>(&s_g[r][4 * g4]);
        }
        for (int q = threadIdx.x; q < a.d_in * 2; q += 256) {
            const int h = q / a.d_in, n = q - h * a.d_in;
            *reinterpret_cast<float4 *>(a.stage_t + tc::lane_major_index(n, b0 + 4 * h, a.stage_t_ld)) =
                make_float4(s_g[4 * h][n], s_g[4 * h + 1][n], s_g[4 * h + 2][n], s_g[4 * h + 3][n]);
        }
    }
    if (threadIdx.x < 4) {
        double t = 0.0;
        for (int w = 0; w < 8; ++w) t += s_part[w][threadIdx.x];
        a.part[(int64_t)blockIdx.x * 4 + threadIdx.x] = t;
    }
    tk_end(tk);
    if (a.fold_later) return;  // loss_fold_kernel does it off the critical path
    if (!last_block_done(&a.ctl->tickets[a.ticket_id], gridDim.x)) return;
    loss_fold(a, gridDim.x);
}

// one block: the running loss sums of the control block (read by the host once per epoch)
__global__ void __launch_bounds__(256) loss_fold_kernel(LossArgs a, int n_blocks) {
    pdl_entry();
    loss_fold(a, (unsigned)n_blocks);
}

// ------------------------------------------------------------------ backward layer (wgrad + dgrad)
struct BwdArgs {
    LdGradOut gy;         // dL/dY [B, N]
    LdInput in;           // layer input [B, K] (+ ones column at K for the bias gradient)
    const float *W;       // [N, K]
    float *gW, *gb;       // gradients [N, K], [N]
    int B, K, N;
    int wg_tiles_m, wg_tiles_n, dg_tiles_m, dg_tiles_n;  // dg_tiles_* == 0: no dgrad (first layer)
    // dgrad epilogue
    int in_kind; float *d_in;   // dL/d(input) [B, K]: dH of the previous hidden block, or dMU for z
    const float *p_prev, *mean_prev, *rstd_prev; double *part_prev; float *m1_prev, *m2_prev; float *g_gamma, *g_beta;
    const float *MU; float kld_w;
    vk_vae_ctl *ctl; int ticket_id;
    int tile_n;           // tensor-core path: output columns per dgrad CTA
    int wg_tile_n;        // ... per wgrad CTA (plain epilogue, off the critical path: wider)
    tc::OpRef wg_a, wg_b, dg_a, dg_b;  // v2: dY^T, X^T(+ones) | dY, W^T
    float *bA_prev, *bB_prev, *bC_prev; const float *gamma_prev; float inv_keep;
    // fused staging of dL/dY of the PREVIOUS layer from the dgrad tile (tensor-core path):
    // 0 off; 1 hidden layer (grid barrier over the dgrad CTAs, fold, BatchNorm/dropout/LeakyReLU backward);
    // 2 plain copy (dL/dmu)
    int stage; float *stage_a; int stage_a_ld; float *stage_t; int stage_t_ld; float slope; int has_dropout;
    int use_tma; VkTmap tm_dg_hi, tm_dg_lo;  // dgrad B operand (W^T and its tf32 remainder) through TMA
    int cluster_rt, n_wg_pad;  // cluster fold: dgrad row tiles of one column tile = one cluster; wgrad CTAs padded to whole clusters
    int b_pow2; double inv_b;  // B is a power of two; 1 / B
};

// Fold the per-row-tile column sums of dH and dH*Phat: BatchNorm weight/bias gradients and the two
// batch means the consumer needs (last block to finish).
__device__ __forceinline__ void bn_backward_finalize(const BwdArgs &a, int nthreads) {
    for (int n = threadIdx.x; n < a.K; n += nthreads) {
        double u = 0.0, v = 0.0;
#pragma unroll 8
        for (int rt = 0; rt < a.dg_tiles_m; ++rt) {
            u += __ldcg(a.part_prev + ((int64_t)rt * 2 + 0) * a.K + n);
            v += __ldcg(a.part_prev + ((int64_t)rt * 2 + 1) * a.K + n);
        }
        a.g_beta[n] = (float)u;   // d/d(beta)  = sum_b dH
        a.g_gamma[n] = (float)v;  // d/d(gamma) = sum_b dH * Phat
        a.m1_prev[n] = (float)(u / a.B);
        a.m2_prev[n] = (float)(v / a.B);
        if (a.bA_prev) {
            // dL/dY = sgn * inv_keep * gamma * rstd * (dH - m1 - (P - mean) * rstd * m2) = sgn * (bA*dH + bB*P + bC)
            const float rs = a.rstd_prev[n], mu = a.mean_prev[n];
            const float m1 = (float)(u / a.B), m2 = (float)(v / a.B);
            const float bA = a.inv_keep * a.gamma_prev[n] * rs;
            const float bB = -bA * rs * m2;
            a.bA_prev[n] = bA;
            a.bB_prev[n] = bB;
            a.bC_prev[n] = -bA * m1 - bB * mu;
        }
    }
}

__global__ void __launch_bounds__(GT) bwd_layer_kernel(BwdArgs a) {
    pdl_entry();
    __shared__ __align__(16) float s_gemm[SMEM_GEMM_FLOATS];
    __shared__ double s_red[2 * 16 * 64];
    float acc[4][4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int n_wg = a.wg_tiles_m * a.wg_tiles_n;
    if ((int)blockIdx.x < n_wg) {
        // ---- wgrad: gW[n, k] = sum_b dY[b, n] * X[b, k];  k == K -> bias gradient ----
        const int m0 = (blockIdx.x / a.wg_tiles_n) * 64, n0 = (blockIdx.x % a.wg_tiles_n) * 64;
        gemm_block<64, 64, true, true>(a.B, m0, n0, a.gy, a.in, acc, s_gemm);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int m = m0 + ty * 4 + i;
            if (m >= a.N) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int n = n0 + tx * 4 + j;
                if (n < a.K) a.gW[(int64_t)m * a.K + n] = acc[i][j];
                else if (n == a.K) a.gb[m] = acc[i][j];
            }
        }
        return;
    }
    // ---- dgrad: dX[b, k] = sum_n dY[b, n] * W[n, k] ----
    const int t = blockIdx.x - n_wg;
    const int m0 = (t / a.dg_tiles_n) * 64, n0 = (t % a.dg_tiles_n) * 64;
    LdPlain w{a.W, a.K, a.N, a.K};
    gemm_block<64, 64, false, true>(a.N, m0, n0, a.gy, w, acc, s_gemm);
    float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
    const float gsc = (float)(a.ctl->wbar / (double)a.B);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int m = m0 + ty * 4 + i;
        if (m >= a.B) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = n0 + tx * 4 + j;
            if (n >= a.K) continue;
            const int64_t o = (int64_t)m * a.K + n;
            float v = acc[i][j];
            if (a.in_kind == VK_IN_Z) {
                v = __fmaf_rn(gsc * a.kld_w, __ldg(a.MU + o), v);  // d(kld)/d(mu), encode.py:331
            } else {
                const float ph = (__ldg(a.p_prev + o) - __ldg(a.mean_prev + n)) * __ldg(a.rstd_prev + n);
                s1[j] += v;
                s2[j] = __fmaf_rn(v, ph, s2[j]);
            }
            a.d_in[o] = v;
        }
    }
    if (a.in_kind != VK_IN_BN) return;
    const int row_tile = t / a.dg_tiles_n;
    double *p0 = a.part_prev + ((int64_t)row_tile * 2 + 0) * a.K;
    double *p1 = a.part_prev + ((int64_t)row_tile * 2 + 1) * a.K;
    tile_colsum2<4>(s1, s2, s_red, p0, p1, n0, a.K);
    if (!last_block_done(&a.ctl->tickets[a.ticket_id], a.dg_tiles_m * a.dg_tiles_n)) return;
    bn_backward_finalize(a, blockDim.x);
}

// ------------------------------------------------------------------ tensor-core (wgmma, 3xTF32) layer kernels
// Same arguments and results as fwd_layer_kernel / bwd_layer_kernel; the GEMM core is the 128 x bn
// tensor-core tile of vk_tc.cuh and the epilogue goes registers -> shared tile -> global.
constexpr int TS = 132;  // padded row stride (floats) of the shared epilogue tile: conflict-free float4 rows

__device__ __forceinline__ uint8_t *align1024(uint8_t *p) {
    return reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(p) + 1023) & ~(uintptr_t)1023);
}

// Column sums of two per-element quantities over the 128 rows of the shared tile(s), in a fixed order, by ALL 256
// epilogue threads: the tile's bn columns (a multiple of 16) are covered by G = 256 / bnp row groups (bnp = bn rounded
// up to a power of two), thread (g, col) sums rows [g * 128 / G, (g + 1) * 128 / G) in double, and thread col folds the
// G partials in order.  (One thread per column would leave most threads idle at small bn: 64 serial double additions
// per column.)
// f(r, c) -> (v0, v1).  Writes out0/out1[n0 + c] for c < bn with n0 + c < N.  s_cs: 512 doubles of shared memory.
template <class F>
__device__ __forceinline__ void tc_colsum2(int bn, int n0, int N, double (*s_cs)[2][128], double *out0, double *out1,
                                           const F &f) {
    double *part = &s_cs[0][0][0];  // [G][2][bnp] with G * bnp = 256
    const int tid = threadIdx.x;
    int bnp = 16;
    while (bnp < bn) bnp <<= 1;
    const int G = 256 / bnp, rows_per = 128 / G;
    const int col = tid & (bnp - 1), g = tid / bnp;
    if (col < bn) {
        double a0 = 0.0, a1 = 0.0;
        const int r0 = g * rows_per;
#pragma unroll 4
        for (int r = r0; r < r0 + rows_per; ++r) {
            float v0, v1;
            f(r, col, v0, v1);
            a0 += (double)v0;
            a1 += (double)v1;
        }
        part[(g * 2 + 0) * bnp + col] = a0;
        part[(g * 2 + 1) * bnp + col] = a1;
    }
    __syncthreads();
    if (tid < bn && n0 + tid < N) {
        double t0 = 0.0, t1 = 0.0;
        for (int gg = 0; gg < G; ++gg) {
            t0 += part[(gg * 2 + 0) * bnp + tid];
            t1 += part[(gg * 2 + 1) * bnp + tid];
        }
        out0[n0 + tid] = t0;
        out1[n0 + tid] = t1;
    }
    __syncthreads();
}

// ---- cluster fold: BatchNorm sums exchanged through distributed shared memory ----
// When the row tiles of one column tile are a small thread-block cluster (B <= 256: 2 CTAs), the per-row-tile
// column sums never leave the SMs: every CTA leaves its two sums per column in shared memory, one hardware cluster
// barrier replaces the software grid barrier (global atomics + polling),
// and every CTA reads its peers' sums with ld.shared::cluster in the SAME order as the global fold below (identical
// doubles, identical results).  A second barrier before exit keeps the shared memory alive while peers read it.
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory"); }
__device__ __forceinline__ double dsmem_ld_f64(const double *own, unsigned rank) {
    const uint32_t la = (uint32_t)__cvta_generic_to_shared(own);
    uint32_t ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(la), "r"(rank));
    double v;
    asm volatile("ld.shared::cluster.f64 %0, [%1];" : "=d"(v) : "r"(ra) : "memory");
    return v;
}
// as fold_rowtile_sums, the partials of row tile rt being s_mine[.][col] of the cluster's CTA of rank rt.  With at most
// four row tiles every (g, col) thread of the global fold holds at most one partial (n_rt <= G), so its result is the
// plain left-to-right sum p_0 + p_1 + ...: thread col reads the 2 n_rt doubles itself (independent remote loads) -- no
// second trip through shared memory, no block barrier.  u / v are valid for tid < bn.
__device__ __forceinline__ void fold_cluster_sums(const double (*s_mine)[128], int n_rt, int N, int n0, int bn, double &u,
                                                  double &v) {
    const int tid = threadIdx.x;
    u = 0.0;
    v = 0.0;
    if (tid < bn && n0 + tid < N) {
        double p[2][4];
#pragma unroll
        for (int rt = 0; rt < 4; ++rt) {
            p[0][rt] = rt < n_rt ? dsmem_ld_f64(&s_mine[0][tid], (unsigned)rt) : 0.0;
            p[1][rt] = rt < n_rt ? dsmem_ld_f64(&s_mine[1][tid], (unsigned)rt) : 0.0;
        }
#pragma unroll
        for (int rt = 0; rt < 4; ++rt) {
            u += p[0][rt];
            v += p[1][rt];
        }
    }
}

// Fold the per-row-tile column partials of this CTA's columns over all n_rt row tiles with ALL 256 epilogue threads
// (thread (g, col) takes row tiles g, g + G, ...; thread col adds the G partials in order): u / v are valid for
// tid < bn.  A single thread per column walking 32 row tiles of L2-resident partials cost 4.8 us at B = 4096.
__device__ __forceinline__ void fold_rowtile_sums(const double *part, int n_rt, int N, int n0, int bn,
                                                  double (*s_cs)[2][128], double &u, double &v) {
    double *sp = &s_cs[0][0][0];  // [G][2][bnp], G * bnp = 256
    const int tid = threadIdx.x;
    int bnp = 16;
    while (bnp < bn) bnp <<= 1;
    const int G = 256 / bnp;
    const int col = tid & (bnp - 1), g = tid / bnp;
    double a0 = 0.0, a1 = 0.0;
    if (col < bn && n0 + col < N) {
#pragma unroll 8
        for (int rt = g; rt < n_rt; rt += G) {
            a0 += __ldcg(part + ((int64_t)rt * 2 + 0) * N + n0 + col);
            a1 += __ldcg(part + ((int64_t)rt * 2 + 1) * N + n0 + col);
        }
    }
    if (col < bn) {
        sp[(g * 2 + 0) * bnp + col] = a0;
        sp[(g * 2 + 1) * bnp + col] = a1;
    }
    __syncthreads();
    u = 0.0;
    v = 0.0;
    if (tid < bn)
        for (int gg = 0; gg < G; ++gg) {
            u += sp[(gg * 2 + 0) * bnp + tid];
            v += sp[(gg * 2 + 1) * bnp + tid];
        }
}

// ---- fused staging: the producing kernel writes the consumer GEMM's operands from its shared tile ----
// Grid barrier over `total` CTAs that are all resident (the host guarantees total <= SM count; every CTA of
// the launch is scheduled before any dependent launch).  Sense-reversing: the last arriver resets the
// counter and bumps the generation.  A lost CTA traps after ~1 s instead of hanging the device.
__device__ __forceinline__ void grid_barrier(int32_t *cnt, int32_t *gen, int total) {
    __syncthreads();
    if (threadIdx.x == 0) {
        const int g = *reinterpret_cast<volatile int32_t *>(gen);
        __threadfence();
        if (atomicAdd(cnt, 1) == total - 1) {
            atomicExch(cnt, 0);
            __threadfence();
            atomicExch(gen, g + 1);
        } else {
            unsigned spins = 0;
            while (*reinterpret_cast<volatile int32_t *>(gen) == g) {  // one thread per CTA polls: no back-off needed
                if (++spins > (1u << 26)) __trap();
            }
        }
        __threadfence();
    }
    __syncthreads();
}

// The staging passes below read the shared tile [128][TS] and write the consumer GEMM's operands.
// f(r, c, v) maps the tile value at (row r, column c) to the staged value (affine, mask); rows m0 + r,
// columns n0 + c.  Lanes are arranged so that both the shared-memory reads and the global writes of a warp
// are (nearly) conflict-free / fully coalesced.
//   lane-major A-role operand, k = column:  consecutive rows are consecutive float4
template <class F>
__device__ __forceinline__ void stage_tile_lane(const float *tile, int bn, float *dst, int ld, int m0, int n0, const F &f) {
#pragma unroll 4
    for (int q = threadIdx.x; q < (bn >> 2) * 128; q += tc::WS_EPI_THREADS) {
        const int g = q >> 7, r = q & 127;
        const float4 v = *reinterpret_cast<const float4 *>(tile + r * TS + 4 * g);
        *reinterpret_cast<float4 *>(dst + tc::lane_major_index(m0 + r, n0 + 4 * g, ld)) =
            make_float4(f(r, 4 * g, v.x), f(r, 4 * g + 1, v.y), f(r, 4 * g + 2, v.z), f(r, 4 * g + 3, v.w));
    }
}
// A warp takes 16 columns x 2 groups of 4 rows: lane = (column % 16) * 2 + (row group % 2) -- conflict-free
// shared-memory reads (bank = 16 (group % 2) + column % 16), one full 32-byte sector per column on the way out.
//   transpose as a plain K-major B-role operand dst[(n0 + c) * ld + m0 + r], columns n0 + c < n_valid
template <class F>
__device__ __forceinline__ void stage_tile_transposed_plain(const float *tile, int bn, float *dst, int ld, int m0, int n0,
                                                            int n_valid, const F &f) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll 4
    for (int t = warp; t < bn; t += 8) {  // task t: row-group pair t & 15, column block t >> 4
        const int g = (t & 15) * 2 + (lane & 1), c = (t >> 4) * 16 + (lane >> 1);
        if (n0 + c < n_valid)
            *reinterpret_cast<float4 *>(dst + (int64_t)(n0 + c) * ld + m0 + 4 * g) =
                make_float4(f(4 * g, c, tile[(4 * g) * TS + c]), f(4 * g + 1, c, tile[(4 * g + 1) * TS + c]),
                            f(4 * g + 2, c, tile[(4 * g + 2) * TS + c]), f(4 * g + 3, c, tile[(4 * g + 3) * TS + c]));
    }
}
//   transpose as a lane-major A-role operand (rows n0 + c < n_valid, k = m0 + r): consecutive columns are
//   consecutive float4
template <class F>
__device__ __forceinline__ void stage_tile_transposed_lane(const float *tile, int bn, float *dst, int ld, int m0, int n0,
                                                           int n_valid, const F &f) {
#pragma unroll 4
    for (int q = threadIdx.x; q < 32 * bn; q += tc::WS_EPI_THREADS) {
        const int g = q / bn, c = q - g * bn;
        if (n0 + c < n_valid)
            *reinterpret_cast<float4 *>(dst + tc::lane_major_index(n0 + c, m0 + 4 * g, ld)) =
                make_float4(f(4 * g, c, tile[(4 * g) * TS + c]), f(4 * g + 1, c, tile[(4 * g + 1) * TS + c]),
                            f(4 * g + 2, c, tile[(4 * g + 2) * TS + c]), f(4 * g + 3, c, tile[(4 * g + 3) * TS + c]));
    }
}

// grid: [wgrad tiles (tiles_m x tiles_n x nsplit)] + [dgrad tiles (dg_tiles_m x dg_tiles_n)], 128-row tiles
struct BwdTcExtra {
    int nsplit, k_per_split;   // split-K over the batch for wgrad
    int64_t slab;              // floats between gradient slabs
    int flush;                 // wgrad: cut the tensor-core accumulation chain every 128 batch rows (vk_tc.cuh: FLUSH)
};

// Forward layer: D = X' W^T on the tensor core, then one coalesced pass over the shared tile does bias,
// LeakyReLU, dropout (one Philox call per four outputs) / the reparameterisation, and the global stores;
// hidden layers in training add the BatchNorm column sums and the last CTA folds them.
// TMA: the weight operand through cp.async.bulk.tensor; FLUSH: accumulation chain cut every 128 K-elements (fp32 register
// sums, vk_tc.cuh) -- used for evaluation (`encode`), where the latent must stay within 1e-4 of fp32 whatever the
// depth of the layer: a shorter accumulation chain on the tensor core bounds its rounding error.  One instantiation per combination keeps every kernel's code (and its cold
// instruction-cache footprint at launch) to the path it runs.
template <bool TMA, bool FLUSH>
__global__ void __launch_bounds__(tc::WS_THREADS, 1) fwd_layer_tc_kernel(const __grid_constant__ FwdArgs a) {
    tl_begin(a.layer_id);
    const int tk = tk_begin(20 + a.layer_id);
    pdl_entry();
    tl_mark(1);
    extern __shared__ uint8_t smem_raw[];
    __shared__ tc::WsShared sh;
    __shared__ double s_cs[2][2][128];
    __shared__ __align__(16) float s_bias[128];
    uint8_t *smem = align1024(smem_raw);
    const int tid = threadIdx.x;
    const int m0 = blockIdx.y * 128, n0 = blockIdx.x * a.tile_n;
    int bn = a.N - n0;
    bn = bn > a.tile_n ? a.tile_n : ((bn + 15) & ~15);
    if (tid < bn) s_bias[tid] = n0 + tid < a.N ? __ldg(a.bias + n0 + tid) : 0.0f;
    const uint32_t k0 = (uint32_t)a.ctl->seed, k1 = (uint32_t)(a.ctl->seed >> 32);
    const uint32_t step_lo = (uint32_t)a.ctl->step, step_hi = (uint32_t)(a.ctl->step >> 32);
    const int nk = (a.K + tc::KT - 1) / tc::KT;
    tc::WsAcc acc;
    tc::ws_mainloop<TMA, FLUSH>(a.a_op.hi, a.a_op.ld, m0, a.b_op.hi, a.b_op.ld, n0, bn, 0, nk, smem, &sh, acc, a.tile_n,
                                &a.tm_b_hi, &a.tm_b_lo);
    tl_mark(2);
    float *tile = reinterpret_cast<float *>(smem);  // [128][TS]; the operand stages are dead now
    tc::ws_acc_to_tile(acc, bn, tile, TS);
    tl_mark(3);
    tc::ws_tile_end();
    tl_mark(44);

    const bool hidden = a.kind == VK_LAYER_HIDDEN, is_mu = a.kind == VK_LAYER_MU;
    const bool drop = hidden && a.training && a.dropout > 0.0f;
    const bool philox_drop = drop && a.keep == nullptr;
    const bool philox_eps = is_mu && a.add_eps && a.eps == nullptr;
    const float keep_scale = 1.0f / (1.0f - a.dropout);
    const bool vec = ((a.N & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.out) & 15) == 0);
    const int q_per_row = bn >> 2;
    // Lean pass for the case that carries the training run -- a hidden layer in training mode with on-device dropout, a
    // tile that lies fully inside [.., N) and a power-of-two tile width: the general loop below spends ~700 SASS
    // instructions per four outputs (64-bit address arithmetic for five optional outputs, per-element bounds, two inlined
    // Philox bodies, an integer division), this one ~150.  Same
    // values, same Philox stream: the keep test (float)(x >> 8) + 1) * 2^-24 > p is the integer test (x >> 8) >= floor(p 2^24).
    const bool lean = hidden && a.training && a.keep == nullptr && vec && (n0 + bn <= a.N) && ((q_per_row & (q_per_row - 1)) == 0);
    if (lean) {
        const int sh = __ffs(q_per_row) - 1;
        const uint32_t thr = (uint32_t)floor((double)a.dropout * 16777216.0);
        const uint32_t c3 = step_hi ^ ((uint32_t)(a.layer_id + 1) << 24);
        const float slope = a.slope;
        float *out_tile = a.out + (int64_t)m0 * a.N + n0;
        const int rows_in = a.B - m0;  // rows of this tile inside the batch (may exceed 128)
        const int N = a.N;
#pragma unroll 2
        for (int q = tid; q < (128 << sh); q += tc::WS_EPI_THREADS) {
            const int r = q >> sh, c = (q & (q_per_row - 1)) << 2;
            const float4 t = *reinterpret_cast<const float4 *>(tile + r * TS + c);
            const float4 bz = *reinterpret_cast<const float4 *>(s_bias + c);
            float p0 = t.x + bz.x, p1 = t.y + bz.y, p2 = t.z + bz.z, p3 = t.w + bz.w;
            p0 = p0 > 0.0f ? p0 : p0 * slope;
            p1 = p1 > 0.0f ? p1 : p1 * slope;
            p2 = p2 > 0.0f ? p2 : p2 * slope;
            p3 = p3 > 0.0f ? p3 : p3 * slope;
            if (drop) {
                uint32_t rnd[4];
                philox4x32((uint32_t)(m0 + r), (uint32_t)((n0 + c) >> 2), step_lo, c3, k0, k1, rnd);
                p0 = (rnd[0] >> 8) >= thr ? p0 * keep_scale : 0.0f;
                p1 = (rnd[1] >> 8) >= thr ? p1 * keep_scale : 0.0f;
                p2 = (rnd[2] >> 8) >= thr ? p2 * keep_scale : 0.0f;
                p3 = (rnd[3] >> 8) >= thr ? p3 * keep_scale : 0.0f;
            }
            const bool in_batch = r < rows_in;
            const float4 o = in_batch ? make_float4(p0, p1, p2, p3) : make_float4(0.f, 0.f, 0.f, 0.f);
            *reinterpret_cast<float4 *>(tile + r * TS + c) = o;
            if (in_batch) *reinterpret_cast<float4 *>(out_tile + r * N + c) = o;
        }
    } else if (a.kind == VK_LAYER_OUT && vec && (n0 + bn <= a.N) && ((q_per_row & (q_per_row - 1)) == 0)) {
        // output layer, full tile: bias and store
        const int sh = __ffs(q_per_row) - 1;
        float *out_tile = a.out + (int64_t)m0 * a.N + n0;
        const int rows_in = a.B - m0, N = a.N;
#pragma unroll 4
        for (int q = tid; q < (128 << sh); q += tc::WS_EPI_THREADS) {
            const int r = q >> sh, c = (q & (q_per_row - 1)) << 2;
            if (r >= rows_in) continue;
            const float4 t = *reinterpret_cast<const float4 *>(tile + r * TS + c);
            const float4 bz = *reinterpret_cast<const float4 *>(s_bias + c);
            *reinterpret_cast<float4 *>(out_tile + r * N + c) = make_float4(t.x + bz.x, t.y + bz.y, t.z + bz.z, t.w + bz.w);
        }
    } else
    for (int q = tid; q < 128 * q_per_row; q += tc::WS_EPI_THREADS) {
        const int r = q / q_per_row, c = (q - r * q_per_row) << 2;
        const int m = m0 + r, nb = n0 + c;
        const float4 t = *reinterpret_cast<const float4 *>(tile + r * TS + c);
        const float4 bz = *reinterpret_cast<const float4 *>(s_bias + c);
        const float y[4] = {t.x + bz.x, t.y + bz.y, t.z + bz.z, t.w + bz.w};
        float o[4], zv[4] = {0.f, 0.f, 0.f, 0.f};
        uint32_t rnd[4] = {0u, 0u, 0u, 0u};
        if (philox_drop)
            philox4x32((uint32_t)m, (uint32_t)(nb >> 2), step_lo, step_hi ^ ((uint32_t)(a.layer_id + 1) << 24), k0, k1, rnd);
        float nrm[4] = {0.f, 0.f, 0.f, 0.f};
        if (philox_eps) {  // reparameterisation noise (encode.py:277)
            philox4x32((uint32_t)m, (uint32_t)(nb >> 2), step_lo, step_hi ^ 0x7F000000u, k0, k1, rnd);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const float u1 = u32_to_unit(rnd[2 * h]), u2 = u32_to_unit(rnd[2 * h + 1]);
                const float rr = sqrtf(-2.0f * logf(u1));
                float sn, cn;
                sincosf(6.28318530717958647692f * u2, &sn, &cn);
                nrm[2 * h] = rr * cn;
                nrm[2 * h + 1] = rr * sn;
            }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const bool inside = m < a.B && nb + j < a.N;
            float p = y[j];
            if (hidden) {
                p = p > 0.0f ? p : p * a.slope;
                if (drop) {
                    bool kp;
                    if (a.keep) kp = inside && a.keep[(int64_t)m * a.N + nb + j] != 0;
                    else kp = u32_to_unit(rnd[j]) > a.dropout;
                    p = kp ? p * keep_scale : 0.0f;
                }
            } else if (is_mu && inside) {
                const int64_t oi = (int64_t)m * a.N + nb + j;
                if (a.add_eps) {
                    zv[j] = p + (a.eps ? __ldg(a.eps + oi) : nrm[j]);
                    a.z[oi] = zv[j];
                }
                if (a.latent_out) a.latent_out[oi] = __uint_as_float(__float_as_uint(p) & ~((1u << a.mask_bits) - 1u));
            }
            o[j] = inside ? p : 0.0f;
        }
        // the tile keeps what later phases need: P (column sums, staging) or z (staging of the decoder input)
        if (is_mu && a.add_eps) *reinterpret_cast<float4 *>(tile + r * TS + c) = make_float4(zv[0], zv[1], zv[2], zv[3]);
        else *reinterpret_cast<float4 *>(tile + r * TS + c) = make_float4(o[0], o[1], o[2], o[3]);
        if (m < a.B) {
            float *dst = a.out + (int64_t)m * a.N + nb;
            if (vec && nb + 3 < a.N) *reinterpret_cast<float4 *>(dst) = make_float4(o[0], o[1], o[2], o[3]);
            else {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (nb + j < a.N) dst[j] = o[j];
            }
        }
    }
    tl_mark(4);
    tk_end(tk);
    __shared__ float s_k[2][128];
    __shared__ double s_mine[2][128];  // cluster fold: this CTA's column sums, read by its cluster peers
    const bool cl_exit = hidden && a.training && a.stage == 1 && a.cluster_rt > 0;
    if (hidden && a.training) {
        __syncthreads();
        const bool cl = a.cluster_rt > 0;  // cluster fold: the sums stay in shared memory (indexed by tile column)
        double *p0 = cl ? &s_mine[0][0] - n0 : a.part + ((int64_t)blockIdx.y * 2 + 0) * a.N;
        double *p1 = cl ? &s_mine[1][0] - n0 : a.part + ((int64_t)blockIdx.y * 2 + 1) * a.N;
        tc_colsum2(bn, n0, a.N, s_cs, p0, p1, [&](int r, int c, float &v0, float &v1) {
            const float p = tile[r * TS + c];  // rows >= B and columns >= N hold zeros
            v0 = p;
            v1 = p * p;
        });
        tl_mark(5);
        if (a.stage != 1) return;  // the consumer (prep_kernel of the next layer) folds the column sums
        double sm, q;
        if (cl) {
            // the row tiles of this column tile are one cluster (cluster dims (1, gridDim.y, 1): rank = blockIdx.y)
            cluster_arrive();
            cluster_wait();
            tl_mark(6);
            fold_cluster_sums(s_mine, (int)gridDim.y, a.N, n0, bn, sm, q);
            cluster_arrive();  // this CTA has read its peers' sums; matched by the wait before exit
        } else {
            // every CTA's column sums are needed: wait for the whole grid, then fold the own columns
            grid_barrier(&a.ctl->tickets[a.layer_id], &a.ctl->barrier_gen[a.layer_id], gridDim.x * gridDim.y);
            tl_mark(6);
            fold_rowtile_sums(a.part, (int)gridDim.y, a.N, n0, bn, s_cs, sm, q);
        }
        if (tid < bn) {
            const int n = n0 + tid;
            float k0 = 0.0f, k1 = 0.0f;
            if (n < a.N) {
                // torch.nn.BatchNorm1d in training mode (as bn_forward_finalize).  fp64 divisions and square roots are
                // ~100-instruction software sequences at 1/64 rate on this part -- the fold was 2.2 us of a 15 us layer
                // kernel -- so: x / B as x * (1 / B) when B is a power of two (the same bits), one rsqrt instead of
                // sqrt + division (<= 1 ulp in double either way, rounded to float), B / (B - 1) from the host.
                const double mean = a.b_pow2 ? sm * a.inv_b : sm / a.B;
                double var = (a.b_pow2 ? q * a.inv_b : q / a.B) - mean * mean;
                if (var < 0.0) var = 0.0;
                const float rstd = (float)rsqrt(var + 1e-5);
                const float fm = (float)mean;
                k0 = a.gamma[n] * rstd;
                k1 = a.beta[n] - fm * k0;
                if (blockIdx.y == 0) {
                    a.bn_mean[n] = fm;
                    a.bn_rstd[n] = rstd;
                    a.bn_a[n] = k0;
                    a.bn_c[n] = k1;
                    const float unb = a.B > 1 ? (float)(var * a.unbias) : (float)var;
                    a.running_mean[n] = 0.9f * a.running_mean[n] + 0.1f * fm;
                    a.running_var[n] = 0.9f * a.running_var[n] + 0.1f * unb;
                    if (n == 0) *a.nbt += 1;
                }
            }
            s_k[0][tid] = k0;
            s_k[1][tid] = k1;
        }
    } else if (a.stage == 2) {
        if (tid < bn) {  // evaluation: the affine of the running statistics; z: identity
            const int n = n0 + tid;
            s_k[0][tid] = (hidden && n < a.N) ? __ldg(a.bn_a + n) : 1.0f;
            s_k[1][tid] = (hidden && n < a.N) ? __ldg(a.bn_c + n) : 0.0f;
        }
    } else {
        return;
    }
    __syncthreads();
    tl_mark(45);
    // the next layer's input X' = BatchNorm(P) (or z): the tile holds P with zeros outside [B, N]
    auto bn_apply = [&](int r, int c, float v) {
        return (m0 + r < a.B && n0 + c < a.N) ? __fmaf_rn(v, s_k[0][c], s_k[1][c]) : 0.0f;
    };
    stage_tile_lane(tile, bn, a.stage_a, a.stage_a_ld, m0, n0, bn_apply);
    if (a.stage_t) {
        stage_tile_transposed_plain(tile, bn, a.stage_t, a.stage_t_ld, m0, n0, a.N, bn_apply);
        // the row of ones that turns the bias gradient into one more column of the wgrad GEMM
        if (blockIdx.x == 0 && tid < 128) a.stage_t[(int64_t)a.N * a.stage_t_ld + m0 + tid] = m0 + tid < a.B ? 1.0f : 0.0f;
    }
    tl_mark(7);
    tk_end(tk);
    if (cl_exit) cluster_wait();  // peers may still be reading s_mine
}

// Backward layer: wgrad slices (split-K over the batch, one gradient slab per split) and dgrad tiles in
// one launch.
template <bool TMA, bool FLUSH>
__global__ void __launch_bounds__(tc::WS_THREADS, 1) bwd_layer_tc_kernel(const __grid_constant__ BwdArgs a, BwdTcExtra x) {
    tl_begin(8 + a.ticket_id);
    const int tk = tk_begin(40 + a.ticket_id);
    pdl_entry();
    tl_mark(1);
    extern __shared__ uint8_t smem_raw[];
    __shared__ tc::WsShared sh;
    __shared__ double s_cs[2][2][128];
    uint8_t *smem = align1024(smem_raw);
    const int tid = threadIdx.x;
    float *tile = reinterpret_cast<float *>(smem);
    const int n_wg = a.wg_tiles_m * a.wg_tiles_n * x.nsplit;
    const bool cl = a.cluster_rt > 0;
    if (cl && (int)blockIdx.x >= n_wg && (int)blockIdx.x < a.n_wg_pad) return;  // padding up to whole clusters
    if ((int)blockIdx.x < n_wg) {
        // ---- wgrad slice: gW[n, k] (+ bias column) over batch rows [b0, b0 + nb) ----
        const int split = blockIdx.x / (a.wg_tiles_m * a.wg_tiles_n);
        const int t = blockIdx.x % (a.wg_tiles_m * a.wg_tiles_n);
        const int m0 = (t / a.wg_tiles_n) * 128, n0 = (t % a.wg_tiles_n) * a.wg_tile_n;
        int bn = a.K + 1 - n0;
        bn = bn > a.wg_tile_n ? a.wg_tile_n : ((bn + 15) & ~15);
        const int b0 = split * x.k_per_split;
        int nb = a.B - b0;
        nb = nb < 0 ? 0 : (nb > x.k_per_split ? x.k_per_split : nb);
        const int nk = (nb + tc::KT - 1) / tc::KT;  // b0 is a multiple of 32; the staged operands are zero padded
        tc::WsAcc acc;
        tc::ws_mainloop<false, FLUSH>(a.wg_a.hi, a.wg_a.ld, m0, a.wg_b.hi, a.wg_b.ld, n0, bn, b0 / tc::KT, nk, smem, &sh, acc);
        tl_mark(2);
        tc::ws_acc_to_tile(acc, bn, tile, TS);
        tl_mark(3);
        tc::ws_tile_end();
        float *gW = a.gW + (int64_t)split * x.slab, *gb = a.gb + (int64_t)split * x.slab;
        for (int q = tid; q < 128 * bn; q += tc::WS_EPI_THREADS) {
            const int r = q / bn, c = q - r * bn;
            const int m = m0 + r, n = n0 + c;
            if (m >= a.N) continue;
            const float val = tile[r * TS + c];
            if (n < a.K) gW[(int64_t)m * a.K + n] = val;
            else if (n == a.K) gb[m] = val;
        }
        tl_mark(4);
        tk_end(tk);
        return;
    }
    // ---- dgrad: dX[b, k] = sum_n dY[b, n] * W[n, k] ----
    // cluster fold: clusters of cluster_rt consecutive CTAs = the row tiles of one column tile (rank = row tile)
    const int t = blockIdx.x - (cl ? a.n_wg_pad : n_wg);
    const int row_tile = cl ? t % a.cluster_rt : t / a.dg_tiles_n, col_tile = cl ? t / a.cluster_rt : t % a.dg_tiles_n;
#define TLD(slot) do { if (t == 0) tl_mark_any(slot); } while (0)
    TLD(1);
    const int m0 = row_tile * 128, n0 = col_tile * a.tile_n;
    int bn = a.K - n0;
    bn = bn > a.tile_n ? a.tile_n : ((bn + 15) & ~15);
    const float gsc = (float)(a.ctl->wbar / (double)a.B);
    const int nk = (a.N + tc::KT - 1) / tc::KT;
    tc::WsAcc acc;
    tc::ws_mainloop<TMA, false>(a.dg_a.hi, a.dg_a.ld, m0, a.dg_b.hi, a.dg_b.ld, n0, bn, 0, nk, smem, &sh, acc, a.tile_n,
                                &a.tm_dg_hi, &a.tm_dg_lo);
    TLD(2);
    const int q_per_row = bn >> 2;
    float *ptile = tile + 128 * TS;  // the previous layer's output P for the same rows / columns (zeros outside)
    // Lean epilogue passes (hidden layer below, full tile, power-of-two width, aligned rows): shifts instead of
    // divisions, one row predicate instead of per-element bounds, 32-bit offsets from a tile pointer -- same values.
    const bool lean_d = a.in_kind == VK_IN_BN && ((a.K & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.p_prev) & 15) == 0) &&
                        ((reinterpret_cast<uintptr_t>(a.d_in) & 15) == 0) && (n0 + bn <= a.K) &&
                        ((q_per_row & (q_per_row - 1)) == 0);
    const int sh_d = __ffs(q_per_row) - 1, rows_in_d = a.B - m0;
    if (lean_d) {
        const float *p_tile = a.p_prev + (int64_t)m0 * a.K + n0;
        const int K = a.K;
#pragma unroll 4
        for (int q = tid; q < (128 << sh_d); q += tc::WS_EPI_THREADS) {
            const int r = q >> sh_d, c = (q & (q_per_row - 1)) << 2;
            float4 pv = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r < rows_in_d) pv = __ldg(reinterpret_cast<const float4 *>(p_tile + r * K + c));
            *reinterpret_cast<float4 *>(ptile + r * TS + c) = pv;
        }
    } else if (a.in_kind == VK_IN_BN) {
        const bool pvec = ((a.K & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.p_prev) & 15) == 0);
#pragma unroll 4
        for (int q = tid; q < 128 * q_per_row; q += tc::WS_EPI_THREADS) {
            const int r = q / q_per_row, c = (q - r * q_per_row) << 2;
            const int m = m0 + r, nb = n0 + c;
            float4 pv = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m < a.B) {
                const float *src = a.p_prev + (int64_t)m * a.K + nb;
                if (pvec && nb + 3 < a.K) pv = __ldg(reinterpret_cast<const float4 *>(src));
                else {
                    if (nb < a.K) pv.x = __ldg(src);
                    if (nb + 1 < a.K) pv.y = __ldg(src + 1);
                    if (nb + 2 < a.K) pv.z = __ldg(src + 2);
                    if (nb + 3 < a.K) pv.w = __ldg(src + 3);
                }
            }
            *reinterpret_cast<float4 *>(ptile + r * TS + c) = pv;
        }
    }
    tc::ws_acc_to_tile(acc, bn, tile, TS);
    tc::ws_tile_end();
    TLD(3);
    const bool vec = ((a.K & 3) == 0) && ((reinterpret_cast<uintptr_t>(a.d_in) & 15) == 0);
    const bool add_kld = a.in_kind == VK_IN_Z;
    if (lean_d) {
        float *d_tile = a.d_in + (int64_t)m0 * a.K + n0;
        const int K = a.K;
#pragma unroll 4
        for (int q = tid; q < (128 << sh_d); q += tc::WS_EPI_THREADS) {
            const int r = q >> sh_d, c = (q & (q_per_row - 1)) << 2;
            if (r < rows_in_d) *reinterpret_cast<float4 *>(d_tile + r * K + c) = *reinterpret_cast<const float4 *>(tile + r * TS + c);
            else *reinterpret_cast<float4 *>(tile + r * TS + c) = make_float4(0.f, 0.f, 0.f, 0.f);
        }
    } else
    for (int q = tid; q < 128 * q_per_row; q += tc::WS_EPI_THREADS) {
        const int r = q / q_per_row, c = (q - r * q_per_row) << 2;
        const int m = m0 + r, nb = n0 + c;
        const float4 tv = *reinterpret_cast<const float4 *>(tile + r * TS + c);
        float o[4] = {tv.x, tv.y, tv.z, tv.w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const bool inside = m < a.B && nb + j < a.K;
            if (add_kld && inside) o[j] = __fmaf_rn(gsc * a.kld_w, __ldg(a.MU + (int64_t)m * a.K + nb + j), o[j]);
            o[j] = inside ? o[j] : 0.0f;
        }
        *reinterpret_cast<float4 *>(tile + r * TS + c) = make_float4(o[0], o[1], o[2], o[3]);
        if (m < a.B) {
            float *dst = a.d_in + (int64_t)m * a.K + nb;
            if (vec && nb + 3 < a.K) *reinterpret_cast<float4 *>(dst) = make_float4(o[0], o[1], o[2], o[3]);
            else {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (nb + j < a.K) dst[j] = o[j];
            }
        }
    }
    TLD(4);
    __shared__ __align__(16) float s_k[3][128];
    __shared__ double s_mine[2][128];  // cluster fold: this CTA's column sums, read by its cluster peers
    if (a.in_kind == VK_IN_BN) {
        __syncthreads();
        double *p0 = cl ? &s_mine[0][0] - n0 : a.part_prev + ((int64_t)row_tile * 2 + 0) * a.K;
        double *p1 = cl ? &s_mine[1][0] - n0 : a.part_prev + ((int64_t)row_tile * 2 + 1) * a.K;
        tc_colsum2(bn, n0, a.K, s_cs, p0, p1, [&](int r, int c, float &v0, float &v1) {
            const float dv = tile[r * TS + c];
            float ph = 0.0f;
            if (m0 + r < a.B && n0 + c < a.K)
                ph = (ptile[r * TS + c] - __ldg(a.mean_prev + n0 + c)) * __ldg(a.rstd_prev + n0 + c);
            v0 = dv;
            v1 = dv * ph;
        });
        TLD(5);
        if (a.stage != 1) return;  // the consumer (prep_kernel staging dL/dY of the previous layer) folds the sums
        double u, v;
        if (cl) {
            cluster_arrive();
            cluster_wait();
            TLD(6);
            fold_cluster_sums(s_mine, a.dg_tiles_m, a.K, n0, bn, u, v);
            cluster_arrive();  // matched by the wait before exit
        } else {
            grid_barrier(&a.ctl->tickets[a.ticket_id], &a.ctl->barrier_gen[a.ticket_id - 1], a.dg_tiles_m * a.dg_tiles_n);
            TLD(6);
            fold_rowtile_sums(a.part_prev, a.dg_tiles_m, a.K, n0, bn, s_cs, u, v);
        }
        if (tid < bn) {
            const int n = n0 + tid;
            float k0 = 0.0f, k1 = 0.0f, k2 = 0.0f;
            if (n < a.K) {
                // BatchNorm weight / bias gradients and the folded dL/dY constants (as bn_backward_finalize)
                const float rs = a.rstd_prev[n], mu = a.mean_prev[n];
                const float m1 = (float)(a.b_pow2 ? u * a.inv_b : u / a.B), m2 = (float)(a.b_pow2 ? v * a.inv_b : v / a.B);
                k0 = a.inv_keep * a.gamma_prev[n] * rs;
                k1 = -k0 * rs * m2;
                k2 = -k0 * m1 - k1 * mu;
                if (row_tile == 0) {
                    a.g_beta[n] = (float)u;
                    a.g_gamma[n] = (float)v;
                    a.m1_prev[n] = m1;
                    a.m2_prev[n] = m2;
                    a.bA_prev[n] = k0;
                    a.bB_prev[n] = k1;
                    a.bC_prev[n] = k2;
                }
            }
            s_k[0][tid] = k0;
            s_k[1][tid] = k1;
            s_k[2][tid] = k2;
        }
        __syncthreads();
        TLD(45);
        // dL/dY of the previous layer = sgn(P) * (bA dH + bB P + bC), 0 for dropped units, replaces dH in the tile
        if (lean_d) {
            const float slope = a.slope;
            const bool hd = a.has_dropout != 0;
#pragma unroll 4
            for (int q = tid; q < (128 << sh_d); q += tc::WS_EPI_THREADS) {
                const int r = q >> sh_d, c = (q & (q_per_row - 1)) << 2;
                const float4 p4 = *reinterpret_cast<const float4 *>(ptile + r * TS + c);
                const float4 dh = *reinterpret_cast<const float4 *>(tile + r * TS + c);
                const float4 k0 = *reinterpret_cast<const float4 *>(&s_k[0][c]), k1 = *reinterpret_cast<const float4 *>(&s_k[1][c]),
                             k2 = *reinterpret_cast<const float4 *>(&s_k[2][c]);
                float v0 = __fmaf_rn(k0.x, dh.x, __fmaf_rn(k1.x, p4.x, k2.x)), v1 = __fmaf_rn(k0.y, dh.y, __fmaf_rn(k1.y, p4.y, k2.y));
                float v2 = __fmaf_rn(k0.z, dh.z, __fmaf_rn(k1.z, p4.z, k2.z)), v3 = __fmaf_rn(k0.w, dh.w, __fmaf_rn(k1.w, p4.w, k2.w));
                v0 = p4.x > 0.0f ? v0 : v0 * slope;
                v1 = p4.y > 0.0f ? v1 : v1 * slope;
                v2 = p4.z > 0.0f ? v2 : v2 * slope;
                v3 = p4.w > 0.0f ? v3 : v3 * slope;
                const bool in_b = r < rows_in_d;
                *reinterpret_cast<float4 *>(tile + r * TS + c) =
                    make_float4((in_b && !(hd && p4.x == 0.0f)) ? v0 : 0.0f, (in_b && !(hd && p4.y == 0.0f)) ? v1 : 0.0f,
                                (in_b && !(hd && p4.z == 0.0f)) ? v2 : 0.0f, (in_b && !(hd && p4.w == 0.0f)) ? v3 : 0.0f);
            }
        } else
#pragma unroll 4
        for (int q = tid; q < 128 * q_per_row; q += tc::WS_EPI_THREADS) {
            const int r = q / q_per_row, c = (q - r * q_per_row) << 2;
            const int m = m0 + r, nb = n0 + c;
            const float4 p4 = *reinterpret_cast<const float4 *>(ptile + r * TS + c);
            const float pv[4] = {p4.x, p4.y, p4.z, p4.w};
            const float4 dh = *reinterpret_cast<const float4 *>(tile + r * TS + c);
            const float dv[4] = {dh.x, dh.y, dh.z, dh.w};
            float o[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float v = __fmaf_rn(s_k[0][c + j], dv[j], __fmaf_rn(s_k[1][c + j], pv[j], s_k[2][c + j]));
                const float val = pv[j] > 0.0f ? v : v * a.slope;
                const bool live = m < a.B && nb + j < a.K && !(a.has_dropout && pv[j] == 0.0f);
                o[j] = live ? val : 0.0f;
            }
            *reinterpret_cast<float4 *>(tile + r * TS + c) = make_float4(o[0], o[1], o[2], o[3]);
        }
    } else if (a.stage != 2) {
        return;
    }
    __syncthreads();
    TLD(46);
    auto ident = [](int, int, float v) { return v; };
    stage_tile_lane(tile, bn, a.stage_a, a.stage_a_ld, m0, n0, ident);
    stage_tile_transposed_lane(tile, bn, a.stage_t, a.stage_t_ld, m0, n0, a.K, ident);
    TLD(7);
    if (cl && a.in_kind == VK_IN_BN && a.stage == 1) cluster_wait();  // peers may still be reading s_mine
#undef TLD
}


// ------------------------------------------------------------------ operand staging ("prep") kernels
// Materialise a transformed operand ONCE per layer as the plain K-major hi/lo arrays the v2 GEMM
// consumes, plus its transpose (the wgrad operands reduce over the batch, so they need the batch as
// their contiguous K dimension).  32 x 32 tiles through shared memory keep both writes coalesced.
//   mode 0: plain copy of src[rows, cols]            (weights, z, dL/dR, dL/dmu)
//   mode 1: BatchNorm on load  src * c0[col] + c1[col]
//   mode 2: dL/dY = sgn(P) * (c0*dH + c1*P + c2), 0 for dropped units   (src = dH, p = P)
//   mode 3: gathered dataset rows
struct PrepArgs {
    int mode;
    const float *src; int ld_src;
    const float *p;
    const float *c0, *c1, *c2;
    const float *data; const int64_t *rows_idx; int data_ld;
    float slope; int has_dropout;
    int rows, cols;            // logical extent
    int rows_w, cols_w;        // extent written (zeros outside the logical extent): rows_w >= rows, multiple of 32
    float *hi, *lo; int ld;    // [row][col]  (nullable)
    float *hiT, *loT; int ldT; // [col][row]  (nullable)
    int ones_row;              // transposed row `cols` = 1 for row < rows (bias-gradient column), 0 = off
    int hi_lane, hiT_lane;     // store in the lane-major layout of an A-role operand (vk_tc.cuh)
    // BatchNorm folding in the consumer: the producing GEMM leaves per-row-tile column sums in `fin_part`;
    // every block folds them for its own 32 columns (c0/c1/c2 then come from shared memory) and the first
    // row of blocks also stores what later kernels need.  fin = 0: off, 1: forward statistics (mode 1),
    // 2: backward sums (mode 2).
    int fin, fin_rt, fin_batch;
    const double *fin_part;
    const float *gamma, *beta, *mean_in, *rstd_in;
    float *bn_mean, *bn_rstd, *bn_a, *bn_c, *running_mean, *running_var; int64_t *nbt;
    float *g_gamma, *g_beta, *m1, *m2, *bA, *bB, *bC; float inv_keep;
    // mode 3 with rows_mode >= 0: the gather draws the batch itself (what batch_rows_kernel did in a launch of its own):
    // every block computes the dataset rows of its 32 batch positions; the first column of blocks also publishes them
    // (batch_rows, read by the loss kernel) and folds the batch-mean weight into ctl->wbar.
    int rows_mode; const int64_t *inject_idx; const float *weights; vk_vae_ctl *ctl; int64_t n_rows_total, row0;
    int steps_per_epoch; int64_t *rows_out; double *wpart; int ticket_id;
};

// k0/k1/k2: the per-column constants of column c (from shared memory)
__device__ __forceinline__ float prep_value(const PrepArgs &a, int r, int c, float k0, float k1, float k2,
                                            const int64_t *rows_local = nullptr, int r_local = 0) {
    if (r >= a.rows || c >= a.cols) return 0.0f;
    if (rows_local) return __ldg(a.data + rows_local[r_local] * (int64_t)a.data_ld + c);
    switch (a.mode) {
        case 0: return __ldg(a.src + (int64_t)r * a.ld_src + c);
        case 1: return __fmaf_rn(__ldg(a.src + (int64_t)r * a.ld_src + c), k0, k1);
        case 2: {
            const float pv = __ldg(a.p + (int64_t)r * a.ld_src + c);
            if (a.has_dropout && pv == 0.0f) return 0.0f;
            const float v = __fmaf_rn(k0, __ldg(a.src + (int64_t)r * a.ld_src + c), __fmaf_rn(k1, pv, k2));
            return pv > 0.0f ? v : v * a.slope;
        }
        default: return __ldg(a.data + a.rows_idx[r] * (int64_t)a.data_ld + c);
    }
}

// Per-column constants of the block's 32 columns -> s_k[0..2][32]; folds the producer's column sums when asked
// (row tiles strided over the eight warps, then the eight partial sums in fixed order).
__device__ __forceinline__ void prep_consts(const PrepArgs &a, int c0, bool first_row_block, float (*s_k)[32],
                                            double (*s_f)[8][32]) {
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int c = c0 + tx;
    if (a.fin) {
        double u = 0.0, v = 0.0;
        if (c < a.cols)
            for (int rt = ty; rt < a.fin_rt; rt += 8) {
                u += __ldcg(a.fin_part + ((int64_t)rt * 2 + 0) * a.cols + c);
                v += __ldcg(a.fin_part + ((int64_t)rt * 2 + 1) * a.cols + c);
            }
        s_f[0][ty][tx] = u;
        s_f[1][ty][tx] = v;
        __syncthreads();
    }
    if (ty == 0) {
        float k0 = 0.0f, k1 = 0.0f, k2 = 0.0f;
        double u = 0.0, v = 0.0;
        if (a.fin) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                u += s_f[0][i][tx];
                v += s_f[1][i][tx];
            }
        }
        if (c < a.cols && a.fin == 1) {
            // torch.nn.BatchNorm1d in training mode (as bn_forward_finalize)
            const double mean = u / a.fin_batch;
            double var = v / a.fin_batch - mean * mean;
            if (var < 0.0) var = 0.0;
            const float rstd = (float)(1.0 / sqrt(var + 1e-5));
            const float fm = (float)mean;
            k0 = a.gamma[c] * rstd;
            k1 = a.beta[c] - fm * k0;
            if (first_row_block) {
                a.bn_mean[c] = fm;
                a.bn_rstd[c] = rstd;
                a.bn_a[c] = k0;
                a.bn_c[c] = k1;
                const float unb = a.fin_batch > 1 ? (float)(var * ((double)a.fin_batch / (double)(a.fin_batch - 1))) : (float)var;
                a.running_mean[c] = 0.9f * a.running_mean[c] + 0.1f * fm;
                a.running_var[c] = 0.9f * a.running_var[c] + 0.1f * unb;
                if (c == 0) *a.nbt += 1;
            }
        } else if (c < a.cols && a.fin == 2) {
            // BatchNorm weight / bias gradients and the folded dL/dY constants (as bn_backward_finalize)
            const float rs = a.rstd_in[c], mu = a.mean_in[c];
            const float m1 = (float)(u / a.fin_batch), m2 = (float)(v / a.fin_batch);
            k0 = a.inv_keep * a.gamma[c] * rs;
            k1 = -k0 * rs * m2;
            k2 = -k0 * m1 - k1 * mu;
            if (first_row_block) {
                a.g_beta[c] = (float)u;
                a.g_gamma[c] = (float)v;
                a.m1[c] = m1;
                a.m2[c] = m2;
                a.bA[c] = k0;
                a.bB[c] = k1;
                a.bC[c] = k2;
            }
        } else if (c < a.cols) {
            if (a.c0) k0 = __ldg(a.c0 + c);
            if (a.c1) k1 = __ldg(a.c1 + c);
            if (a.c2) k2 = __ldg(a.c2 + c);
        }
        s_k[0][tx] = k0;
        s_k[1][tx] = k1;
        s_k[2][tx] = k2;
    }
    __syncthreads();
}

__device__ __forceinline__ void prep_tile(const PrepArgs &a, int r0, int c0, float (*tile)[33], float (*s_k)[32],
                                          const int64_t *rows_local = nullptr) {
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8 threads
    const float k0 = s_k[0][tx], k1 = s_k[1][tx], k2 = s_k[2][tx];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int r = r0 + ty * 4 + i, c = c0 + tx;
        float v = prep_value(a, r, c, k0, k1, k2, rows_local, ty * 4 + i);
        if (a.hi && !a.hi_lane && r < a.rows_w && c < a.cols_w) {
            a.hi[(int64_t)r * a.ld + c] = v;
            if (a.lo) a.lo[(int64_t)r * a.ld + c] = v - __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
        }
        tile[ty * 4 + i][tx] = v;
    }
    __syncthreads();
    if (a.hi && a.hi_lane) {
        // thread = (row tx, float4 group ty): consecutive rows are consecutive float4 of the lane-major block
        const int r = r0 + tx, c = c0 + 4 * ty;
        if (r < a.rows_w && c < a.cols_w)
            *reinterpret_cast<float4 *>(a.hi + tc::lane_major_index(r, c, a.ld)) =
                make_float4(tile[tx][4 * ty], tile[tx][4 * ty + 1], tile[tx][4 * ty + 2], tile[tx][4 * ty + 3]);
    }
    if (a.hiT && a.hiT_lane) {
        // transposed operand: row = source column, k = source row
        const int c = c0 + tx, r = r0 + 4 * ty;
        if (c < a.cols && r < a.rows_w)
            *reinterpret_cast<float4 *>(a.hiT + tc::lane_major_index(c, r, a.ldT)) =
                make_float4(tile[4 * ty][tx], tile[4 * ty + 1][tx], tile[4 * ty + 2][tx], tile[4 * ty + 3][tx]);
    } else if (a.hiT) {
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int c = c0 + ty * 4 + i, r = r0 + tx;  // transposed element (c, r)
            if (c < a.cols + (a.ones_row ? 1 : 0) && r < a.rows_w) {
                float v = tile[tx][ty * 4 + i];
                if (a.ones_row && c == a.cols) v = r < a.rows ? 1.0f : 0.0f;
                a.hiT[(int64_t)c * a.ldT + r] = v;
                if (a.loT) a.loT[(int64_t)c * a.ldT + r] = v - __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
            }
        }
    }
}

__global__ void __launch_bounds__(256) prep_kernel(PrepArgs a) {
    const int tk = tk_begin(10 + a.mode);
    pdl_entry();
    __shared__ float tile[32][33];
    __shared__ float s_k[3][32];
    __shared__ double s_f[2][8][32];
    if (a.mode == 1 || a.mode == 2) prep_consts(a, blockIdx.x * 32, blockIdx.y == 0, s_k, s_f);
    if (a.mode == 3 && a.rows_mode >= 0) {
        // the batch is drawn here: rows of this block's 32 batch positions (uniform branch for the whole block)
        __shared__ int64_t s_rows[32];
        const int tid = threadIdx.x, b = blockIdx.y * 32 + tid;
        if (tid < 32) {
            const int64_t r = b < a.rows ? batch_row_index(a.rows_mode, b, a.rows, a.inject_idx, a.ctl, a.n_rows_total, a.row0,
                                                           a.steps_per_epoch) : 0;
            s_rows[tid] = r;
            if (blockIdx.x == 0) {
                if (b < a.rows) a.rows_out[b] = r;
                double w = b < a.rows ? (double)a.weights[r] : 0.0;
                for (int o = 16; o; o >>= 1) w += __shfl_xor_sync(0xffffffffu, w, o);
                if (tid == 0) a.wpart[blockIdx.y] = w;
            }
        }
        __syncthreads();
        prep_tile(a, blockIdx.y * 32, blockIdx.x * 32, tile, s_k, s_rows);
        tk_end(tk);
        if (blockIdx.x != 0) return;
        if (!last_block_done(&a.ctl->tickets[a.ticket_id], gridDim.y)) return;
        if (tid == 0) {  // batch-mean weight: the per-32-row sums in block order (fixed order -> reproducible)
            double tot = 0.0;
            for (unsigned i = 0; i < gridDim.y; ++i) tot += __ldcg(a.wpart + i);
            a.ctl->wbar = tot / (double)a.rows;
        }
        return;
    }
    prep_tile(a, blockIdx.y * 32, blockIdx.x * 32, tile, s_k);
    tk_end(tk);
}

struct PrepMulti {
    PrepArgs l[VK_VAE_MAX_LAYERS];
    int n;
};

// every layer's weights in one launch (blockIdx.z = layer)
__global__ void __launch_bounds__(256) prep_weights_kernel(PrepMulti m) {
    const int tk = tk_begin(14);
    pdl_entry();
    __shared__ float tile[32][33];
    const PrepArgs &a = m.l[blockIdx.z];
    const int r0 = blockIdx.y * 32, c0 = blockIdx.x * 32;
    __shared__ float s_k[3][32];
    if (r0 >= a.rows_w || c0 >= a.cols + 1) return;
    prep_tile(a, r0, c0, tile, s_k);  // mode 0: the constants are not used
    tk_end(tk);
}

// ------------------------------------------------------------------ D-Adaptation Adam
// One pass over the flat arenas (dadaptation.DAdaptAdam.step with lr=1, betas=(0.9, 0.999),
// eps=1e-8, weight_decay=0, growth_rate=inf, no bias correction).  The parameter update of
// step t uses d_t; the two global sums only feed d_{t+1}, so everything fits in one kernel.
constexpr int OPT_ELEMS = 1024;  // elements per block

__global__ void __launch_bounds__(256)
dadapt_kernel(float *__restrict__ p, const float *__restrict__ g, float *__restrict__ m, float *__restrict__ v,
              float *__restrict__ s, int64_t n, double *part, vk_vae_ctl *ctl, int ticket_id, int nslab, int64_t slab) {
    const int tk = tk_begin(50);
    pdl_entry();
    __shared__ double s_a[256], s_b[256];
    const double beta1 = 0.9, beta2 = 0.999, eps = 1e-8;
    const double sqrt_beta2 = sqrt(beta2);
    const double dlr = ctl->d;  // d * lr * bias_correction with lr = 1
    const float f_beta1 = (float)beta1, f_beta2 = (float)beta2, f_sb2 = (float)sqrt_beta2;
    const float a_m = (float)(dlr * (1.0 - beta1)), a_v = (float)(1.0 - beta2), a_s = (float)(dlr * (1.0 - sqrt_beta2));
    const float f_eps = (float)eps;
    double acc_num = 0.0, acc_l1 = 0.0;
    // 4 independent elements per thread (their loads are issued together), 1024 elements per block
#pragma unroll
    for (int u = 0; u < 4; ++u) {
        const int64_t i = (int64_t)blockIdx.x * 1024 + u * 256 + threadIdx.x;
        if (i >= n) continue;
        float gi = g[i];
        for (int sl = 1; sl < nslab; ++sl) gi += g[(int64_t)sl * slab + i];  // split-K partial gradients, fixed order
        float mi = m[i], vi = v[i], si = s[i];
        const float pi = p[i];
        const float denom_old = sqrtf(vi) + f_eps;
        acc_num += (double)(gi * (si / denom_old));
        mi = __fmaf_rn(a_m, gi, mi * f_beta1);
        vi = __fmaf_rn(a_v * gi, gi, vi * f_beta2);
        si = __fmaf_rn(a_s, gi, si * f_sb2);
        acc_l1 += (double)fabsf(si);
        m[i] = mi; v[i] = vi; s[i] = si;
        p[i] = pi - mi / (sqrtf(vi) + f_eps);
    }
    {
        const double ta = block_sum256(acc_num, s_a), tb = block_sum256(acc_l1, s_b);
        if (threadIdx.x == 0) {
            part[2 * blockIdx.x] = ta;
            part[2 * blockIdx.x + 1] = tb;
        }
    }
    tk_end(tk);
    if (!last_block_done(&ctl->tickets[ticket_id], gridDim.x)) return;
    {   // fixed-order parallel fold of the block partials
        double num = 0.0, l1 = 0.0;
        for (unsigned i = threadIdx.x; i < gridDim.x; i += 256) {
            num += __ldcg(part + 2 * i);
            l1 += __ldcg(part + 2 * i + 1);
        }
        num = block_sum256(num, s_a);
        l1 = block_sum256(l1, s_b);
        if (threadIdx.x == 0) { s_a[8] = num; s_b[8] = l1; }
    }
    if (threadIdx.x == 0) {
        const double num = s_a[8], l1 = s_b[8];
        const double numerator_acum = dlr * num;
        const double num_w = sqrt_beta2 * ctl->num_w + (1.0 - sqrt_beta2) * numerator_acum;
        ctl->num_w = num_w;
        if (l1 > 0.0) {
            const double d_hat = num_w / ((1.0 - sqrt_beta2) * l1);
            if (d_hat > ctl->d) ctl->d = d_hat;  // d = max(d, min(d_hat, d * inf))
        }
        ctl->step += 1;
    }
}

__global__ void eval_affine_kernel(float *bn_a, float *bn_c, const float *gamma, const float *beta,
                                   const float *rm, const float *rv, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float sc = gamma[i] / sqrtf(rv[i] + 1e-5f);
    bn_a[i] = sc;
    bn_c[i] = beta[i] - rm[i] * sc;
}

// ------------------------------------------------------------------ host side
// Optional per-launch event marks (vk_vae_profile_step): one event before every launch.
static thread_local cudaEvent_t *g_prof_events = nullptr;
static thread_local int *g_prof_kinds = nullptr;
static thread_local int g_prof_n = 0, g_prof_cap = 0;
enum { PK_ROWS = 0, PK_FWD = 1, PK_LOSS = 2, PK_BWD = 3, PK_OPT = 4, PK_PREP = 5 };
#define PROF_MARK_K(s, kind)                                                            \
    do {                                                                                \
        if (g_prof_events && g_prof_n < g_prof_cap) {                                   \
            g_prof_kinds[g_prof_n] = (kind);                                            \
            cudaEventRecord(g_prof_events[g_prof_n++], (s));                            \
        }                                                                               \
    } while (0)

extern "C" int64_t vk_vae_sizeof(int which) {
    switch (which) {
        case 0: return (int64_t)sizeof(vk_vae);
        case 1: return (int64_t)sizeof(vk_vae_layer);
        case 2: return (int64_t)sizeof(vk_vae_ctl);
        case 3: return (int64_t)sizeof(vk_vae_inject);
    }
    return -1;
}

static int env_int_early(const char *name) {
    const char *v = getenv(name);
    return v ? atoi(v) : 0;
}

// ---- side stream: work that is off the critical path of a step (weight staging, loss bookkeeping) runs on a
// second stream, forked from / joined to the caller's stream with events (also inside a stream capture).
struct SideCtx {
    cudaStream_t side;
    cudaEvent_t fork, weights_done, loss_done, fold_done;
};
static SideCtx *g_side[64];

static SideCtx *side_ctx() {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    return g_side[dev];
}

// Create the per-device helper objects outside any stream capture (called once by the host wrapper).
extern "C" int vk_vae_init_device(void) {
    int dev = 0;
    VK_CUDA(cudaGetDevice(&dev));
    if (dev < 0 || dev >= 64 || g_side[dev]) return 0;
    static const int off = env_int_early("VK_SIDE_STREAM_OFF");
    if (off > 0) return 0;
    SideCtx *c = new SideCtx();
    VK_CUDA(cudaStreamCreateWithFlags(&c->side, cudaStreamNonBlocking));
    VK_CUDA(cudaEventCreateWithFlags(&c->fork, cudaEventDisableTiming));
    VK_CUDA(cudaEventCreateWithFlags(&c->weights_done, cudaEventDisableTiming));
    VK_CUDA(cudaEventCreateWithFlags(&c->loss_done, cudaEventDisableTiming));
    VK_CUDA(cudaEventCreateWithFlags(&c->fold_done, cudaEventDisableTiming));
    g_side[dev] = c;
    return 0;
}

static int check_net(const vk_vae *net, int batch) {
    if (!net || net->n_layers < 2 || net->n_layers > VK_VAE_MAX_LAYERS) {
        vk_set_error("vk_vae: bad layer count");
        return 1;
    }
    if (batch < 1 || batch > net->bmax) {
        vk_set_error("vk_vae: batch %d outside [1, bmax=%d]", batch, net->bmax);
        return 1;
    }
    return 0;
}

static bool use_tc(const vk_vae *net, int B) { return net->tc_min_batch > 0 && B >= net->tc_min_batch; }

static int env_int(const char *name) {
    const char *v = getenv(name);
    return v ? atoi(v) : 0;
}

static int tc_nsplit(const vk_vae *net, int B) {
    static const int forced = env_int("VK_TC_NSPLIT");  // tuning / debugging override
    if (forced > 0) return forced > net->n_grad_slabs ? net->n_grad_slabs : forced;
    int ns = B / 512;
    if (ns < 1) ns = 1;
    if (ns > net->n_grad_slabs) ns = net->n_grad_slabs;
    return ns;
}

// output columns per CTA: narrower tiles for small batches so that enough CTAs exist.  Chosen on an H100 SXM (400 W
// power limit) with tools/train_speed.py, us per step with every width forced: B = 256: 16 -> 193, 32 -> 212;
// B = 512: 32 -> 258, 64 -> 281; B = 1024: 32 / 64 -> 318 / 320; B = 2048: 64 -> 435, 128 -> 454; B = 4096: 128 -> 638,
// 64 -> 702.
static int tc_tile_n(int B) {
    static const int forced = env_int("VK_TC_TILE_N");  // tuning / debugging override
    if (forced >= 16 && forced <= 128 && (forced & 15) == 0) return forced;
    return B <= 256 ? 16 : (B <= 1024 ? 32 : (B <= 2048 ? 64 : 128));
}
// ... per wgrad CTA: their epilogue is a plain store, so wider tiles (fewer CTAs next to the dgrad ones)
static int tc_wg_tile_n(int B) {
    static const int forced = env_int("VK_TC_WG_TILE_N");
    if (forced >= 16 && forced <= 128 && (forced & 15) == 0) return forced;
    const int t = tc_tile_n(B);
    return t < 32 ? 32 : t;  // 32 for B <= 1024, the dgrad width above (tools/train_speed.py compares widths)
}

// ---- tensor-core path: operand staging + warp-specialised GEMMs ------------------------------------
static inline int r32(int v) { return (v + 31) & ~31; }
static inline int r128(int v) { return (v + 127) & ~127; }

// dynamic shared memory: the B-operand ring, and never less than the 128 x TS epilogue tile(s) (the backward
// kernel keeps a second tile: the previous layer's output)
static int tc_smem_for(int tile_n, int epi_tiles) {
    const int need = tc::ws_smem_bytes(tile_n), epi = epi_tiles * 128 * TS * 4 + 1024;
    return need > epi ? need : epi;
}

// B operand of the forward / dgrad GEMMs through TMA (needs the pre-split remainders w_lo / wt_lo); vk_vae.use_tma = 0
// keeps the cp.async ring (same results) for A/B timing.
static bool use_tma(const vk_vae *net, const vk_vae_layer &L) {
    return net->use_tma && L.w_lo != nullptr && L.wt_lo != nullptr;
}

static int tc_prepare() {
    static bool done = false;
    if (done) return 0;
#define VK_TC_ATTR(T, F)                                                                                                          \
    VK_CUDA(cudaFuncSetAttribute(fwd_layer_tc_kernel<T, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc_smem_for(128, 1))); \
    VK_CUDA(cudaFuncSetAttribute(bwd_layer_tc_kernel<T, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, tc_smem_for(128, 2)))
    VK_TC_ATTR(false, false);
    VK_TC_ATTR(false, true);
    VK_TC_ATTR(true, false);
    VK_TC_ATTR(true, true);
#undef VK_TC_ATTR
    done = true;
    return 0;
}

// Fused staging needs every CTA of a forward / dgrad grid resident at once (in-kernel grid barrier).
static bool fused_staging(const vk_vae *net, int B) {
    if (net->staging != 0) return false;
    static int n_sm = 0;
    if (n_sm == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
            n_sm = -1;
    }
    const int tile_n = tc_tile_n(B), rt = (B + 127) / 128;
    for (int j = 0; j < net->n_layers; ++j) {
        const vk_vae_layer &L = net->layers[j];
        const int widest = L.n_out > L.k_in ? L.n_out : L.k_in;
        if (((widest + tile_n - 1) / tile_n) * rt > n_sm) return false;
    }
    return true;
}

// Cluster fold (see fold_cluster_sums): on for 2 row tiles (129 <= B <= 256) unless VK_CLUSTER_FOLD=0.  Larger clusters of
// co-scheduled 1-CTA-per-SM blocks are harder to place on a GPC than the software barrier they replace costs: on an
// H100 SXM (400 W power limit, tools/train_speed.py, us per step, cluster fold / grid barrier) B = 256: 195 / 208, but
// B = 512 (clusters of 4): 257 / 248.
static int cluster_fold_rt(int B) {
    static const int on = [] {
        const char *v = getenv("VK_CLUSTER_FOLD");
        return v ? atoi(v) : 1;
    }();
    const int rt = (B + 127) / 128;
    return (on && rt == 2) ? rt : 0;
}

static int launch_prep(const PrepArgs &a, cudaStream_t s) {
    const int cx = a.cols + (a.ones_row ? 1 : 0);
    dim3 grid((cx + 31) / 32, (a.rows_w + 31) / 32);
    PROF_MARK_K(s, PK_PREP);
    VK_CUDA(vk_launch(prep_kernel, dim3(grid), dim3(256), (size_t)(0), s, a));
    VK_LAUNCH_CHECK();
    return 0;
}

// stage the input of layer j (A of its forward GEMM; its transpose is B of its wgrad)
// How the batch of the current step is drawn (consumed by the gather of layer 0 on the tensor-core path, which replaces
// the batch_rows launch): mode < 0 = batch_rows already holds the rows.
struct BatchDraw {
    int mode = -1;
    int64_t row0 = 0;
    const vk_vae_inject *inj = nullptr;
};

static int launch_prep_input(const vk_vae *net, int j, int B, int training, cudaStream_t s, const BatchDraw *draw = nullptr) {
    const vk_vae_layer &L = net->layers[j];
    PrepArgs a;
    memset(&a, 0, sizeof(a));
    a.rows_mode = -1;
    a.rows = B; a.cols = L.k_in; a.rows_w = r128(B); a.cols_w = L.k_in;
    a.hi = L.xop_hi; a.lo = nullptr; a.ld = r32(L.k_in); a.hi_lane = 1;  // A of the forward GEMM
    if (training) { a.hiT = L.xt_hi; a.loT = nullptr; a.ldT = net->bmax; a.ones_row = 1; }
    if (L.in_kind == VK_IN_DATA) {
        a.mode = 3; a.data = net->data; a.rows_idx = net->batch_rows; a.data_ld = net->data_ld;
        if (draw && draw->mode >= 0) {
            const int64_t n = net->n_rows;
            a.rows_mode = draw->mode; a.inject_idx = draw->inj ? draw->inj->batch_idx : nullptr;
            a.weights = net->weights; a.ctl = net->ctl; a.n_rows_total = n; a.row0 = draw->row0;
            a.steps_per_epoch = n > B ? (int)(n / B) : 1;
            a.rows_out = net->batch_rows;
            a.wpart = net->opt_part + 2 * ((net->n_params + OPT_ELEMS - 1) / OPT_ELEMS);  // bmax / 32 + 8 doubles
            a.ticket_id = 2 * VK_VAE_MAX_LAYERS + 3;
        }
    } else if (L.in_kind == VK_IN_BN) {
        const vk_vae_layer &P = net->layers[j - 1];
        a.mode = 1; a.src = P.act; a.ld_src = P.n_out; a.c0 = P.bn_a; a.c1 = P.bn_c;
        if (training) {  // fold the batch statistics the forward GEMM of layer j - 1 left behind
            a.fin = 1; a.fin_rt = (B + 127) / 128; a.fin_batch = B; a.fin_part = P.fwd_part;
            a.gamma = net->params + P.g_off; a.beta = net->params + P.beta_off;
            a.bn_mean = P.bn_mean; a.bn_rstd = P.bn_rstd; a.bn_a = P.bn_a; a.bn_c = P.bn_c;
            a.running_mean = P.running_mean; a.running_var = P.running_var; a.nbt = P.num_batches_tracked;
        }
    } else {
        a.mode = 0; a.src = net->z; a.ld_src = L.k_in;
    }
    return launch_prep(a, s);
}

// stage dL/dY of layer j (A of its dgrad; its transpose is A of its wgrad)
static int launch_prep_grad(const vk_vae *net, int j, int B, cudaStream_t s) {
    const vk_vae_layer &L = net->layers[j];
    PrepArgs a;
    memset(&a, 0, sizeof(a));
    a.rows = B; a.cols = L.n_out; a.rows_w = r128(B); a.cols_w = L.n_out;
    a.hi = L.dy_hi; a.lo = nullptr; a.ld = r32(L.n_out); a.hi_lane = 1;
    a.hiT = L.dyt_hi; a.loT = nullptr; a.ldT = net->bmax; a.hiT_lane = 1;
    a.src = L.dact; a.ld_src = L.n_out;
    if (L.kind == VK_LAYER_HIDDEN) {
        a.mode = 2; a.p = L.act; a.c0 = L.bn_bA; a.c1 = L.bn_bB; a.c2 = L.bn_bC;
        a.slope = net->slope; a.has_dropout = net->dropout > 0.0f ? 1 : 0;
        // fold the column sums the dgrad of layer j + 1 left behind
        a.fin = 2; a.fin_rt = (B + 127) / 128; a.fin_batch = B; a.fin_part = L.bwd_part;
        a.gamma = net->params + L.g_off; a.mean_in = L.bn_mean; a.rstd_in = L.bn_rstd;
        a.g_gamma = net->grads + L.g_off; a.g_beta = net->grads + L.beta_off;
        a.m1 = L.bn_m1; a.m2 = L.bn_m2; a.bA = L.bn_bA; a.bB = L.bn_bB; a.bC = L.bn_bC;
        a.inv_keep = net->dropout > 0.0f ? 1.0f / (1.0f - net->dropout) : 1.0f;
    }
    return launch_prep(a, s);
}

static int launch_prep_weights(const vk_vae *net, cudaStream_t s) {
    PrepMulti m;
    memset(&m, 0, sizeof(m));
    m.n = net->n_layers;
    int gx = 1, gy = 1;
    for (int j = 0; j < net->n_layers; ++j) {
        const vk_vae_layer &L = net->layers[j];
        PrepArgs &a = m.l[j];
        a.mode = 0; a.src = net->params + L.w_off; a.ld_src = L.k_in;
        a.rows = L.n_out; a.cols = L.k_in; a.rows_w = r32(L.n_out); a.cols_w = L.k_in;
        a.hi = L.w_hi; a.lo = L.w_lo; a.ld = r32(L.k_in);        // the remainders feed the TMA path (nullable)
        a.hiT = L.wt_hi; a.loT = L.wt_lo; a.ldT = r32(L.n_out);
        gx = gx > (L.k_in + 32) / 32 ? gx : (L.k_in + 32) / 32;
        gy = gy > a.rows_w / 32 ? gy : a.rows_w / 32;
    }
    PROF_MARK_K(s, PK_PREP);
    VK_CUDA(vk_launch(prep_weights_kernel, dim3(dim3(gx, gy, net->n_layers)), dim3(256), (size_t)(0), s, m));
    VK_LAUNCH_CHECK();
    return 0;
}

static LdInput make_input(const vk_vae *net, int j, int B, int ones_col) {
    const vk_vae_layer &L = net->layers[j];
    LdInput in;
    in.in_kind = L.in_kind;
    in.ones_col = ones_col;
    in.d = LdData{net->data, net->batch_rows, net->data_ld, B, L.k_in};
    in.a = LdAffine{nullptr, nullptr, nullptr, L.k_in, B, L.k_in};
    in.z = LdPlain{net->z, L.k_in, B, L.k_in};
    if (L.in_kind == VK_IN_BN) {
        const vk_vae_layer &P = net->layers[j - 1];
        in.a = LdAffine{P.act, P.bn_a, P.bn_c, P.n_out, B, L.k_in};
    }
    return in;
}

static int launch_batch_rows(const vk_vae *net, int B, int mode, int64_t row0, const vk_vae_inject *inj,
                             cudaStream_t s) {
    const int64_t n = net->n_rows;
    const int spe = n > B ? (int)(n / B) : 1;
    PROF_MARK_K(s, PK_ROWS);
    VK_CUDA(vk_launch(batch_rows_kernel, dim3((B + 255) / 256), dim3(256), (size_t)(0), s, net->batch_rows, inj ? inj->batch_idx : nullptr, net->weights,
                                                       net->ctl, B, n, mode, row0, spe,
                                                       net->opt_part + 2 * ((net->n_params + OPT_ELEMS - 1) / OPT_ELEMS),
                                                       2 * VK_VAE_MAX_LAYERS + 3));
    VK_LAUNCH_CHECK();
    return 0;
}

static int launch_forward(const vk_vae *net, int B, int training, int upto /*exclusive layer index*/,
                          const vk_vae_inject *inj, int mask_bits, float *latent_out, cudaStream_t s,
                          cudaEvent_t weights_ready = nullptr, const BatchDraw *draw = nullptr) {
    for (int j = 0; j < upto; ++j) {
        const vk_vae_layer &L = net->layers[j];
        FwdArgs a;
        memset(&a, 0, sizeof(a));
        a.in = make_input(net, j, B, -1);
        a.W = net->params + L.w_off;
        a.bias = net->params + L.b_off;
        a.B = B; a.K = L.k_in; a.N = L.n_out; a.kind = L.kind; a.training = training;
        a.out = L.act;
        a.dropout = net->dropout;
        a.keep = (inj && L.kind == VK_LAYER_HIDDEN) ? inj->keep[j] : nullptr;
        a.part = L.fwd_part;
        a.bn_a = L.bn_a; a.bn_c = L.bn_c; a.bn_mean = L.bn_mean; a.bn_rstd = L.bn_rstd;
        if (L.kind == VK_LAYER_HIDDEN) {
            a.gamma = net->params + L.g_off;
            a.beta = net->params + L.beta_off;
        }
        a.running_mean = L.running_mean; a.running_var = L.running_var; a.nbt = L.num_batches_tracked;
        a.z = net->z;
        a.eps = inj ? inj->eps : nullptr;
        a.add_eps = (L.kind == VK_LAYER_MU && latent_out == nullptr) ? 1 : 0;
        a.mask_bits = mask_bits;
        a.latent_out = (L.kind == VK_LAYER_MU) ? latent_out : nullptr;
        a.ctl = net->ctl; a.layer_id = j; a.slope = net->slope;
        a.b_pow2 = (B & (B - 1)) == 0; a.inv_b = 1.0 / (double)B; a.unbias = B > 1 ? (double)B / (double)(B - 1) : 1.0;
        const bool tcp = use_tc(net, B);
        const bool fused = tcp && fused_staging(net, B);
        if (tcp && (!fused || j == 0))  // fused: layer j - 1 staged this layer's operands from its output tile
            if (launch_prep_input(net, j, B, training, s, j == 0 ? draw : nullptr)) return 1;
        if (fused && j + 1 < upto && L.kind != VK_LAYER_OUT) {
            const vk_vae_layer &Nx = net->layers[j + 1];
            a.stage = (L.kind == VK_LAYER_HIDDEN && training) ? 1 : 2;
            a.stage_a = Nx.xop_hi; a.stage_a_ld = r32(Nx.k_in);
            a.stage_t = training ? Nx.xt_hi : nullptr; a.stage_t_ld = net->bmax;
        }
        if (j == 0 && weights_ready) VK_CUDA(cudaStreamWaitEvent(s, weights_ready, 0));  // staged on the side stream
        PROF_MARK_K(s, PK_FWD);
        if (tcp) {
            if (tc_prepare()) return 1;
            a.tile_n = tc_tile_n(B);
            a.a_op = tc::OpRef{L.xop_hi, L.xop_lo, r32(L.k_in)};
            a.b_op = tc::OpRef{L.w_hi, L.w_lo, r32(L.k_in)};
            a.use_tma = use_tma(net, L) ? 1 : 0;
            if (a.use_tma && (vk_make_tmap_2d(&a.tm_b_hi, L.w_hi, r32(L.k_in), r128(L.n_out), a.tile_n) ||
                              vk_make_tmap_2d(&a.tm_b_lo, L.w_lo, r32(L.k_in), r128(L.n_out), a.tile_n)))
                return 1;
            dim3 grid((L.n_out + a.tile_n - 1) / a.tile_n, (B + 127) / 128);
            // evaluation (encode): the flushed accumulation keeps the latent within 1e-4 of fp32 (net->wgrad_flush == 2
            // forces it in training too, for measurements)
            const bool flush = !training || net->wgrad_flush == 2;
            const size_t smem = (size_t)tc_smem_for(a.tile_n, 1);
            a.cluster_rt = (a.stage == 1 && L.kind == VK_LAYER_HIDDEN && training) ? cluster_fold_rt(B) : 0;
            if (a.cluster_rt) {
                const dim3 cluster(1, a.cluster_rt, 1);
                if (a.use_tma) {
                    if (flush) VK_CUDA(vk_launch_cluster(fwd_layer_tc_kernel<true, true>, dim3(grid), dim3(tc::WS_THREADS), smem, s, cluster, a));
                    else VK_CUDA(vk_launch_cluster(fwd_layer_tc_kernel<true, false>, dim3(grid), dim3(tc::WS_THREADS), smem, s, cluster, a));
                } else {
                    if (flush) VK_CUDA(vk_launch_cluster(fwd_layer_tc_kernel<false, true>, dim3(grid), dim3(tc::WS_THREADS), smem, s, cluster, a));
                    else VK_CUDA(vk_launch_cluster(fwd_layer_tc_kernel<false, false>, dim3(grid), dim3(tc::WS_THREADS), smem, s, cluster, a));
                }
            } else if (a.use_tma) {
                if (flush) VK_CUDA(vk_launch(fwd_layer_tc_kernel<true, true>, dim3(grid), dim3(tc::WS_THREADS), smem, s, a));
                else VK_CUDA(vk_launch(fwd_layer_tc_kernel<true, false>, dim3(grid), dim3(tc::WS_THREADS), smem, s, a));
            } else {
                if (flush) VK_CUDA(vk_launch(fwd_layer_tc_kernel<false, true>, dim3(grid), dim3(tc::WS_THREADS), smem, s, a));
                else VK_CUDA(vk_launch(fwd_layer_tc_kernel<false, false>, dim3(grid), dim3(tc::WS_THREADS), smem, s, a));
            }
        } else {
            dim3 grid((L.n_out + 63) / 64, (B + 63) / 64);
            VK_CUDA(vk_launch(fwd_layer_kernel, dim3(grid), dim3(GT), (size_t)(0), s, a));
        }
        VK_LAUNCH_CHECK();
    }
    return 0;
}

static int launch_loss(const vk_vae *net, int B, int write_grad, cudaStream_t s, SideCtx *sc = nullptr) {
    const int nl = net->n_layers;
    int mu_j = -1;
    for (int j = 0; j < nl; ++j)
        if (net->layers[j].kind == VK_LAYER_MU) mu_j = j;
    LossArgs a;
    a.R = net->layers[nl - 1].act; a.MU = net->layers[mu_j].act; a.data = net->data; a.batch_rows = net->batch_rows;
    a.dR = net->layers[nl - 1].dact;
    a.B = B; a.S = net->nsamples; a.ntnf = net->ntnf; a.d_in = net->d_in; a.nlatent = net->nlatent;
    a.data_ld = net->data_ld;
    a.ce_w = net->ce_w; a.ab_w = net->ab_w; a.sse_w = net->sse_w; a.kld_w = net->kld_w;
    a.part = net->loss_part; a.ctl = net->ctl; a.ticket_id = VK_VAE_MAX_LAYERS; a.write_grad = write_grad;
    a.stage_a = a.stage_t = nullptr; a.stage_a_ld = a.stage_t_ld = 0;
    a.fold_later = sc ? 1 : 0;
    int blocks = (B + 7) / 8;
    if (write_grad && use_tc(net, B) && fused_staging(net, B) && net->d_in <= LOSS_STAGE_MAX_D) {
        const vk_vae_layer &L = net->layers[nl - 1];
        a.stage_a = L.dy_hi; a.stage_a_ld = r32(L.n_out);
        a.stage_t = L.dyt_hi; a.stage_t_ld = net->bmax;
        blocks = r32(B) / 8;  // whole k-tiles of the wgrad reduction: rows beyond the batch are staged as zeros
    }
    // loss_part holds 4 doubles per 8-row block of the largest batch (r32(bmax) / 8 blocks): vk_vae.loss_part
    PROF_MARK_K(s, PK_LOSS);
    VK_CUDA(vk_launch(loss_kernel, dim3(blocks), dim3(256), (size_t)(0), s, a));
    VK_LAUNCH_CHECK();
    if (sc) {  // the running loss sums are bookkeeping: fold them next to the backward pass
        VK_CUDA(cudaEventRecord(sc->loss_done, s));
        VK_CUDA(cudaStreamWaitEvent(sc->side, sc->loss_done, 0));
        VK_CUDA(vk_launch(loss_fold_kernel, dim3(1), dim3(256), (size_t)(0), sc->side, a, blocks));
        VK_LAUNCH_CHECK();
        VK_CUDA(cudaEventRecord(sc->fold_done, sc->side));
    }
    return 0;
}

static int launch_backward(const vk_vae *net, int B, cudaStream_t s) {
    const int nl = net->n_layers;
    int mu_j = -1;
    for (int j = 0; j < nl; ++j)
        if (net->layers[j].kind == VK_LAYER_MU) mu_j = j;
    for (int j = nl - 1; j >= 0; --j) {
        const vk_vae_layer &L = net->layers[j];
        BwdArgs a;
        memset(&a, 0, sizeof(a));
        a.gy.hidden = (L.kind == VK_LAYER_HIDDEN);
        a.gy.pl = LdPlain{L.dact, L.n_out, B, L.n_out};
        if (a.gy.hidden) {
            a.gy.h = LdDY{L.dact, L.act, net->params + L.g_off, L.bn_mean, L.bn_rstd, L.bn_m1, L.bn_m2,
                          L.n_out, B, L.n_out, net->dropout > 0.0f ? 1.0f / (1.0f - net->dropout) : 1.0f,
                          net->slope, net->dropout > 0.0f ? 1 : 0};
        }
        a.in = make_input(net, j, B, L.k_in);
        a.W = net->params + L.w_off;
        a.gW = net->grads + L.w_off;
        a.gb = net->grads + L.b_off;
        a.B = B; a.K = L.k_in; a.N = L.n_out;
        a.b_pow2 = (B & (B - 1)) == 0; a.inv_b = 1.0 / (double)B;
        a.wg_tiles_m = (L.n_out + 63) / 64;
        a.wg_tiles_n = (L.k_in + 1 + 63) / 64;
        a.in_kind = L.in_kind;
        a.ctl = net->ctl;
        a.ticket_id = VK_VAE_MAX_LAYERS + 1 + j;
        if (L.in_kind == VK_IN_DATA) {
            a.dg_tiles_m = a.dg_tiles_n = 0;
        } else {
            a.dg_tiles_m = (B + 63) / 64;
            a.dg_tiles_n = (L.k_in + 63) / 64;
            if (L.in_kind == VK_IN_BN) {
                const vk_vae_layer &P = net->layers[j - 1];
                a.d_in = P.dact; a.p_prev = P.act; a.mean_prev = P.bn_mean; a.rstd_prev = P.bn_rstd;
                a.part_prev = P.bwd_part; a.m1_prev = P.bn_m1; a.m2_prev = P.bn_m2;
                a.g_gamma = net->grads + P.g_off; a.g_beta = net->grads + P.beta_off;
                a.bA_prev = P.bn_bA; a.bB_prev = P.bn_bB; a.bC_prev = P.bn_bC;
                a.gamma_prev = net->params + P.g_off;
                a.inv_keep = net->dropout > 0.0f ? 1.0f / (1.0f - net->dropout) : 1.0f;
            } else {
                a.d_in = net->layers[mu_j].dact;
                a.MU = net->layers[mu_j].act;
                a.kld_w = net->kld_w;
            }
        }
        const bool fused = use_tc(net, B) && fused_staging(net, B);
        // fused: dL/dY of this layer was staged by the loss kernel (output layer) or by the dgrad of layer j + 1
        if (use_tc(net, B) && (!fused || (j == nl - 1 && net->d_in > LOSS_STAGE_MAX_D)))
            if (launch_prep_grad(net, j, B, s)) return 1;
        if (fused && L.in_kind != VK_IN_DATA) {
            const vk_vae_layer &P = net->layers[L.in_kind == VK_IN_BN ? j - 1 : mu_j];
            a.stage = L.in_kind == VK_IN_BN ? 1 : 2;
            a.stage_a = P.dy_hi; a.stage_a_ld = r32(P.n_out);
            a.stage_t = P.dyt_hi; a.stage_t_ld = net->bmax;
            a.slope = net->slope; a.has_dropout = net->dropout > 0.0f ? 1 : 0;
        }
        PROF_MARK_K(s, PK_BWD);
        if (use_tc(net, B)) {
            if (tc_prepare()) return 1;
            BwdTcExtra x;
            x.nsplit = tc_nsplit(net, B);
            x.k_per_split = (((B + x.nsplit - 1) / x.nsplit) + 31) & ~31;
            x.slab = net->grad_slab;
            x.flush = net->wgrad_flush != 0;
            a.tile_n = tc_tile_n(B);
            a.wg_tiles_m = (L.n_out + 127) / 128;
            a.wg_tile_n = tc_wg_tile_n(B);
            a.wg_tiles_n = (L.k_in + 1 + a.wg_tile_n - 1) / a.wg_tile_n;
            if (a.dg_tiles_m) {
                a.dg_tiles_m = (B + 127) / 128;
                a.dg_tiles_n = (L.k_in + a.tile_n - 1) / a.tile_n;
            }
            a.wg_a = tc::OpRef{L.dyt_hi, L.dyt_lo, net->bmax};
            a.wg_b = tc::OpRef{L.xt_hi, L.xt_lo, net->bmax};
            a.dg_a = tc::OpRef{L.dy_hi, L.dy_lo, r32(L.n_out)};
            a.dg_b = tc::OpRef{L.wt_hi, L.wt_lo, r32(L.n_out)};
            a.use_tma = (a.dg_tiles_m && use_tma(net, L)) ? 1 : 0;
            if (a.use_tma && (vk_make_tmap_2d(&a.tm_dg_hi, L.wt_hi, r32(L.n_out), r128(L.k_in), a.tile_n) ||
                              vk_make_tmap_2d(&a.tm_dg_lo, L.wt_lo, r32(L.n_out), r128(L.k_in), a.tile_n)))
                return 1;
            int blocks = a.wg_tiles_m * a.wg_tiles_n * x.nsplit + a.dg_tiles_m * a.dg_tiles_n;
            const size_t smem = (size_t)tc_smem_for(a.tile_n > a.wg_tile_n ? a.tile_n : a.wg_tile_n, 2);
            a.cluster_rt = (a.stage == 1 && L.in_kind == VK_IN_BN && a.dg_tiles_m) ? cluster_fold_rt(B) : 0;
            if (a.cluster_rt) {
                const int n_wg = a.wg_tiles_m * a.wg_tiles_n * x.nsplit;
                a.n_wg_pad = ((n_wg + a.cluster_rt - 1) / a.cluster_rt) * a.cluster_rt;
                blocks = a.n_wg_pad + a.dg_tiles_m * a.dg_tiles_n;  // dg_tiles_m == cluster_rt
                const dim3 cluster(a.cluster_rt, 1, 1);
                if (a.use_tma) {
                    if (x.flush) VK_CUDA(vk_launch_cluster(bwd_layer_tc_kernel<true, true>, dim3(blocks), dim3(tc::WS_THREADS), smem, s, cluster, a, x));
                    else VK_CUDA(vk_launch_cluster(bwd_layer_tc_kernel<true, false>, dim3(blocks), dim3(tc::WS_THREADS), smem, s, cluster, a, x));
                } else {
                    if (x.flush) VK_CUDA(vk_launch_cluster(bwd_layer_tc_kernel<false, true>, dim3(blocks), dim3(tc::WS_THREADS), smem, s, cluster, a, x));
                    else VK_CUDA(vk_launch_cluster(bwd_layer_tc_kernel<false, false>, dim3(blocks), dim3(tc::WS_THREADS), smem, s, cluster, a, x));
                }
            } else if (a.use_tma) {
                if (x.flush) VK_CUDA(vk_launch(bwd_layer_tc_kernel<true, true>, dim3(blocks), dim3(tc::WS_THREADS), smem, s, a, x));
                else VK_CUDA(vk_launch(bwd_layer_tc_kernel<true, false>, dim3(blocks), dim3(tc::WS_THREADS), smem, s, a, x));
            } else {
                if (x.flush) VK_CUDA(vk_launch(bwd_layer_tc_kernel<false, true>, dim3(blocks), dim3(tc::WS_THREADS), smem, s, a, x));
                else VK_CUDA(vk_launch(bwd_layer_tc_kernel<false, false>, dim3(blocks), dim3(tc::WS_THREADS), smem, s, a, x));
            }
        } else {
            const int blocks = a.wg_tiles_m * a.wg_tiles_n + a.dg_tiles_m * a.dg_tiles_n;
            VK_CUDA(vk_launch(bwd_layer_kernel, dim3(blocks), dim3(GT), (size_t)(0), s, a));
        }
        VK_LAUNCH_CHECK();
    }
    return 0;
}

__global__ void reduce_slabs_kernel(float *g, int64_t n, int nslab, int64_t slab) {
    pdl_entry();
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        float t = g[i];
        for (int sl = 1; sl < nslab; ++sl) t += g[(int64_t)sl * slab + i];
        g[i] = t;
    }
}

static int launch_dadapt(const vk_vae *net, int nslab, cudaStream_t s) {
    PROF_MARK_K(s, PK_OPT);
    // opt_part holds two doubles per block (sized from n_params by the host: vk_vae.opt_part), no fixed cap
    const int opt_blocks = (int)((net->n_params + OPT_ELEMS - 1) / OPT_ELEMS);
    VK_CUDA(vk_launch(dadapt_kernel, dim3(opt_blocks), dim3(256), (size_t)(0), s, net->params, net->grads, net->exp_avg, net->exp_avg_sq, net->s,
                                             net->n_params, net->opt_part, net->ctl, 2 * VK_VAE_MAX_LAYERS + 2,
                                             nslab, net->grad_slab));
    VK_LAUNCH_CHECK();
    return 0;
}

static int grad_step_impl(const vk_vae *net, int batch, const vk_vae_inject *inject, void *stream) {
    if (check_net(net, batch)) return 1;
    cudaStream_t s = (cudaStream_t)stream;
    const int mode = (inject && inject->batch_idx) ? 0 : 1;
    SideCtx *sc = (use_tc(net, batch) && g_prof_events == nullptr) ? side_ctx() : nullptr;
    if (sc) {  // weight staging only depends on the previous optimiser step: next to batch rows + gather
        VK_CUDA(cudaEventRecord(sc->fork, s));
        VK_CUDA(cudaStreamWaitEvent(sc->side, sc->fork, 0));
        if (launch_prep_weights(net, sc->side)) return 1;
        VK_CUDA(cudaEventRecord(sc->weights_done, sc->side));
    }
    // tensor-core path: the gather of the first layer draws the batch itself (one launch less on the critical path)
    BatchDraw draw;
    if (use_tc(net, batch)) { draw.mode = mode; draw.row0 = 0; draw.inj = inject; }
    else if (launch_batch_rows(net, batch, mode, 0, inject, s)) return 1;
    if (!sc && use_tc(net, batch) && launch_prep_weights(net, s)) return 1;
    if (launch_forward(net, batch, 1, net->n_layers, inject, 0, nullptr, s, sc ? sc->weights_done : nullptr, &draw)) return 1;
    if (launch_loss(net, batch, 1, s, sc)) return 1;
    if (launch_backward(net, batch, s)) return 1;
    if (sc) VK_CUDA(cudaStreamWaitEvent(s, sc->fold_done, 0));  // join before the optimiser / the end of a capture
    return 0;
}

extern "C" int vk_vae_grad_step(const vk_vae *net, int batch, const vk_vae_inject *inject, void *stream) {
    if (grad_step_impl(net, batch, inject, stream)) return 1;
    if (use_tc(net, batch) && tc_nsplit(net, batch) > 1) {
        // leave the complete gradient in slab 0 (all-reduce / inspection read only that slab)
        VK_CUDA(vk_launch(reduce_slabs_kernel, dim3(296), dim3(256), (size_t)(0), (cudaStream_t)stream, net->grads, net->n_params,
                                                                          tc_nsplit(net, batch), net->grad_slab));
        VK_LAUNCH_CHECK();
    }
    return 0;
}

extern "C" int vk_vae_dadapt_step(const vk_vae *net, void *stream) {
    if (check_net(net, 1)) return 1;
    return launch_dadapt(net, 1, (cudaStream_t)stream);
}

extern "C" int vk_vae_train_step(const vk_vae *net, int batch, const vk_vae_inject *inject, void *stream) {
    if (grad_step_impl(net, batch, inject, stream)) return 1;
    return launch_dadapt(net, use_tc(net, batch) ? tc_nsplit(net, batch) : 1, (cudaStream_t)stream);
}

extern "C" int vk_vae_forward(const vk_vae *net, int64_t row0, int batch, int training, int with_loss,
                              const vk_vae_inject *inject, void *stream) {
    if (check_net(net, batch)) return 1;
    cudaStream_t s = (cudaStream_t)stream;
    const int mode = (inject && inject->batch_idx) ? 0 : 2;
    BatchDraw draw;
    if (use_tc(net, batch)) { draw.mode = mode; draw.row0 = row0; draw.inj = inject; }
    else if (launch_batch_rows(net, batch, mode, row0, inject, s)) return 1;
    if (use_tc(net, batch) && launch_prep_weights(net, s)) return 1;
    if (launch_forward(net, batch, training, net->n_layers, inject, 0, nullptr, s, nullptr, &draw)) return 1;
    if (with_loss && launch_loss(net, batch, 0, s)) return 1;
    return 0;
}

extern "C" int vk_vae_prepare_eval(const vk_vae *net, void *stream) {
    if (check_net(net, 1)) return 1;
    for (int j = 0; j < net->n_layers; ++j) {
        const vk_vae_layer &L = net->layers[j];
        if (L.kind != VK_LAYER_HIDDEN) continue;
        eval_affine_kernel<<<(L.n_out + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
            L.bn_a, L.bn_c, net->params + L.g_off, net->params + L.beta_off, L.running_mean, L.running_var, L.n_out);
        VK_LAUNCH_CHECK();
    }
    return 0;
}

extern "C" int vk_vae_encode(const vk_vae *net, int64_t row0, int64_t n, int mask_bits, float *latent_out,
                             void *stream) {
    if (check_net(net, 1)) return 1;
    if (mask_bits < 0 || mask_bits > 23) {
        vk_set_error("Must mask between 0 and 23 bits");
        return 1;
    }
    cudaStream_t s = (cudaStream_t)stream;
    int mu_j = -1;
    for (int j = 0; j < net->n_layers; ++j)
        if (net->layers[j].kind == VK_LAYER_MU) mu_j = j;
    if (vk_vae_prepare_eval(net, stream)) return 1;
    if (use_tc(net, (int)(n < net->bmax ? n : net->bmax)) && launch_prep_weights(net, s)) return 1;
    for (int64_t off = 0; off < n; off += net->bmax) {
        const int B = (int)((n - off) < net->bmax ? (n - off) : net->bmax);
        BatchDraw draw;
        if (use_tc(net, B)) { draw.mode = 2; draw.row0 = row0 + off; }
        else if (launch_batch_rows(net, B, 2, row0 + off, nullptr, s)) return 1;
        if (launch_forward(net, B, 0, mu_j + 1, nullptr, mask_bits, latent_out + off * net->nlatent, s, nullptr, &draw)) return 1;
    }
    return 0;
}

// One training step with a CUDA event before every launch: ms_out_host[i] = device time of the i-th
// launch, kinds_out_host[i] = what it was (0 batch rows, 1 forward layer, 2 loss, 3 backward layer,
// 4 optimiser, 5 operand staging).  Returns the number of launches through *n_launches.  Synchronises.
extern "C" int vk_vae_profile_step(const vk_vae *net, int batch, const vk_vae_inject *inject, float *ms_out_host,
                                   int *kinds_out_host, int capacity, int *n_launches, void *stream) {
    if (check_net(net, batch)) return 1;
    cudaStream_t s = (cudaStream_t)stream;
    const int cap = 96;
    cudaEvent_t ev[96];
    int kinds[96];
    for (int i = 0; i < cap; ++i) VK_CUDA(cudaEventCreate(&ev[i]));
    g_prof_events = ev; g_prof_kinds = kinds; g_prof_n = 0; g_prof_cap = cap - 1;
    int rc = vk_vae_train_step(net, batch, inject, stream);
    const int n = g_prof_n;
    g_prof_events = nullptr;
    if (!rc) {
        cudaEventRecord(ev[n], s);
        if (cudaStreamSynchronize(s) != cudaSuccess) rc = 1;
        for (int i = 0; i < n && i < capacity && !rc; ++i) {
            float ms = 0.f;
            if (cudaEventElapsedTime(&ms, ev[i], ev[i + 1]) != cudaSuccess) rc = 1;
            ms_out_host[i] = ms;
            kinds_out_host[i] = kinds[i];
        }
        *n_launches = n < capacity ? n : capacity;
    }
    for (int i = 0; i < cap; ++i) cudaEventDestroy(ev[i]);
    if (rc && !vk_last_error()[0]) vk_set_error("vk_vae_profile_step failed");
    return rc;
}

#ifdef VK_TIMELINE
extern "C" int vk_timeline_read(unsigned long long *out_host) {
    VK_CUDA(cudaDeviceSynchronize());
    VK_CUDA(cudaMemcpyFromSymbol(out_host, vk_tl, sizeof(unsigned long long) * 4096));
    return 0;
}
// launch records since the last reset (at most 4096): out_host[4096 * 4], *n_out = launches recorded
extern "C" int vk_timeline_kernels(unsigned long long *out_host, unsigned int *n_out, int reset) {
    VK_CUDA(cudaDeviceSynchronize());
    VK_CUDA(cudaMemcpyFromSymbol(out_host, vk_tk, sizeof(unsigned long long) * 4096 * 4));
    VK_CUDA(cudaMemcpyFromSymbol(n_out, vk_tk_seq, sizeof(unsigned int)));
    if (reset) {
        const unsigned int zero = 0;
        VK_CUDA(cudaMemcpyToSymbol(vk_tk_seq, &zero, sizeof(zero)));
    }
    return 0;
}
#endif

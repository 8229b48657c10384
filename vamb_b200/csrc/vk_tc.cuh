// Hopper (sm_90a) tensor-core building blocks: raw PTX wrappers for mbarrier, TMA and wgmma, shared-memory matrix
// descriptors, and a 128 x BN x K tile GEMM in error-compensated 3xTF32.
//
// Operands are materialised ONCE per layer by the producing kernel (vk_vae.cu: fused staging / prep kernels) as
// plain zero-padded fp32 arrays; the main loop below (ws_mainloop) feeds the 128-row operand to wgmma from registers
// and streams the narrow operand through a shared-memory ring.
//
// 3xTF32: a .tf32 MMA reads the top 19 bits of each fp32 operand word (low 13 mantissa bits ignored),
// so hi = x as stored, lo = x - (x & 0xFFFFE000) (exact).  D += A_lo*B_hi + A_hi*B_lo + A_hi*B_hi leaves
// a relative error of ~2^-21 per product, i.e. fp32-grade results from the tensor pipe.
#pragma once
#include "vk_common.cuh"

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
// The bare try_wait loop (the hardware suspends the thread inside try_wait for a bounded time), plus a poll counter: a
// wait that never completes (a bulk copy that never lands) traps after 2^26 failed polls (seconds) instead of hanging
// the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t"
        ".reg .pred p, q;\n\t"
        ".reg .u32 n;\n\t"
        "mov.u32 n, 0;\n\t"
        "LAB_WAIT%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra LAB_DONE%=;\n\t"
        "add.u32 n, n, 1;\n\t"
        "setp.lt.u32 q, n, 0x4000000;\n\t"
        "@q bra LAB_WAIT%=;\n\t"
        "trap;\n\t"
        "LAB_DONE%=:\n\t"
        "}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

// shared-memory writes of the generic proxy (st.shared, cp.async) made visible to wgmma / TMA (async proxy)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- wgmma (warpgroup MMA, sm_90a) ----
// shared-memory matrix descriptor (cute/arch/mma_sm90_desc.hpp: GmmaDescriptor): start>>4 [0,14) | LBO>>4 [16,30) |
// SBO>>4 [32,46) | base_offset [49,52) | layout_type [62,64) (0 = no swizzle, 1 = 128B swizzle).
// No swizzle, K-major: SBO = byte stride between 8-row core matrices along N, LBO = byte stride between the two 16-byte
// K chunks of one K = 8 step.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFFu);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32;
    return d;
}
// K-major tile written by TMA with CU_TENSOR_MAP_SWIZZLE_128B: rows of 128 bytes (one 32-float k-tile), 8-row swizzle
// atoms of 1024 bytes (SBO); the tile base must be 1024-byte aligned; a K = 8 (32-byte) step advances the start address
// by 32 bytes inside the atom.
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr >> 4) & 0x3FFFu);
    d |= (uint64_t)1 << 16;             // LBO: unused for swizzled K-major operands
    d |= (uint64_t)(1024u >> 4) << 32;  // SBO: next group of 8 rows
    d |= (uint64_t)1 << 62;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// D[64 x N] += A[64 x 8] * B[N x 8]^T, fp32 accumulate: A from registers (the warpgroup's m64k8 tf32 fragment: warp w of
// the group, lane l holds A[16 w + l/4 (+8)][l%4 (+4)] as a[0] = (r, k), a[1] = (r + 8, k), a[2] = (r, k + 4),
// a[3] = (r + 8, k + 4)), B K-major in shared memory (descriptor).  d[i] (i < N / 2) is D[16 w + l/4 + 8 ((i/2) % 2)]
// [8 (i/4) + 2 (l%4) + i%2].
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], const float *a, uint64_t bdesc);
template <>
__device__ __forceinline__ void wgmma_tf32<16>(float (&d)[64], const float *a, uint64_t bdesc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %13, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7"
        "}, {%8, %9, %10, %11}, %12, p, 1, 1;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])), "l"(bdesc), "r"(1));
}
template <>
__device__ __forceinline__ void wgmma_tf32<32>(float (&d)[64], const float *a, uint64_t bdesc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
        "}, {%16, %17, %18, %19}, %20, p, 1, 1;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])), "l"(bdesc), "r"(1));
}
template <>
__device__ __forceinline__ void wgmma_tf32<64>(float (&d)[64], const float *a, uint64_t bdesc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
        "}, {%32, %33, %34, %35}, %36, p, 1, 1;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])), "l"(bdesc), "r"(1));
}
template <>
__device__ __forceinline__ void wgmma_tf32<128>(float (&d)[64], const float *a, uint64_t bdesc) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %69, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{"
        "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
        "}, {%64, %65, %66, %67}, %68, p, 1, 1;\n}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
          "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
          "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
          "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
          "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
          "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
          "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
          "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(__float_as_uint(a[0])), "r"(__float_as_uint(a[1])), "r"(__float_as_uint(a[2])), "r"(__float_as_uint(a[3])), "l"(bdesc), "r"(1));
}

// ---- operand tiles in shared memory (fp32 words) ----
// Tile = ROWS (N extent, multiple of 8) x KT (=32) elements, K-major, no swizzle: core matrix = 8 rows x 16 B;
// offset(r, k) = (r/8)*1024 + (k/4)*128 + (r%8)*16 + (k%4)*4 -> SBO = 1024, LBO = 128; k8-step j starts at +256*j.
constexpr int KT = 32;
__host__ __device__ constexpr int b_tile_bytes(int bn) { return bn * KT * 4; }

__device__ __forceinline__ float tf32_lo(float x) { return x - __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }
__device__ __forceinline__ float4 tf32_lo(const float4 v) {
    return make_float4(tf32_lo(v.x), tf32_lo(v.y), tf32_lo(v.z), tf32_lo(v.w));
}

struct OpRef {
    const float *hi, *lo;
    int ld;  // floats per row (multiple of 4)
};

__device__ __forceinline__ void cp_async16(uint32_t saddr, const void *gptr) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(saddr), "l"(gptr) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// ---- TMA: bulk tensor copies global -> shared, completion counted in bytes on an mbarrier ----
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// box of the 2-D tensor map `tmap` at (c0 = innermost element, c1 = row) -> shared memory at smem_dst
__device__ __forceinline__ void tma_load_2d(uint32_t smem_dst, const void *tmap, uint64_t *bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_dst),
        "l"(tmap), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}

// "Lane-major" storage of an A-role operand (the 128-row side of the GEMM): 128-row panels of an
// [rows][ld] array, each k-tile of a panel is one 16 KB block  [k / 4 (8)][row (128)][k % 4 (4)]  so that
// consecutive rows are consecutive float4 for the producers, and the eight rows x four k of one wgmma fragment
// register are 128 contiguous bytes for the main loop.  Same footprint as the row-major array.
__host__ __device__ __forceinline__ size_t lane_major_index(int r, int k, int ld) {
    return (size_t)(r >> 7) * 128 * ld + (size_t)(k >> 5) * 4096 + (size_t)((k & 31) >> 2) * 512 + (size_t)(r & 127) * 4 + (k & 3);
}

// Main loop of the layer GEMMs.  A CTA is two warpgroups (WS_THREADS = 256); warpgroup g computes rows
// [64 g, 64 g + 64) of the 128-row tile with one wgmma chain, its accumulator in registers.
//   A (128-row operand): each thread loads its wgmma fragment of a k-tile straight from the lane-major array into
//     registers (coalesced 128-byte rows, PA tiles in flight), the fp32 word serving as tf32 "hi" and the remainder
//     "lo" derived in registers -- A never touches shared memory;
//   B (narrow operand): a ring of WS_STAGES shared-memory stages [hi tile | lo tile] filled PB tiles ahead, either with
//     cp.async by all threads (each deriving "lo" of the chunk it copied) or, TMA_B, by one thread through two bulk
//     tensor copies (the weights and their tf32 remainders, pre-split once per step by prep_weights);
//   per k-tile: one block barrier (the stage is complete; every warpgroup is done with the stage refilled next), then
//     12 wgmma per warpgroup (4 K = 8 steps x {lo x hi, hi x lo, hi x hi}: small terms first), committed as one group
//     that is waited for one k-tile later, so the tensor core runs while the next tile's barrier and split happen.
// Runtime widths bn are computed with the next wgmma width N in {16, 32, 64, 128}; the columns past bn read stale ring
// rows and are discarded by the epilogue.
constexpr int WS_THREADS = 256;
constexpr int WS_EPI_THREADS = 256;
constexpr int WS_STAGES = 5;
__host__ __device__ constexpr int wg_n(int bn) { return bn <= 16 ? 16 : (bn <= 32 ? 32 : (bn <= 64 ? 64 : 128)); }
// ring bytes for tiles up to bn columns (+ 1024 for the alignment of the dynamic shared memory base)
__host__ __device__ constexpr int ws_smem_bytes(int bn) { return WS_STAGES * 2 * b_tile_bytes(wg_n(bn)) + 1024; }

struct WsShared {
    uint64_t full[WS_STAGES];  // TMA_B: bytes of stage s landed
};

// The accumulator of one thread: d[i] as in wgmma_tf32, rows of its warpgroup's half of the tile.
struct WsAcc {
    float d[64];
};

// FLUSH (wgrad: the reduction runs over the batch, hundreds of rows): the chain of tensor-core accumulations is cut
// every WS_FLUSH_KT k-tiles (128 batch rows), and each finished group is added into separate fp32 registers (round to
// nearest), so that the error of a long chain stops growing with its length.
constexpr int WS_FLUSH_KT = 4;

template <int N, bool TMA_B, bool FLUSH>
__device__ __forceinline__ void ws_loop(const float *A, int lda, int m0, const float *B, int ldb, int n0, int bn, int kt0, int nk,
                                        uint8_t *smem, WsShared *sh, int slot_rows, const void *tm_hi, const void *tm_lo,
                                        float (&d)[64]) {
    constexpr int S = WS_STAGES, PB = S - 2, PA = FLUSH ? 2 : 4;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // ring stage = [hi: R rows | lo: R rows]; TMA boxes are slot_rows rows, the wgmma reads N rows
    const int R = TMA_B ? wg_n(slot_rows) : N;
    const int bbytes = b_tile_bytes(R), sbytes = 2 * bbytes;
    const uint32_t smem_base = smem_u32(smem);
    // B chunk q = tid + 256 i of a tile: row ((q >> 6) << 3) | (q & 7) = r0 + 32 i, 16-byte column k4, at byte q * 16
    const int r0 = ((tid >> 6) << 3) | (tid & 7), k4 = (tid >> 3) & 7;
    const float *pb = B + (size_t)(n0 + r0) * ldb + (size_t)kt0 * KT + k4 * 4;
    const size_t b_step = (size_t)32 * ldb;
    const int nbi = bn >> 5;                  // whole 32-row groups of the B tile
    const bool b_tail = tid < (bn & 31) * 8;  // + 16 rows when bn is an odd multiple of 16
    const uint32_t soff = (uint32_t)tid * 16u;
    // A: fragment rows r1 = 64 (warp / 4) + 16 (warp % 4) + lane / 4 and r1 + 8, k = 4 j + lane % 4 (j < 8)
    const int r1 = 64 * (warp >> 2) + 16 * (warp & 3) + (lane >> 2);
    const float *pa = A + (size_t)(m0 >> 7) * 128 * lda + (size_t)kt0 * 4096 + r1 * 4 + (lane & 3);
    auto issue_b = [&](int kt, int slot) {
        if (TMA_B) {
            if (tid == 0) {
                mbar_arrive_expect_tx(&sh->full[slot], (uint32_t)(2 * b_tile_bytes(slot_rows)));
                tma_load_2d(smem_base + slot * sbytes, tm_hi, &sh->full[slot], (kt0 + kt) * KT, n0);
                tma_load_2d(smem_base + slot * sbytes + bbytes, tm_lo, &sh->full[slot], (kt0 + kt) * KT, n0);
            }
            return;
        }
        const uint32_t st = smem_base + slot * sbytes + soff;
        const float *gb = pb + (size_t)kt * KT;
        for (int i = 0; i < nbi; ++i) cp_async16(st + i * 4096, gb + i * b_step);
        if (b_tail) cp_async16(st + nbi * 4096, gb + nbi * b_step);
    };
    auto split_b = [&](int slot) {
        uint8_t *st = smem + slot * sbytes + soff;
        for (int i = 0; i < nbi; ++i)
            *reinterpret_cast<float4 *>(st + bbytes + i * 4096) = tf32_lo(*reinterpret_cast<const float4 *>(st + i * 4096));
        if (b_tail)
            *reinterpret_cast<float4 *>(st + bbytes + nbi * 4096) = tf32_lo(*reinterpret_cast<const float4 *>(st + nbi * 4096));
    };
    // v[4 s .. 4 s + 3] = the fragment of K = 8 step s: (r1, 8s + l%4), (r1 + 8, ..), (r1, 8s + 4 + l%4), (r1 + 8, ..)
    auto load_a = [&](int kt, float (&v)[16]) {
        const float *g = pa + (size_t)kt * 4096;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            v[2 * j] = __ldg(g + j * 512);
            v[2 * j + 1] = __ldg(g + j * 512 + 32);
        }
    };

    float ra[PA][16], lo[2][16];
    float racc[FLUSH ? 64 : 1];
    if constexpr (FLUSH) {
#pragma unroll
        for (int i = 0; i < 64; ++i) racc[i] = 0.0f;
    }
    if (TMA_B && tid == 0) {
#pragma unroll
        for (int s = 0; s < S; ++s) mbar_init(&sh->full[s], 1);
        mbar_fence_init();
    }
    if (!TMA_B) {
#pragma unroll
        for (int t = 0; t < PB; ++t) {
            if (t < nk) issue_b(t, t);
            cp_async_commit();
        }
    }
#pragma unroll
    for (int t = 0; t < PA; ++t)
        if (t < nk) load_a(t, ra[t]);
    __syncthreads();  // barriers initialised
    if (TMA_B) {
        for (int t = 0; t < PB; ++t)
            if (t < nk) issue_b(t, t);
    }
    const uint64_t desc0 = TMA_B ? make_smem_desc_sw128(smem_base) : make_smem_desc(smem_base, 128, 1024);
    const uint32_t kstep = TMA_B ? 2u : 16u;  // start-address units (16 bytes) per K = 8 step
    for (int kb = 0; kb < nk; kb += PA) {
#pragma unroll
        for (int i = 0; i < PA; ++i) {
            const int kt = kb + i;
            if (kt >= nk) break;
            const int slot = kt % S;
            if (TMA_B) {
                mbar_wait(&sh->full[slot], (uint32_t)((kt / S) & 1));
            } else {
                cp_async_wait<PB - 1>();  // this thread's copies of tile kt have landed (one group per tile)
                split_b(slot);
                fence_async_smem();
            }
            // stage kt complete for everyone; every warpgroup has retired the wgmma of tile kt - 2 (waited for below),
            // the last reader of the stage of tile kt + PB
            __syncthreads();
            if (kt + PB < nk) issue_b(kt + PB, (kt + PB) % S);
            if (!TMA_B) cp_async_commit();
            float(&hi)[16] = ra[i];
            float(&l)[16] = lo[i & 1];
#pragma unroll
            for (int e = 0; e < 16; ++e) l[e] = tf32_lo(hi[e]);
            const uint64_t bh = desc0 + (uint64_t)((uint32_t)(slot * sbytes) >> 4);
            const uint64_t bl = bh + (uint64_t)((uint32_t)bbytes >> 4);
            wgmma_fence();
#pragma unroll
            for (int s = 0; s < KT / 8; ++s) {
                wgmma_tf32<N>(d, l + 4 * s, bh + kstep * s);
                wgmma_tf32<N>(d, hi + 4 * s, bl + kstep * s);
                wgmma_tf32<N>(d, hi + 4 * s, bh + kstep * s);
            }
            wgmma_commit();
            if constexpr (FLUSH) {
                if ((kt + 1) % WS_FLUSH_KT == 0 && kt != nk - 1) {
                    wgmma_wait<0>();
#pragma unroll
                    for (int e = 0; e < N / 2; ++e) {
                        racc[e] += d[e];
                        d[e] = 0.0f;
                    }
                } else {
                    wgmma_wait<1>();
                }
            } else {
                wgmma_wait<1>();  // tile kt - 1 retired: its A registers are free
            }
            if (kt >= 1 && kt - 1 + PA < nk) load_a(kt - 1 + PA, ra[(i + PA - 1) % PA]);
        }
    }
    wgmma_wait<0>();
    if constexpr (FLUSH) {
#pragma unroll
        for (int e = 0; e < N / 2; ++e) d[e] += racc[e];
    }
    __syncthreads();  // every warpgroup is done with the ring: the caller may reuse the shared memory
}

// acc = A[m0.., k] * B[n0.., k]^T over k-tiles [kt0, kt0 + nk) (rows of this thread's warpgroup, see WsAcc).
// A: lane-major (m0 a multiple of 128), B: plain K-major; both fp32, zero padded to whole tiles (ld = floats per
// row, multiple of 32), B rows up to n0 + bn (bn a multiple of 16, <= 128).  nk == 0 (an empty split) yields zeros.
// TMA_B: B through tm_hi / tm_lo, CUtensorMap objects in kernel-parameter space (__grid_constant__) of 128B-swizzled
// boxes of 32 floats x slot_rows rows (slot_rows = the launch's tile width, >= bn).  All WS_THREADS threads call it.
template <bool TMA_B = false, bool FLUSH = false>
__device__ __forceinline__ void ws_mainloop(const float *A, int lda, int m0, const float *B, int ldb, int n0, int bn,
                                            int kt0, int nk, uint8_t *smem, WsShared *sh, WsAcc &acc, int slot_rows = 0,
                                            const void *tm_hi = nullptr, const void *tm_lo = nullptr) {
#pragma unroll
    for (int e = 0; e < 64; ++e) acc.d[e] = 0.0f;
    switch (wg_n(bn)) {
        case 16: ws_loop<16, TMA_B, FLUSH>(A, lda, m0, B, ldb, n0, bn, kt0, nk, smem, sh, slot_rows, tm_hi, tm_lo, acc.d); break;
        case 32: ws_loop<32, TMA_B, FLUSH>(A, lda, m0, B, ldb, n0, bn, kt0, nk, smem, sh, slot_rows, tm_hi, tm_lo, acc.d); break;
        case 64: ws_loop<64, TMA_B, FLUSH>(A, lda, m0, B, ldb, n0, bn, kt0, nk, smem, sh, slot_rows, tm_hi, tm_lo, acc.d); break;
        default: ws_loop<128, TMA_B, FLUSH>(A, lda, m0, B, ldb, n0, bn, kt0, nk, smem, sh, slot_rows, tm_hi, tm_lo, acc.d); break;
    }
}

// Accumulator -> shared tile [128][ts] (raw values), columns < bn.
__device__ __forceinline__ void ws_acc_to_tile(const WsAcc &acc, int bn, float *tile, int ts) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int row = 64 * (warp >> 2) + 16 * (warp & 3) + (lane >> 2), col = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
        const int c = 8 * (i >> 2) + col, r = row + 8 * ((i >> 1) & 1);
        if (c < bn) *reinterpret_cast<float2 *>(tile + r * ts + c) = make_float2(acc.d[i], acc.d[i + 1]);
    }
}

// all threads: the tile in shared memory is complete for everyone
__device__ __forceinline__ void ws_tile_end() { __syncthreads(); }

}  // namespace tc

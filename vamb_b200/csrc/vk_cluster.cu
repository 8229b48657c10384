// vamb_b200 clustering kernels (sm_90a).  HBM-streaming integer/compare work: no tensor
// cores; the rules that matter are coalescing (8 lanes x float4 = one 128 B row, one warp =
// 4 consecutive rows = 512 contiguous bytes per load instruction), several independent
// loads in flight per thread, shared-memory staging of the sparse outputs, and a persistent
// grid sized to the SM count.
//
// Replaces (reference file:line, RasmussenLab/vamb):
//   normalize_rows_kernel   vamb/cluster.py:653-669   _normalize
//   probe_kernel            vamb/cluster.py:672-676   _calc_distances
//                           vamb/cluster.py:619-629   sample_medoid (within set, density)
//                           vamb/cluster.py:457-481   find_threshold (loner count, histogram)
//   eval_candidates_kernel  vamb/cluster.py:427-448   the sample_medoid calls of one wander round
//   select_members_kernel   vamb/cluster.py:640-650, 308-309   _smaller_indices + kept_mask update
//   compact_*_kernel        vamb/cluster.py:318-335   pack (vambcore.overwrite_matrix)
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include "vk_common.cuh"

// ------------------------------------------------------------------ error plumbing
static thread_local char g_err[512] = "";

void vk_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char *vk_last_error(void) { return g_err; }

bool vk_pdl_enabled() {
    static const bool on = [] {
        const char *v = getenv("VK_PDL");
        return v ? atoi(v) != 0 : true;
    }();
    return on;
}
extern "C" int vk_abi_version(void) { return VK_ABI_VERSION; }

int vk_num_sms() {
    static int sms = 0;
    if (sms == 0) {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return 132;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) sms = 132;
    }
    return sms;
}

extern "C" int vk_check_device(void) {
    int dev = 0, major = 0, minor = 0;
    VK_CUDA(cudaGetDevice(&dev));
    VK_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
    VK_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
    if (major != 9 || minor != 0) {
        vk_set_error("vamb_b200 kernels are built for sm_90a only; device is sm_%d%d", major, minor);
        return 1;
    }
    return 0;
}

// ------------------------------------------------------------------ normalize
// One thread per row (one-off pass).  ss = sum_k (double)x_k^2 in ascending k (products exact).
__global__ void __launch_bounds__(256) normalize_rows_kernel(float *__restrict__ m, int64_t n, int d) {
    const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    float *x = m + row * (int64_t)d;
    bool allzero = true;
    for (int k = 0; k < d; ++k)
        if (x[k] != 0.0f) { allzero = false; break; }
    const float fill = (float)(1.0 / (double)d);
    double ss = 0.0;
    for (int k = 0; k < d; ++k) {
        const double v = allzero ? (double)fill : (double)x[k];
        ss += v * v;
    }
    const float nrm = (float)sqrt(ss);
    const float den = __fmul_rn(nrm, 1.41421356237309504880f);
    for (int k = 0; k < d; ++k) {
        const float v = allzero ? fill : x[k];
        x[k] = __fdiv_rn(v, den);
    }
}

extern "C" int vk_normalize_rows(float *matrix, int64_t n, int d, void *stream) {
    if (n <= 0) return 0;
    const int threads = 256;
    const int64_t blocks = (n + threads - 1) / threads;
    normalize_rows_kernel<<<(unsigned)blocks, threads, 0, (cudaStream_t)stream>>>(matrix, n, d);
    VK_LAUNCH_CHECK();
    return 0;
}

__global__ void __launch_bounds__(256) check_normalized_kernel(const float *__restrict__ m, int64_t n, int d,
                                                               float tol, int32_t *n_bad) {
    const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    const float *x = m + row * (int64_t)d;
    double ss = 0.0;
    for (int k = 0; k < d; ++k) ss += (double)x[k] * (double)x[k];
    if (!(fabs(2.0 * ss - 1.0) <= (double)tol)) atomicAdd(n_bad, 1);
}

extern "C" int vk_check_normalized(const float *matrix, int64_t n, int d, float tol, int32_t *n_bad, void *stream) {
    VK_CUDA(cudaMemsetAsync(n_bad, 0, sizeof(int32_t), (cudaStream_t)stream));
    if (n <= 0) return 0;
    const int64_t blocks = (n + 255) / 256;
    check_normalized_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(matrix, n, d, tol, n_bad);
    VK_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------ mapped completion
// "Last block done" with ONE fencing thread per block: after the block barrier, thread 0's device-scope fence is
// cumulative over everything the block wrote before the barrier (the release pattern of the PTX memory model, as in
// cutlass/semaphore.h); having all 256 threads of every block execute MEMBAR (let alone the system-scope one, which
// also invalidates L1) turns every launch into a long stall on the memory barrier.
// Returns true in every thread of the block that finishes last; that block has acquired the other blocks' writes.
__device__ __forceinline__ bool vk_last_block(int32_t *ticket, int *s_last) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        const int t = atomicAdd(ticket, 1);
        *s_last = (t == (int)gridDim.x - 1);
        if (*s_last) {
            *ticket = 0;
            __threadfence();
        }
    }
    __syncthreads();
    return *s_last != 0;
}
// Publish: after the last block's writes to the pinned result buffers, one thread orders them (system scope) before
// the flag the host spins on.
__device__ __forceinline__ void vk_raise_flag(volatile int32_t *flag, int32_t seq) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        *flag = seq;
    }
}

// ------------------------------------------------------------------ probe
constexpr int PB_THREADS = 256;
constexpr int PB_GROUPS = PB_THREADS / 8;  // rows per pass
constexpr int PB_R = 4;                    // independent rows (float4 loads) in flight per lane
constexpr int PB_TILE = 512;               // rows per tile (= PB_GROUPS * PB_R * 4 passes)
constexpr int PB_MAX_D = 1024;             // generic path: query vector staged in shared memory

__device__ __forceinline__ int hist_bin(float dd, const float *edges) {
    // upper_bound(edges, dd) - 1 with the last bin right-inclusive (torch.histogram, linear bins
    // + local search against the fp32 edge table).  Caller guarantees edges[0] <= dd <= edges[60].
    int b = (int)(dd * 200.0f);
    b = max(0, min(VK_NBINS - 1, b));
    while (b > 0 && dd < edges[b]) --b;
    while (b < VK_NBINS - 1 && dd >= edges[b + 1]) ++b;
    return b;
}

struct ProbeAcc {
    u64 dens;
    u64 dens_hi;
    unsigned nlt;
    unsigned rank;
};

// One pass over the live rows.  The hot loop is load + 4 fma + 3 shuffles per lane; everything else
// (mask lookup, length load, histogram / density / list bookkeeping) happens only for the few rows whose
// distance is small enough to matter.  Neighbour-list entries are staged per WARP (ballot-compacted,
// no block barrier) and flushed with one global reservation per ~48 entries.
constexpr int PB_WBUF = 64;  // staged entries per warp (<= 16 appended per iteration)

// R = independent rows (float4 loads) in flight per lane and per buffer (the chunk being processed and the next one);
// BPS = resident blocks per SM the register budget is held to.
template <int DFIX, int R, int BPS>
__global__ void __launch_bounds__(PB_THREADS, BPS)
probe_kernel(const float *__restrict__ matrix, const float *__restrict__ lengths,
             const uint8_t *__restrict__ kept, int64_t n, int d_rt, int64_t mrow, float nl_radius,
             const float *__restrict__ edges_g, vk_probe_header *hdr, int32_t *within_overflow,
             int32_t *nl_rows, float *nl_dists, int n_tiles, vk_probe_header *hdr_mapped, int32_t *done_ticket,
             volatile int32_t *done_flag, int32_t seq, int32_t *work_counter, int unit_chunks) {
    const int d = DFIX ? DFIX : d_rt;
    tl_begin(0);
    __shared__ float s_edges[VK_NBINS + 1];
    __shared__ u64 s_hist[VK_NBINS];
    __shared__ int32_t s_wrows[PB_THREADS / 32][PB_WBUF];
    __shared__ float s_wd[PB_THREADS / 32][PB_WBUF];
    __shared__ ProbeAcc s_acc;
    __shared__ __align__(16) float s_q[DFIX ? DFIX : PB_MAX_D];

    const int tid = threadIdx.x;
    const int lane8 = tid & 7, lane = tid & 31, warp = tid >> 5;
    const int g = tid >> 3;
    const unsigned gmask = group8_mask();
    const unsigned lt_mask = (1u << lane) - 1u;
    const bool vec4 = (d & 3) == 0;

    if (tid <= VK_NBINS) s_edges[tid] = edges_g[tid];
    if (tid < VK_NBINS) s_hist[tid] = 0ull;
    if (tid == 0) { s_acc.dens = 0ull; s_acc.dens_hi = 0ull; s_acc.nlt = 0u; s_acc.rank = 0u; }
    for (int k = tid; k < d; k += PB_THREADS) s_q[k] = matrix[mrow * (int64_t)d + k];
    // rank = number of kept rows before the medoid row (the reference's packed index of the seed,
    // vamb/cluster.py:370): a grid-strided pass over kept[0, mrow) (1 byte per row) instead of a launch of its own
    {
        unsigned cnt = 0;
        const int64_t words = mrow >> 2;  // kept is at least 4-byte aligned (a tensor of its own)
        const uint32_t *k4 = reinterpret_cast<const uint32_t *>(kept);
        for (int64_t i = (int64_t)blockIdx.x * PB_THREADS + tid; i < words; i += (int64_t)gridDim.x * PB_THREADS)
            cnt += __popc(__ldg(k4 + i) & 0x01010101u);  // the mask holds 0 / 1 bytes
        if (blockIdx.x == 0 && tid < (int)(mrow & 3)) cnt += kept[(words << 2) + tid] != 0;
        for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        if (lane == 0 && cnt) atomicAdd(&hdr->rank, (int)cnt);
    }
    __syncthreads();

    tl_mark(1);
    float4 qv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (DFIX == 32) qv = *reinterpret_cast<const float4 *>(s_q + 4 * lane8);
    const float e_lo = s_edges[0], e_hi = s_edges[VK_NBINS];
    const float rad = 0.05f;
    const float lim = fmaxf(fmaxf(nl_radius, e_hi), rad);  // rows beyond this distance need no bookkeeping

    u64 t_dens = 0ull, t_dens_hi = 0ull;
    unsigned t_nlt = 0u;
    int wcnt = 0;  // entries staged by this warp (warp-uniform)

    auto flush_warp = [&]() {
        __syncwarp();
        int base = 0;
        if (lane == 0 && wcnt) base = atomicAdd(&hdr->n_nl, wcnt);
        base = __shfl_sync(0xffffffffu, base, 0);
        for (int i = lane; i < wcnt; i += 32) {
            nl_rows[base + i] = s_wrows[warp][i];
            nl_dists[base + i] = s_wd[warp][i];
        }
        __syncwarp();
        wcnt = 0;
    };

    // for D = 32 the next chunk's loads are issued before the current chunk is processed (register double buffering)
    // so that every resident warp keeps 128 bytes per lane in flight.
    constexpr int PB_R = R;
    const int n32 = (int)n;
    float4 vnext[PB_R];
    // Work distribution, PER WARP and without any block barrier: a warp-chunk is 4 x R consecutive rows (one 512-byte
    // load per k for the warp, 2 KB at R = 4), a unit is `unit_chunks` warp-chunks.  Default: units strided over the
    // warps of the grid, four chunks (8 KB) per unit (VK_PROBE_UNIT) -- at any moment the grid streams one contiguous
    // window of the matrix.  The alternative VK_PROBE_DYNAMIC=1 draws units from one atomic counter, two ahead, so that
    // faster SMs scan more rows (tools/probe_speed.py compares the two).
    constexpr int WCHUNK = 4 * PB_R;
    const int PB_WUNIT = unit_chunks;
    const int n_wchunks = (n32 + WCHUNK - 1) / WCHUNK;
    const int n_units = (n_wchunks + PB_WUNIT - 1) / PB_WUNIT;
    const int gw = lane >> 3;  // group of the lane inside its warp
    int static_unit = (int)blockIdx.x * (PB_THREADS / 32) + warp;  // lane 0 only
    auto fetch_lane0 = [&]() -> int {  // called by lane 0; the result is consumed later (no immediate dependency)
        if (work_counter) return atomicAdd(work_counter, 1);
        const int u = static_unit;
        static_unit += (int)gridDim.x * (PB_THREADS / 32);
        return u;
    };
    auto load_wchunk = [&](int wc, float4 (&v)[PB_R]) {
#pragma unroll
        for (int k = 0; k < PB_R; ++k) {
            const int row = wc * WCHUNK + k * 4 + gw;
            v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (row < n32) v[k] = ldg_stream4(matrix + (int64_t)row * 32 + 4 * lane8);
        }
    };
    int cur = 0, nxt = 0;
    {
        int a0 = 0, a1 = 0;
        if (lane == 0) { a0 = fetch_lane0(); a1 = fetch_lane0(); }
        cur = __shfl_sync(0xffffffffu, a0, 0);
        nxt = __shfl_sync(0xffffffffu, a1, 0);
    }
    if (DFIX == 32 && cur < n_units) load_wchunk(cur * PB_WUNIT, vnext);
#pragma unroll 1
    while (cur < n_units) {
        int pending = 0;
        if (lane == 0) pending = fetch_lane0();  // the unit after next
#pragma unroll 1
        for (int it = 0; it < PB_WUNIT; ++it) {
        const int c = cur * PB_WUNIT + it;
        if (c >= n_wchunks) break;
        float acc[PB_R];
        int rows[PB_R];
#pragma unroll
        for (int k = 0; k < PB_R; ++k) rows[k] = c * WCHUNK + k * 4 + gw;
        if (DFIX == 32) {
            float4 v[PB_R];
#pragma unroll
            for (int k = 0; k < PB_R; ++k) v[k] = vnext[k];
            // the warp's next chunk: the following one of the unit, else the first one of its next unit
            const bool unit_end = (it + 1 == PB_WUNIT) || (c + 1 >= n_wchunks);
            if (!unit_end) load_wchunk(c + 1, vnext);
            else if (nxt < n_units) load_wchunk(nxt * PB_WUNIT, vnext);
#pragma unroll
            for (int k = 0; k < PB_R; ++k) acc[k] = chain4(v[k], qv);
        } else {
#pragma unroll
            for (int k = 0; k < PB_R; ++k) {
                acc[k] = 0.0f;
                if (rows[k] < n32) acc[k] = lane_chain_generic(matrix + rows[k] * (int64_t)d, s_q, d, lane8, vec4);
            }
        }
#pragma unroll
        for (int k = 0; k < PB_R; ++k) acc[k] = group8_sum(acc[k], gmask);

#pragma unroll
        for (int k = 0; k < PB_R; ++k) {
            const int row = rows[k];
            float dd = __fsub_rn(0.5f, acc[k]);
            if (row == (int)mrow) dd = 0.0f;
            bool cand = (lane8 == 0) && (row < n32) && (dd <= lim);
            if (cand) cand = kept[row] != 0;  // rare: the mask is only consulted for near rows
            const bool nl_hit = cand && (dd <= nl_radius);
            const unsigned ballot = __ballot_sync(0xffffffffu, nl_hit);
            if (ballot) {
                if (nl_hit) {
                    const int pos = wcnt + __popc(ballot & lt_mask);
                    s_wrows[warp][pos] = row;
                    s_wd[warp][pos] = dd;
                }
                wcnt += __popc(ballot);
            }
            if (cand) {
                if (dd < rad) ++t_nlt;
                const bool in_hist = (dd >= e_lo) && (dd <= e_hi);
                const bool within = dd <= rad;
                if (in_hist || within) {
                    const u64 len = __float2ull_rz(__ldg(lengths + row));
                    if (within) {
                        density_add(t_dens, t_dens_hi, len, closeness_fx(rad, dd));
                        const int pos = atomicAdd(&hdr->n_within, 1);
                        if (pos < VK_PROBE_INLINE) hdr->within[pos] = row;
                        else within_overflow[pos] = row;
                    }
                    if (in_hist) atomicAdd(&s_hist[hist_bin(dd, s_edges)], len);
                }
            }
        }
        if (wcnt > PB_WBUF - 4 * PB_R) flush_warp();  // a warp appends at most 4 entries per row slot
        }
        cur = nxt;
        nxt = __shfl_sync(0xffffffffu, pending, 0);
    }
    tl_mark(2);
    flush_warp();

    if (lane8 == 0 && (t_dens | t_dens_hi | t_nlt)) {
        if (t_dens) atomicAdd(&s_acc.dens, t_dens);
        if (t_dens_hi) atomicAdd(&s_acc.dens_hi, t_dens_hi);
        if (t_nlt) atomicAdd(&s_acc.nlt, t_nlt);
    }
    __syncthreads();
    if (tid < VK_NBINS) {
        const u64 h = s_hist[tid];
        if (h) atomicAdd(reinterpret_cast<u64 *>(&hdr->hist[tid]), h);
    }
    if (tid == 64) {
        if (s_acc.dens) atomicAdd(reinterpret_cast<u64 *>(&hdr->density_lo), s_acc.dens);
        if (s_acc.dens_hi) atomicAdd(reinterpret_cast<u64 *>(&hdr->density_hi), s_acc.dens_hi);
        if (s_acc.nlt) atomicAdd(&hdr->n_lt, (int)s_acc.nlt);
    }
    tl_mark(3);
    if (hdr_mapped == nullptr) return;
    // Mapped completion (vk_probe_mapped): the last block to finish copies the header into pinned host memory,
    // leaves the device accumulators zeroed for the next probe and raises the flag the host is spinning on --
    // one launch per probe instead of memset + kernel + copy + stream synchronisation.
    __shared__ int s_last;
    tl_mark(4);
    if (!vk_last_block(done_ticket, &s_last)) return;
    tl_mark_any(5);
    if (tid == 0 && work_counter) *work_counter = 0;  // every block has drawn its last unit before its ticket
    constexpr int HEAD_WORDS = (int)(offsetof(vk_probe_header, within) / sizeof(u64));  // accumulators + counters
    if (tid < HEAD_WORDS) reinterpret_cast<u64 *>(hdr_mapped)[tid] = __ldcg(reinterpret_cast<const u64 *>(hdr) + tid);
    int nw = __ldcg(&hdr->n_within);
    nw = nw < VK_PROBE_INLINE ? nw : VK_PROBE_INLINE;
    for (int i = tid; i < nw; i += PB_THREADS) hdr_mapped->within[i] = __ldcg(&hdr->within[i]);
    __syncthreads();
    if (tid < HEAD_WORDS) reinterpret_cast<u64 *>(hdr)[tid] = 0ull;
    tl_mark_any(6);
    vk_raise_flag(done_flag, seq);
    tl_mark_any(7);
}

// Launch shape of the probe: rows in flight per lane (VK_PROBE_R = 4 | 8) and persistent blocks per SM
// (VK_PROBE_BPS = 2..8).  Chosen on an H100 SXM (400 W power limit) with tools/probe_speed.py, one launch, warm L2,
// N = 1M / 5M: R = 4 with BPS = 4 -> 71 / 242 us, BPS = 3 -> 72 / 241 us, BPS = 2 -> 76 / 263 us, BPS = 6 -> 80 / 278 us,
// BPS = 8 -> 91 / 286 us; R = 8 with BPS = 2 -> 80 / 255 us, BPS = 4 -> 84 / 279 us.
static int probe_env(const char *name, int dflt, int lo, int hi) {
    const char *v = getenv(name);
    const int x = v ? atoi(v) : dflt;
    return x < lo ? lo : (x > hi ? hi : x);
}
static int probe_r() {
    static const int r = probe_env("VK_PROBE_R", 4, 4, 8) >= 8 ? 8 : 4;
    return r;
}
static int probe_bps() {
    static const int b = probe_env("VK_PROBE_BPS", 4, 1, 8);
    return b;
}
static int probe_grid(int n_chunks) {
    const int cap = vk_num_sms() * probe_bps();
    return n_chunks < cap ? n_chunks : cap;
}

static int probe_launch(const float *matrix, const float *lengths, const uint8_t *kept, int64_t n, int d,
                        int64_t medoid_row, float nl_radius, const float *edges, vk_probe_header *hdr,
                        int32_t *within_overflow, int32_t *nl_rows, float *nl_dists, vk_probe_header *hdr_mapped,
                        int32_t *done_ticket, int32_t *done_flag, int32_t seq, int32_t *work_counter, cudaStream_t s) {
    if (n <= 0 || medoid_row < 0 || medoid_row >= n) {
        vk_set_error("vk_probe: bad arguments (n=%lld, medoid_row=%lld)", (long long)n, (long long)medoid_row);
        return 1;
    }
    if (d < 1 || d > PB_MAX_D) {
        vk_set_error("vk_probe: d=%d outside [1, %d]", d, PB_MAX_D);
        return 1;
    }
    if (n > 2147483647LL) {
        vk_set_error("vk_probe: n=%lld exceeds int32 row ids", (long long)n);
        return 1;
    }
    // only the accumulators need zeroing, not the inline id list (the mapped variant leaves them zeroed itself)
    if (!hdr_mapped) VK_CUDA(cudaMemsetAsync(hdr, 0, offsetof(vk_probe_header, within), s));
    if ((reinterpret_cast<uintptr_t>(kept) & 3) != 0) {
        vk_set_error("vk_probe: the kept mask must be 4-byte aligned");
        return 1;
    }
    const int r = probe_r();
    static const int unit = probe_env("VK_PROBE_UNIT", 4, 1, 64);
    static const int dynamic_units = probe_env("VK_PROBE_DYNAMIC", 0, 0, 1);
    if (!dynamic_units) work_counter = nullptr;
    const int n_chunks = (int)((n + PB_GROUPS * r - 1) / (PB_GROUPS * r));
    const int grid = probe_grid(n_chunks);
#define VK_PROBE_LAUNCH(DF, RR, BB)                                                                                  \
    probe_kernel<DF, RR, BB><<<grid, PB_THREADS, 0, s>>>(matrix, lengths, kept, n, d, medoid_row, nl_radius, edges, hdr, \
                                                         within_overflow, nl_rows, nl_dists, n_chunks, hdr_mapped,       \
                                                         done_ticket, done_flag, seq, work_counter, unit)
    if (d == 32) {
        if (r == 8) VK_PROBE_LAUNCH(32, 8, 3);
        else if (probe_bps() > 4) VK_PROBE_LAUNCH(32, 4, 6);
        else VK_PROBE_LAUNCH(32, 4, 4);
    } else {
        VK_PROBE_LAUNCH(0, 4, 4);
    }
#undef VK_PROBE_LAUNCH
    VK_LAUNCH_CHECK();
    return 0;
}

extern "C" int vk_probe(const float *matrix, const float *lengths, const uint8_t *kept, int64_t n, int d,
                        int64_t medoid_row, float nl_radius, const float *edges, vk_probe_header *hdr,
                        int32_t *within_overflow, int32_t *nl_rows, float *nl_dists, void *stream) {
    return probe_launch(matrix, lengths, kept, n, d, medoid_row, nl_radius, edges, hdr, within_overflow, nl_rows,
                        nl_dists, nullptr, nullptr, nullptr, 0, nullptr, (cudaStream_t)stream);
}

// Spin on a flag in pinned host memory that the last block of a kernel sets to `seq`; the stream is only
// queried now and then, to turn a failed launch into an error instead of a hang.
static int wait_flag(const volatile int32_t *flag, int32_t seq, cudaStream_t s, const char *what) {
    for (uint64_t it = 1;; ++it) {
        if (*flag == seq) return 0;
        if ((it & 0x3FFFFull) == 0) {
            const cudaError_t e = cudaStreamQuery(s);
            if (e == cudaSuccess) {
                if (*flag == seq) return 0;
                vk_set_error("%s: the stream drained without raising the completion flag", what);
                return 1;
            }
            if (e != cudaErrorNotReady) {
                vk_set_error("%s: %s", what, cudaGetErrorString(e));
                return 1;
            }
        }
    }
}

extern "C" int vk_probe_mapped(const float *matrix, const float *lengths, const uint8_t *kept, int64_t n, int d,
                               int64_t medoid_row, float nl_radius, const float *edges, vk_probe_header *hdr,
                               int32_t *within_overflow, int32_t *nl_rows, float *nl_dists,
                               vk_probe_header *hdr_pinned, int32_t *done_ticket, int32_t *done_flag_pinned, int32_t seq,
                               int32_t *work_counter, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (probe_launch(matrix, lengths, kept, n, d, medoid_row, nl_radius, edges, hdr, within_overflow, nl_rows, nl_dists,
                     hdr_pinned, done_ticket, done_flag_pinned, seq, work_counter, s))
        return 1;
    return wait_flag(done_flag_pinned, seq, s, "vk_probe_mapped");
}

extern "C" int vk_probe_sync(const float *matrix, const float *lengths, const uint8_t *kept, int64_t n, int d,
                             int64_t medoid_row, float nl_radius, const float *edges, vk_probe_header *hdr,
                             int32_t *within_overflow, int32_t *nl_rows, float *nl_dists,
                             vk_probe_header *hdr_host, void *stream) {
    if (vk_probe(matrix, lengths, kept, n, d, medoid_row, nl_radius, edges, hdr, within_overflow, nl_rows,
                 nl_dists, stream))
        return 1;
    cudaStream_t s = (cudaStream_t)stream;
    VK_CUDA(cudaMemcpyAsync(hdr_host, hdr, sizeof(vk_probe_header), cudaMemcpyDeviceToHost, s));
    VK_CUDA(cudaStreamSynchronize(s));
    return 0;
}

// ------------------------------------------------------------------ plain distance vector
template <int DFIX>
__global__ void __launch_bounds__(PB_THREADS, 4)
distances_kernel(const float *__restrict__ matrix, int64_t n, int d_rt, int64_t mrow, float *__restrict__ dists,
                 int n_tiles) {
    const int d = DFIX ? DFIX : d_rt;
    __shared__ __align__(16) float s_q[DFIX ? DFIX : PB_MAX_D];
    const int tid = threadIdx.x, lane8 = tid & 7, g = tid >> 3;
    const unsigned gmask = group8_mask();
    const bool vec4 = (d & 3) == 0;
    for (int k = tid; k < d; k += PB_THREADS) s_q[k] = matrix[mrow * (int64_t)d + k];
    __syncthreads();
    float4 qv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (DFIX == 32) qv = *reinterpret_cast<const float4 *>(s_q + 4 * lane8);
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int64_t row0 = (int64_t)tile * PB_TILE;
#pragma unroll 1
        for (int it = 0; it < PB_TILE / (PB_GROUPS * PB_R); ++it) {
            float acc[PB_R];
            int64_t rows[PB_R];
            if (DFIX == 32) {
                float4 v[PB_R];
#pragma unroll
                for (int k = 0; k < PB_R; ++k) {
                    rows[k] = row0 + (int64_t)(it * PB_R + k) * PB_GROUPS + g;
                    v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (rows[k] < n) v[k] = ldg_stream4(matrix + rows[k] * 32 + 4 * lane8);
                }
#pragma unroll
                for (int k = 0; k < PB_R; ++k) acc[k] = chain4(v[k], qv);
            } else {
#pragma unroll
                for (int k = 0; k < PB_R; ++k) {
                    rows[k] = row0 + (int64_t)(it * PB_R + k) * PB_GROUPS + g;
                    acc[k] = 0.0f;
                    if (rows[k] < n) acc[k] = lane_chain_generic(matrix + rows[k] * (int64_t)d, s_q, d, lane8, vec4);
                }
            }
#pragma unroll
            for (int k = 0; k < PB_R; ++k) {
                acc[k] = group8_sum(acc[k], gmask);
                if (lane8 == 0 && rows[k] < n) dists[rows[k]] = rows[k] == mrow ? 0.0f : __fsub_rn(0.5f, acc[k]);
            }
        }
    }
}

extern "C" int vk_distances(const float *matrix, int64_t n, int d, int64_t medoid_row, float *dists, void *stream) {
    if (n <= 0 || medoid_row < 0 || medoid_row >= n || d < 1 || d > PB_MAX_D) {
        vk_set_error("vk_distances: bad arguments");
        return 1;
    }
    const int n_tiles = (int)((n + PB_TILE - 1) / PB_TILE);
    const int grid = probe_grid(n_tiles);
    cudaStream_t s = (cudaStream_t)stream;
    if (d == 32) distances_kernel<32><<<grid, PB_THREADS, 0, s>>>(matrix, n, d, medoid_row, dists, n_tiles);
    else distances_kernel<0><<<grid, PB_THREADS, 0, s>>>(matrix, n, d, medoid_row, dists, n_tiles);
    VK_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------ candidate evaluation
struct CandRows {
    int32_t rows[VK_MAX_CAND];
};

constexpr int EC_THREADS = 256;

__global__ void __launch_bounds__(EC_THREADS)
eval_candidates_kernel(const float *__restrict__ matrix, const float *__restrict__ lengths, int d,
                       const int32_t *__restrict__ nl_rows, const float *__restrict__ nl_dists, int n_nl,
                       float prune_radius, CandRows cand, int n_cand, u64 *out, u64 *out_mapped, int32_t *done_ticket,
                       volatile int32_t *done_flag, int32_t seq) {
    extern __shared__ __align__(16) float s_qs[];  // [n_cand][dpad]
    __shared__ u64 s_dens[VK_MAX_CAND];
    __shared__ u64 s_dens_hi[VK_MAX_CAND];
    __shared__ unsigned s_cnt[VK_MAX_CAND];
    const int tid = threadIdx.x, lane8 = tid & 7, g = tid >> 3;
    const unsigned gmask = group8_mask();
    const int dpad = (d + 3) & ~3;
    const bool vec4 = (d & 3) == 0;
    __shared__ int32_t s_crow[VK_MAX_CAND];  // static-index copy of the by-value parameter (no local-memory spill)
#pragma unroll
    for (int k = 0; k < VK_MAX_CAND; ++k)
        if (tid == k) s_crow[k] = k < n_cand ? cand.rows[k] : -1;
    if (tid < VK_MAX_CAND) { s_dens[tid] = 0ull; s_dens_hi[tid] = 0ull; s_cnt[tid] = 0u; }
    __syncthreads();
    for (int i = tid; i < n_cand * dpad; i += EC_THREADS) {
        const int k = i / dpad, c = i - k * dpad;
        s_qs[i] = c < d ? matrix[(int64_t)s_crow[k] * d + c] : 0.0f;
    }
    __syncthreads();

    const float rad = 0.05f;
    const int groups_total = gridDim.x * (EC_THREADS / 8);
    for (int j = blockIdx.x * (EC_THREADS / 8) + g; j < n_nl; j += groups_total) {
        const float dj = nl_dists[j];
        if (!(dj <= prune_radius)) continue;  // uniform within the 8-lane group
        const int row = nl_rows[j];
        const float *x = matrix + (int64_t)row * d;
        float4 xv = make_float4(0.f, 0.f, 0.f, 0.f);
        const bool fast = (d == 32);
        if (fast) xv = ldg_stream4(x + 4 * lane8);
        u64 lenq = 0ull;
        if (lane8 == 0) lenq = __float2ull_rz(__ldg(lengths + row));
        for (int k = 0; k < n_cand; ++k) {
            const float *q = s_qs + k * dpad;
            float acc;
            if (fast) acc = chain4(xv, *reinterpret_cast<const float4 *>(q + 4 * lane8));
            else acc = lane_chain_generic(x, q, d, lane8, vec4);
            acc = group8_sum(acc, gmask);
            if (lane8 == 0) {
                float dd = __fsub_rn(0.5f, acc);
                if (row == s_crow[k]) dd = 0.0f;
                if (dd <= rad) {
                    const u64 cq = closeness_fx(rad, dd);
                    atomicAdd(&s_dens[k], lenq * (cq & 4095ull));
                    atomicAdd(&s_dens_hi[k], lenq * (cq >> 12));
                    atomicAdd(&s_cnt[k], 1u);
                }
            }
        }
    }
    __syncthreads();
    if (tid < n_cand) {
        if (s_dens[tid]) atomicAdd(&out[tid], s_dens[tid]);
        if (s_dens_hi[tid]) atomicAdd(&out[VK_MAX_CAND + tid], s_dens_hi[tid]);
        if (s_cnt[tid]) atomicAdd(&out[2 * VK_MAX_CAND + tid], (u64)s_cnt[tid]);
    }
    if (out_mapped == nullptr) return;
    // mapped completion, as in probe_kernel: results to pinned host memory, accumulators left zeroed, flag raised
    __shared__ int s_last;
    if (!vk_last_block(done_ticket, &s_last)) return;
    if (tid < 3 * VK_MAX_CAND) {
        out_mapped[tid] = __ldcg(out + tid);
        out[tid] = 0ull;
    }
    vk_raise_flag(done_flag, seq);
}

extern "C" int vk_eval_candidates_sync(const float *matrix, const float *lengths, int d, const int32_t *nl_rows,
                                       const float *nl_dists, int32_t n_nl, float prune_radius,
                                       const int32_t *cand_rows_host, int n_cand, uint64_t *out_dev,
                                       uint64_t *out_host, void *stream) {
    if (n_cand < 1 || n_cand > VK_MAX_CAND) {
        vk_set_error("vk_eval_candidates_sync: n_cand=%d outside [1, %d]", n_cand, VK_MAX_CAND);
        return 1;
    }
    if (d < 1 || d > PB_MAX_D) {
        vk_set_error("vk_eval_candidates_sync: d=%d outside [1, %d]", d, PB_MAX_D);
        return 1;
    }
    cudaStream_t s = (cudaStream_t)stream;
    CandRows cand;
    memset(&cand, 0, sizeof(cand));
    for (int k = 0; k < n_cand; ++k) cand.rows[k] = cand_rows_host[k];
    VK_CUDA(cudaMemsetAsync(out_dev, 0, sizeof(uint64_t) * 3 * VK_MAX_CAND, s));
    if (n_nl > 0) {
        const int dpad = (d + 3) & ~3;
        const size_t smem = sizeof(float) * (size_t)n_cand * dpad;
        if (smem > 48 * 1024) {
            VK_CUDA(cudaFuncSetAttribute(eval_candidates_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        }
        const int per_block = EC_THREADS / 8;
        int grid = (n_nl + per_block - 1) / per_block;
        const int cap = vk_num_sms() * 4;
        if (grid > cap) grid = cap;
        eval_candidates_kernel<<<grid, EC_THREADS, smem, s>>>(matrix, lengths, d, nl_rows, nl_dists, n_nl,
                                                              prune_radius, cand, n_cand, (u64 *)out_dev, nullptr,
                                                              nullptr, nullptr, 0);
        VK_LAUNCH_CHECK();
    }
    VK_CUDA(cudaMemcpyAsync(out_host, out_dev, sizeof(uint64_t) * 3 * VK_MAX_CAND, cudaMemcpyDeviceToHost, s));
    VK_CUDA(cudaStreamSynchronize(s));
    return 0;
}

// Same results through the mapped completion: out_dev must be all zero on entry (it is left zeroed again).
extern "C" int vk_eval_candidates_mapped(const float *matrix, const float *lengths, int d, const int32_t *nl_rows,
                                         const float *nl_dists, int32_t n_nl, float prune_radius,
                                         const int32_t *cand_rows_host, int n_cand, uint64_t *out_dev,
                                         uint64_t *out_pinned, int32_t *done_ticket, int32_t *done_flag_pinned,
                                         int32_t seq, void *stream) {
    if (n_cand < 1 || n_cand > VK_MAX_CAND) {
        vk_set_error("vk_eval_candidates_mapped: n_cand=%d outside [1, %d]", n_cand, VK_MAX_CAND);
        return 1;
    }
    if (d < 1 || d > PB_MAX_D) {
        vk_set_error("vk_eval_candidates_mapped: d=%d outside [1, %d]", d, PB_MAX_D);
        return 1;
    }
    if (n_nl <= 0) {
        memset(out_pinned, 0, sizeof(uint64_t) * 3 * VK_MAX_CAND);
        return 0;
    }
    cudaStream_t s = (cudaStream_t)stream;
    CandRows cand;
    memset(&cand, 0, sizeof(cand));
    for (int k = 0; k < n_cand; ++k) cand.rows[k] = cand_rows_host[k];
    const int dpad = (d + 3) & ~3;
    const size_t smem = sizeof(float) * (size_t)n_cand * dpad;
    if (smem > 48 * 1024) {
        VK_CUDA(cudaFuncSetAttribute(eval_candidates_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    const int per_block = EC_THREADS / 8;
    int grid = (n_nl + per_block - 1) / per_block;
    const int cap = vk_num_sms() * 4;
    if (grid > cap) grid = cap;
    eval_candidates_kernel<<<grid, EC_THREADS, smem, s>>>(matrix, lengths, d, nl_rows, nl_dists, n_nl, prune_radius, cand,
                                                          n_cand, (u64 *)out_dev, (u64 *)out_pinned, done_ticket,
                                                          done_flag_pinned, seq);
    VK_LAUNCH_CHECK();
    return wait_flag(done_flag_pinned, seq, s, "vk_eval_candidates_mapped");
}

// ------------------------------------------------------------------ candidate evaluation with within-lists
struct CandRowsL {
    int32_t rows[VK_LIST_CAND];
};
// Device accumulators of eval_candidates_lists_kernel: VK_EVAL_SUBS copies ("subs", picked by blockIdx) of one 128-byte
// line per candidate (u64 words: 0 density lo, 1 density hi, 2 count, 3 float bits of d(candidate, base)).  With the
// compact [field][candidate] layout all counts of a launch shared 3-4 lines and every block's atomics queued up behind
// each other in the same L2 slices: the last block finished ~15 us after the first whatever was done inside the blocks
// (tools/probe_timeline.py); one line per (sub, candidate) spreads them over 4 x n_cand lines.
constexpr int EV_LINE = 16;  // u64 words per (sub, candidate)
constexpr int EC_QS = 36;    // floats between candidate rows / row buffers in shared memory (d = 32): 8 lanes reading 8
                             // different rows with float4 loads touch 8 distinct bank quads
__device__ __forceinline__ u64 *ev_slot(u64 *out, int sub, int k, int field) {
    return out + ((size_t)(sub * VK_LIST_CAND + k) * EV_LINE + field);
}
static_assert(VK_EVAL_SUBS * VK_LIST_CAND * EV_LINE == VK_EVAL_SCRATCH_U64, "eval scratch size");

// As eval_candidates_kernel, plus what lets the host MOVE the medoid to a winning candidate without another full
// scan: the ids of the rows within 0.05 of every candidate (the candidate's `cluster` of sample_medoid,
// vamb/cluster.py:626) go straight into pinned host memory, and the distance of every candidate to the medoid whose
// neighbour list is being used (`base_row`) is reported so that the host can tell whether that list covers the
// candidate's whole 0.05-neighbourhood (d(candidate, base) <= 0.12: angles add, DESIGN.md section 5).
// out / out_mapped: [0, C) density lo | [C, 2C) density hi | [2C, 3C) counts | [3C, 4C) d(candidate, base) as float bits.
__global__ void __launch_bounds__(EC_THREADS)
eval_candidates_lists_kernel(const float *__restrict__ matrix, const float *__restrict__ lengths, int d,
                             const int32_t *__restrict__ nl_rows, const float *__restrict__ nl_dists, int n_nl,
                             float prune_radius, const __grid_constant__ CandRowsL cand, int n_cand, int32_t base_row, u64 thr_hi, u64 thr_lo, u64 *out,
                             u64 *out_mapped,
                             int32_t *within_dev, int32_t *within_mapped, int within_cap, int32_t *done_ticket,
                             volatile int32_t *done_flag, int32_t seq) {
    tl_begin(1);
    // per-block stamps (stamped build only; tools/probe_timeline.py): point i of block b < 320 at vk_tl[EVT_BASE(i) + b]
#ifdef VK_TIMELINE
#define EVT(i)                                                                        \
    do {                                                                              \
        if (threadIdx.x == 0 && blockIdx.x < 320) {                                   \
            unsigned long long t_;                                                    \
            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_));                    \
            vk_tl[((i) < 4 ? 512 + 320 * (i) : 2560 + 320 * ((i) - 4)) + blockIdx.x] = t_; \
        }                                                                             \
    } while (0)
#else
#define EVT(i) ((void)0)
#endif
    EVT(0);
    extern __shared__ __align__(16) float s_qs[];  // [n_cand][qs]: qs = 36 for d = 32 (conflict-free float4 reads by 8 lanes
                                                   // holding 8 different candidates), else dpad
    // A hit = (row within 0.05 of candidate k).  The lane that scans a row of a dense core finds a hit for almost every
    // candidate; doing the bookkeeping there (shared atomics + a returning global atomic per hit) serialised 40 x ~1 us
    // in that one lane, and folding recorded hits with 64-bit shared atomics (CAS loops, 32 hits of one candidate in
    // consecutive threads) still left the last block 16 us behind the first (tools/probe_timeline.py).  So the scan only
    // WRITES each hit into its own cell of a dense [row slot][candidate] table -- no atomic at all -- and the fold is a
    // fixed ownership: thread (candidate k, quarter p) reads the 8 row slots of its quarter, keeps the candidate's sums
    // in REGISTERS over all rounds, one thread per candidate reserves ONE range in the global id list per round, and the
    // owners scatter the ids (and clear their cells).
    constexpr int EC_SLOTS = EC_THREADS / 8;             // rows per block and round
    constexpr int EC_PARTS = EC_THREADS / VK_LIST_CAND;  // owners per candidate
    constexpr int EC_PER = EC_SLOTS / EC_PARTS;          // row slots per owner
    static_assert(EC_THREADS % VK_LIST_CAND == 0 && EC_SLOTS % EC_PARTS == 0, "eval ownership");
    __shared__ uint32_t s_cell[EC_SLOTS][VK_LIST_CAND];  // closeness + 1 of (row slot, candidate), 0 = no hit
    __shared__ int32_t s_slot_row[EC_SLOTS];
    __shared__ __align__(16) float s_rowbuf[EC_SLOTS][EC_QS];  // the row of every slot, readable by all lanes of its group
    __shared__ uint32_t s_slot_len[EC_SLOTS];
    __shared__ unsigned s_pcnt[EC_PARTS][VK_LIST_CAND];
    __shared__ u64 s_base[VK_LIST_CAND];
    __shared__ int32_t s_crow[VK_LIST_CAND];  // candidate rows out of the parameter
    __shared__ float s_reach[VK_LIST_CAND];
    const int tid = threadIdx.x, lane8 = tid & 7, g = tid >> 3;
    const unsigned gmask = group8_mask();
    const int dpad = (d + 3) & ~3;
    const bool vec4 = (d & 3) == 0;
    const bool fast = (d == 32);
    const int qs = fast ? EC_QS : dpad;
    if (tid < VK_LIST_CAND) s_crow[tid] = tid < n_cand ? cand.rows[tid] : -1;  // __grid_constant__: indexed constant load
    for (int i = tid; i < EC_SLOTS * VK_LIST_CAND; i += EC_THREADS) (&s_cell[0][0])[i] = 0u;
    __syncthreads();
    if (fast) {  // 8 float4 per candidate row, all loads independent
        for (int i = tid; i < n_cand * 8; i += EC_THREADS)
            *reinterpret_cast<float4 *>(s_qs + (i >> 3) * EC_QS + (i & 7) * 4) = ldg_stream4(matrix + (int64_t)s_crow[i >> 3] * 32 + (i & 7) * 4);
    } else {
        for (int i = tid; i < n_cand * dpad; i += EC_THREADS) {
            const int k = i / dpad, c = i - k * dpad;
            s_qs[i] = c < d ? matrix[(int64_t)s_crow[k] * d + c] : 0.0f;
        }
    }
    // the base row (for the candidates' distances to it) is loaded alongside
    const float *xb = matrix + (int64_t)base_row * d;
    float4 xbv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (fast) xbv = ldg_stream4(xb + 4 * lane8);
    __syncthreads();

    const float rad = 0.05f;
    // d(candidate, base) in the same arithmetic as every other distance -- every block computes all of them (n_cand dot
    // products): block 0 reports them, and each gives the candidate's REACH: a row within 0.05 of candidate k lies within
    // angle(d_k) + acos(0.9) of the base, i.e. at a base distance of at most
    //     reach_k = 0.5 * (1 - ((1 - 2 d_k) * 0.9 - sqrt(1 - (1 - 2 d_k)^2) * sqrt(0.19)))      (+ 1e-4 of slack).
    // Neighbour-list entries beyond max_k reach_k (and beyond `prune_radius`) cannot matter and are not gathered.
    for (int k = g; k < n_cand; k += EC_THREADS / 8) {
        const float *q = s_qs + k * qs;
        float acc = fast ? chain4(xbv, *reinterpret_cast<const float4 *>(q + 4 * lane8)) : lane_chain_generic(xb, q, d, lane8, vec4);
        acc = group8_sum(acc, gmask);
        if (lane8 == 0) {
            float dd = __fsub_rn(0.5f, acc);
            if (s_crow[k] == base_row) dd = 0.0f;
            if (blockIdx.x == 0) *ev_slot(out, 0, k, 3) = (u64)__float_as_uint(dd);
            const float ca = 1.0f - 2.0f * fmaxf(dd, 0.0f);
            const float sa = sqrtf(fmaxf(1.0f - ca * ca, 0.0f));
            const float cs = ca * 0.9f - sa * 0.43588990f;  // cos(angle(d_k) + acos(0.9))
            s_reach[k] = (ca <= -0.9f) ? 1e30f : 0.5f * (1.0f - cs) + 1e-4f;  // beyond 180 degrees: everything
        }
    }
    __syncthreads();
    tl_mark(1);
    // the bound is geometry on unit-norm rows: an infinite prune_radius (rows not verified as normalised) switches it off
    const bool geo = prune_radius < 1e29f;
    float reach = 0.0f;
    for (int k = 0; k < n_cand; ++k) reach = fmaxf(reach, s_reach[k]);
    const float visit_radius = geo ? fminf(prune_radius, reach) : prune_radius;
    const int groups_total = gridDim.x * EC_SLOTS;
    const int n_rounds = (n_nl + groups_total - 1) / groups_total;  // block-uniform
    const int own_k = tid & (VK_LIST_CAND - 1), own_p = tid / VK_LIST_CAND;
    const int sub = blockIdx.x & (VK_EVAL_SUBS - 1);
    u64 r_dens = 0ull, r_dens_hi = 0ull;  // sums of candidate own_k over this owner's row slots, all rounds
    for (int round = 0; round < n_rounds; ++round) {
        const int j = round * groups_total + blockIdx.x * EC_SLOTS + g;
        const float dj = j < n_nl ? nl_dists[j] : 1e30f;
        bool any = false;
        if (dj <= visit_radius) {  // uniform within the 8-lane group
            const int row = nl_rows[j];
            const float *x = matrix + (int64_t)row * d;
            float4 xv = make_float4(0.f, 0.f, 0.f, 0.f);
            if (fast) xv = ldg_stream4(x + 4 * lane8);
            if (lane8 == 0) {
                s_slot_row[g] = row;
                s_slot_len[g] = (uint32_t)__float2ull_rz(__ldg(lengths + row));  // integral, < 2^24 per contig
            }
            if (fast) {
                // Every lane of the group takes whole (row, candidate) pairs -- candidates lane8, lane8 + 8, ... -- with the
                // full row in registers: 8 independent fmaf chains and the butterfly's additions in the same order
                // ((p0+p1)+(p2+p3))+((p4+p5)+(p6+p7)), i.e. the same bits as group8_sum(chain4) without a shuffle.  (One
                // candidate at a time per group was a serial chain of n_cand x ~150 cycles, and the four groups of a warp
                // diverge on `dj`: blocks with rows near the candidates took 14 us against 3 us, tools/probe_timeline.py.)
                *reinterpret_cast<float4 *>(&s_rowbuf[g][4 * lane8]) = xv;
                __syncwarp(gmask);
                float4 xr[8];
#pragma unroll
                for (int l = 0; l < 8; ++l) xr[l] = *reinterpret_cast<const float4 *>(&s_rowbuf[g][4 * l]);
                for (int k = lane8; k < n_cand; k += 8) {
                    if (geo && !(dj <= s_reach[k])) continue;  // this row cannot be within 0.05 of candidate k
                    const float4 *q = reinterpret_cast<const float4 *>(s_qs + k * EC_QS);
                    float p[8];
#pragma unroll
                    for (int l = 0; l < 8; ++l) p[l] = chain4(xr[l], q[l]);
                    const float acc = __fadd_rn(__fadd_rn(__fadd_rn(p[0], p[1]), __fadd_rn(p[2], p[3])),
                                                __fadd_rn(__fadd_rn(p[4], p[5]), __fadd_rn(p[6], p[7])));
                    float dd = __fsub_rn(0.5f, acc);
                    if (row == s_crow[k]) dd = 0.0f;
                    if (dd <= rad) {
                        s_cell[g][k] = (uint32_t)closeness_fx(rad, dd) + 1u;  // closeness <= 0.05 * 2^29 < 2^25
                        any = true;
                    }
                }
                __syncwarp(gmask);  // the row buffer is rewritten in the next round
            } else
            for (int k = 0; k < n_cand; ++k) {
                if (geo && !(dj <= s_reach[k])) continue;  // this row cannot be within 0.05 of candidate k
                const float *q = s_qs + k * qs;
                float acc = lane_chain_generic(x, q, d, lane8, vec4);
                acc = group8_sum(acc, gmask);
                if (lane8 == 0) {
                    float dd = __fsub_rn(0.5f, acc);
                    if (row == s_crow[k]) dd = 0.0f;
                    if (dd <= rad) {
                        s_cell[g][k] = (uint32_t)closeness_fx(rad, dd) + 1u;
                        any = true;
                    }
                }
            }
        }
        EVT(1);
        if (!__syncthreads_or(any)) continue;  // no hit in this block and round (the common case away from the core)
        unsigned cnt = 0;
#pragma unroll 1
        for (int i = 0; i < EC_PER; ++i) {
            const int slot = own_p * EC_PER + i;
            const uint32_t c1 = s_cell[slot][own_k];
            if (c1) {
                const u64 cq = c1 - 1u, len = s_slot_len[slot];
                r_dens += len * (cq & 4095ull);
                r_dens_hi += len * (cq >> 12);
                ++cnt;
            }
        }
        s_pcnt[own_p][own_k] = cnt;
        __syncthreads();
        if (tid < n_cand) {
            unsigned tot = 0;
#pragma unroll 1
            for (int p = 0; p < EC_PARTS; ++p) tot += s_pcnt[p][tid];
            if (tot) s_base[tid] = atomicAdd(ev_slot(out, sub, tid, 2), (u64)tot);
        }
        __syncthreads();
        EVT(2);
        if (cnt) {
            u64 pos = s_base[own_k];
            for (int p = 0; p < own_p; ++p) pos += s_pcnt[p][own_k];
#pragma unroll 1
            for (int i = 0; i < EC_PER; ++i) {
                const int slot = own_p * EC_PER + i;
                if (s_cell[slot][own_k]) {
                    if (pos < (u64)within_cap) within_dev[((size_t)sub * VK_LIST_CAND + own_k) * within_cap + pos] = s_slot_row[slot];
                    ++pos;
                    s_cell[slot][own_k] = 0u;
                }
            }
        }
        __syncthreads();
    }
    EVT(3);
    tl_mark(2);
    tl_mark(3);
    // the owners of a candidate are combined in shared memory first: one pair of global atomics per (block, candidate)
    // -- with four times as many, on the same 2 x n_cand addresses from every block, the last block finished ~15 us
    // after the first (tools/probe_timeline.py)
    __shared__ u64 s_own[EC_PARTS][2][VK_LIST_CAND];
    s_own[own_p][0][own_k] = r_dens;
    s_own[own_p][1][own_k] = r_dens_hi;
    __syncthreads();
    if (tid < 2 * VK_LIST_CAND) {
        const int kk = tid & (VK_LIST_CAND - 1), which = tid / VK_LIST_CAND;
        u64 tot = 0ull;
#pragma unroll 1
        for (int p = 0; p < EC_PARTS; ++p) tot += s_own[p][which][kk];
        if (tot) atomicAdd(ev_slot(out, sub, kk, which), tot);
    }
    __shared__ int s_last;
    tl_mark(4);
    EVT(4);
    if (!vk_last_block(done_ticket, &s_last)) return;
    tl_mark_any(5);
    // The last block publishes: the id lists (device -> pinned host memory), then the sums and counts; ONE system-scope
    // fence (vk_raise_flag) orders all of it before the flag.  The lists are flattened so that every thread copies a few
    // ids with independent loads (a warp per candidate walked them one after the other: 6 us).
    __shared__ int s_off[VK_LIST_CAND + 1];
    __shared__ int s_len_k[VK_LIST_CAND];
    __shared__ int s_sub_len[VK_EVAL_SUBS][VK_LIST_CAND];
    static_assert(EC_THREADS >= VK_EVAL_SUBS * VK_LIST_CAND, "one thread per (sub, candidate)");
    if (tid < VK_EVAL_SUBS * VK_LIST_CAND) {  // the counts: independent loads, then a serial prefix in shared memory
        const int kk = tid & (VK_LIST_CAND - 1), sb = tid / VK_LIST_CAND;
        u64 cnt = kk < n_cand ? __ldcg(ev_slot(out, sb, kk, 2)) : 0ull;
        if (cnt > (u64)within_cap) cnt = (u64)within_cap;
        s_sub_len[sb][kk] = (int)cnt;
    }
    __syncthreads();
    if (tid < VK_LIST_CAND) {
        u64 lo = 0ull, hi = 0ull, cnt = 0ull;
#pragma unroll 1
        for (int sb = 0; sb < VK_EVAL_SUBS; ++sb) {
            lo += __ldcg(ev_slot(out, sb, tid, 0));
            hi += __ldcg(ev_slot(out, sb, tid, 1));
            cnt += __ldcg(ev_slot(out, sb, tid, 2));
        }
        out_mapped[tid] = lo;
        out_mapped[VK_LIST_CAND + tid] = hi;
        out_mapped[2 * VK_LIST_CAND + tid] = cnt;
        out_mapped[3 * VK_LIST_CAND + tid] = __ldcg(ev_slot(out, 0, tid, 3));
        // The ids are only ever needed for a candidate the medoid can MOVE to: one whose density exceeds the current
        // medoid's (thr = that density, which only grows during a wander).  density = hi * 4096 + lo, compared in the
        // normalised form (hi + (lo >> 12), lo & 4095).  Everything else skips the copy to host memory.
        const u64 nh = hi + (lo >> 12), nl = lo & 4095ull;
        const bool wanted = nh > thr_hi || (nh == thr_hi && nl > thr_lo);
        int tot = 0;
#pragma unroll 1
        for (int sb = 0; sb < VK_EVAL_SUBS; ++sb) tot += s_sub_len[sb][tid];
        s_len_k[tid] = !wanted ? 0 : (tot > within_cap ? within_cap : tot);
    }
    __syncthreads();
    if (tid == 0) {
        int run = 0;
        for (int kk = 0; kk < n_cand; ++kk) {
            s_off[kk] = run;
            run += s_len_k[kk];
        }
        s_off[n_cand] = run;
    }
    __syncthreads();
    for (int e = tid; e < s_off[n_cand]; e += EC_THREADS) {
        int lo = 0, hi = n_cand;  // the candidate whose range holds e: s_off[kk] <= e < s_off[kk + 1]
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (s_off[mid] <= e) lo = mid;
            else hi = mid;
        }
        int r = e - s_off[lo], sb = 0;  // position in the candidate's list = the subs' lists one after the other
        while (sb < VK_EVAL_SUBS - 1 && r >= s_sub_len[sb][lo]) {
            r -= s_sub_len[sb][lo];
            ++sb;
        }
        within_mapped[(size_t)lo * within_cap + (e - s_off[lo])] = __ldcg(within_dev + ((size_t)sb * VK_LIST_CAND + lo) * within_cap + r);
    }
    __syncthreads();  // every count has been read before the accumulators are zeroed below
    for (int i = tid; i < VK_EVAL_SUBS * VK_LIST_CAND * 4; i += EC_THREADS) *ev_slot(out, i >> 8, (i >> 2) & (VK_LIST_CAND - 1), i & 3) = 0ull;
    static_assert(VK_LIST_CAND == 64, "index split above");
    tl_mark_any(6);
    vk_raise_flag(done_flag, seq);
    tl_mark_any(7);
}

extern "C" int vk_eval_candidates_lists(const float *matrix, const float *lengths, int d, const int32_t *nl_rows,
                                        const float *nl_dists, int32_t n_nl, float prune_radius,
                                        const int32_t *cand_rows_host, int n_cand, int32_t base_row,
                                        uint64_t min_density_hi, uint64_t min_density_lo, uint64_t *out_dev,
                                        uint64_t *out_pinned, int32_t *within_dev, int32_t *within_pinned,
                                        int32_t within_cap, int32_t *done_ticket, int32_t *done_flag_pinned, int32_t seq,
                                        void *stream) {
    if (n_cand < 1 || n_cand > VK_LIST_CAND || within_cap < 1) {
        vk_set_error("vk_eval_candidates_lists: n_cand=%d outside [1, %d] or bad capacity", n_cand, VK_LIST_CAND);
        return 1;
    }
    if (d < 1 || d > PB_MAX_D || n_nl <= 0) {
        vk_set_error("vk_eval_candidates_lists: d=%d outside [1, %d] or empty neighbour list", d, PB_MAX_D);
        return 1;
    }
    cudaStream_t s = (cudaStream_t)stream;
    CandRowsL cand;
    memset(&cand, 0, sizeof(cand));
    for (int k = 0; k < n_cand; ++k) cand.rows[k] = cand_rows_host[k];
    const int dpad = (d + 3) & ~3;
    const size_t smem = sizeof(float) * (size_t)n_cand * (d == 32 ? EC_QS : dpad);
    if (smem > 48 * 1024)
        VK_CUDA(cudaFuncSetAttribute(eval_candidates_lists_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int per_block = EC_THREADS / 8;
    int grid = (n_nl + per_block - 1) / per_block;
    const int cap = vk_num_sms() * 4;
    if (grid > cap) grid = cap;
    eval_candidates_lists_kernel<<<grid, EC_THREADS, smem, s>>>(matrix, lengths, d, nl_rows, nl_dists, n_nl, prune_radius,
                                                                cand, n_cand, base_row, (u64)min_density_hi, (u64)min_density_lo, (u64 *)out_dev,
                                                                (u64 *)out_pinned,
                                                                within_dev, within_pinned, within_cap, done_ticket,
                                                                done_flag_pinned, seq);
    VK_LAUNCH_CHECK();
    return wait_flag(done_flag_pinned, seq, s, "vk_eval_candidates_lists");
}

// ------------------------------------------------------------------ member selection
__global__ void __launch_bounds__(256)
select_members_kernel(const int32_t *__restrict__ nl_rows, const float *__restrict__ nl_dists, int n_nl,
                      float threshold, const int32_t *__restrict__ orig_ids, uint8_t *kept, int32_t *members) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool hit = i < n_nl && nl_dists[i] <= threshold;
    const unsigned ballot = __ballot_sync(0xffffffffu, hit);
    if (ballot == 0u) return;
    const int lane = threadIdx.x & 31;
    int base = 0;
    if (lane == 0) base = atomicAdd(&members[0], __popc(ballot));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (hit) {
        const int row = nl_rows[i];
        members[1 + base + __popc(ballot & ((1u << lane) - 1u))] = orig_ids[row];
        kept[row] = 0;
    }
}

extern "C" int vk_select_members_sync(const int32_t *nl_rows, const float *nl_dists, int32_t n_nl, float threshold,
                                      const int32_t *orig_ids, uint8_t *kept, int32_t *members,
                                      int32_t *members_host, int32_t capacity_host, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (capacity_host < 2) {
        vk_set_error("vk_select_members_sync: capacity_host must be >= 2");
        return 1;
    }
    VK_CUDA(cudaMemsetAsync(members, 0, sizeof(int32_t), s));
    if (n_nl > 0) {
        const int grid = (n_nl + 255) / 256;
        select_members_kernel<<<grid, 256, 0, s>>>(nl_rows, nl_dists, n_nl, threshold, orig_ids, kept, members);
        VK_LAUNCH_CHECK();
    }
    const int64_t first = (int64_t)n_nl + 1 < capacity_host ? (int64_t)n_nl + 1 : capacity_host;
    VK_CUDA(cudaMemcpyAsync(members_host, members, sizeof(int32_t) * (size_t)first, cudaMemcpyDeviceToHost, s));
    VK_CUDA(cudaStreamSynchronize(s));
    return 0;
}

__global__ void mask_clear_kernel(uint8_t *kept, const int32_t *rows, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) kept[rows[i]] = 0;
}

extern "C" int vk_mask_clear(uint8_t *kept, const int32_t *rows, int32_t n, void *stream) {
    if (n <= 0) return 0;
    mask_clear_kernel<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(kept, rows, n);
    VK_LAUNCH_CHECK();
    return 0;
}

// ------------------------------------------------------------------ stable row compaction
constexpr int CP_TILE = 1024;

// tile_scratch[0] = ticket, [1] = total kept, [2 + t] = kept count of tile t, turned into an
// exclusive prefix by the last block to finish.
__global__ void __launch_bounds__(CP_TILE)
compact_count_kernel(const uint8_t *__restrict__ kept, int64_t n, int32_t *tile_scratch, int n_tiles) {
    __shared__ int s_warp[CP_TILE / 32];
    __shared__ int s_last;
    const int tid = threadIdx.x;
    const int64_t row = (int64_t)blockIdx.x * CP_TILE + tid;
    const bool p = row < n && kept[row];
    const unsigned b = __ballot_sync(0xffffffffu, p);
    if ((tid & 31) == 0) s_warp[tid >> 5] = __popc(b);
    __syncthreads();
    if (tid == 0) {
        int c = 0;
        for (int w = 0; w < CP_TILE / 32; ++w) c += s_warp[w];
        tile_scratch[2 + blockIdx.x] = c;
        __threadfence();
        s_last = (atomicAdd(&tile_scratch[0], 1) == n_tiles - 1);
    }
    __syncthreads();
    if (s_last && tid == 0) {
        __threadfence();
        int run = 0;
        for (int t = 0; t < n_tiles; ++t) {
            const int c = ((volatile int32_t *)tile_scratch)[2 + t];
            tile_scratch[2 + t] = run;
            run += c;
        }
        tile_scratch[1] = run;
        tile_scratch[0] = 0;
    }
}

__global__ void __launch_bounds__(CP_TILE)
compact_scatter_kernel(const float *__restrict__ matrix, const float *__restrict__ lengths,
                       const int32_t *__restrict__ orig_ids, const uint8_t *__restrict__ kept, int64_t n, int d,
                       float *__restrict__ matrix_out, float *__restrict__ lengths_out,
                       int32_t *__restrict__ orig_out, uint8_t *__restrict__ kept_out,
                       const int32_t *__restrict__ tile_scratch) {
    __shared__ int s_warp[CP_TILE / 32];
    __shared__ int s_dest[CP_TILE];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int64_t row0 = (int64_t)blockIdx.x * CP_TILE;
    const int64_t row = row0 + tid;
    const bool p = row < n && kept[row];
    const unsigned b = __ballot_sync(0xffffffffu, p);
    if (lane == 0) s_warp[warp] = __popc(b);
    __syncthreads();
    int off = tile_scratch[2 + blockIdx.x];
    for (int w = 0; w < warp; ++w) off += s_warp[w];
    const int dest = p ? off + __popc(b & ((1u << lane) - 1u)) : -1;
    s_dest[tid] = dest;
    if (p) {
        lengths_out[dest] = lengths[row];
        orig_out[dest] = orig_ids[row];
        kept_out[dest] = 1;
    }
    __syncthreads();
    // rows are copied warp-cooperatively so that both sides stay coalesced
    for (int r = warp; r < CP_TILE; r += CP_TILE / 32) {
        const int dst = s_dest[r];
        if (dst < 0) continue;
        const float *src = matrix + (row0 + r) * (int64_t)d;
        float *out = matrix_out + (int64_t)dst * d;
        for (int k = lane; k < d; k += 32) out[k] = src[k];
    }
}

extern "C" int vk_compact_rows_sync(const float *matrix, const float *lengths, const int32_t *orig_ids,
                                    const uint8_t *kept, int64_t n, int d, float *matrix_out, float *lengths_out,
                                    int32_t *orig_out, uint8_t *kept_out, int32_t *tile_scratch,
                                    int64_t *n_out_host, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (n <= 0) {
        *n_out_host = 0;
        return 0;
    }
    const int n_tiles = (int)((n + CP_TILE - 1) / CP_TILE);
    VK_CUDA(cudaMemsetAsync(tile_scratch, 0, sizeof(int32_t) * 2, s));
    compact_count_kernel<<<n_tiles, CP_TILE, 0, s>>>(kept, n, tile_scratch, n_tiles);
    VK_LAUNCH_CHECK();
    compact_scatter_kernel<<<n_tiles, CP_TILE, 0, s>>>(matrix, lengths, orig_ids, kept, n, d, matrix_out,
                                                       lengths_out, orig_out, kept_out, tile_scratch);
    VK_LAUNCH_CHECK();
    int32_t total = 0;
    VK_CUDA(cudaMemcpyAsync(&total, tile_scratch + 1, sizeof(int32_t), cudaMemcpyDeviceToHost, s));
    VK_CUDA(cudaStreamSynchronize(s));
    *n_out_host = total;
    return 0;
}

#ifdef VK_TIMELINE
// stamps of the probe kernel (slots 0 entry, 1 prologue done, 2 scan done, 3 block sums merged, 4 before the ticket
// [block 0]; 5 last block elected, 6 results written to pinned memory, 7 flag raised [last block])
extern "C" int vk_cluster_timeline_read(unsigned long long *out_host) {
    VK_CUDA(cudaDeviceSynchronize());
    VK_CUDA(cudaMemcpyFromSymbol(out_host, vk_tl, sizeof(unsigned long long) * 4096));
    return 0;
}
#endif

// Stand-alone check of the production wgmma 3xTF32 main loop (tc::ws_mainloop, vk_tc.cuh): C[M, N] = A * B^T on
// staged operands, every tile width and split-K offsets.  Used by tests/test_tc_gpu.py.
#include "vk_tc.cuh"

namespace {

// C[M, N] = A * B^T through the PRODUCTION main loop (tc::ws_mainloop, the one fwd_layer_tc_kernel /
// bwd_layer_tc_kernel run): A in the lane-major layout (zero padded to 128-row panels and whole k-tiles),
// B plain K-major (zero padded to whole tiles), k-tiles [kt0, kt0 + nk) only (split-K slices as in wgrad).
struct WsTestMaps {
    int use_tma, flush;
    VkTmap hi, lo;
};

__global__ void __launch_bounds__(tc::WS_THREADS, 1)
ws_gemm_test_kernel(const float *A, int lda, const float *B, int ldb, float *C, int M, int N, int tile_n, int kt0, int nk,
                    const __grid_constant__ WsTestMaps tm) {
    extern __shared__ uint8_t smem_raw[];
    __shared__ tc::WsShared sh;
    uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    const int m0 = blockIdx.y * 128, n0 = blockIdx.x * tile_n;
    int bn = N - n0;
    bn = bn > tile_n ? tile_n : ((bn + 15) & ~15);
    tc::WsAcc acc;
    if (tm.flush) tc::ws_mainloop<false, true>(A, lda, m0, B, ldb, n0, bn, kt0, nk, smem, &sh, acc);
    else if (tm.use_tma) tc::ws_mainloop<true>(A, lda, m0, B, ldb, n0, bn, kt0, nk, smem, &sh, acc, tile_n, &tm.hi, &tm.lo);
    else tc::ws_mainloop<false>(A, lda, m0, B, ldb, n0, bn, kt0, nk, smem, &sh, acc);
    constexpr int TS = 132;
    float *tile = reinterpret_cast<float *>(smem);
    tc::ws_acc_to_tile(acc, bn, tile, TS);
    tc::ws_tile_end();
    for (int q = threadIdx.x; q < 128 * bn; q += tc::WS_EPI_THREADS) {
        const int r = q / bn, c = q - r * bn;
        if (m0 + r < M && n0 + c < N) C[(int64_t)(m0 + r) * N + n0 + c] = tile[r * TS + c];
    }
}

}  // namespace

// A_lane: [ceil(M / 128) * 128 rows, lda] in tc::lane_major_index order; B: [ceil(N / tile_n) * tile_n rows, ldb]
// row-major; lda, ldb multiples of 32 covering k-tiles [0, kt0 + nk).  tile_n: multiple of 16 in [16, 128].
// B_lo != NULL: B through TMA (B_lo = the tf32 remainders of B, same shape), as the forward / dgrad GEMMs fetch weights.
// flush != 0 (with B_lo == NULL): the wgrad variant -- accumulation chain cut every 4 k-tiles.
extern "C" int vk_tc_gemm_test(const float *A_lane, int lda, const float *B, const float *B_lo, int ldb, float *C, int M, int N,
                               int tile_n, int kt0, int nk, int flush, void *stream) {
    cudaStream_t s = (cudaStream_t)stream;
    if (tile_n < 16 || tile_n > 128 || (tile_n & 15) || (lda & 31) || (ldb & 31)) {
        vk_set_error("vk_tc_gemm_test: bad tile / leading dimensions");
        return 1;
    }
    dim3 grid((N + tile_n - 1) / tile_n, (M + 127) / 128);
    int smem = tc::ws_smem_bytes(tile_n);
    if (smem < 128 * 132 * 4 + 1024) smem = 128 * 132 * 4 + 1024;  // the epilogue tile reuses the operand ring
    VK_CUDA(cudaFuncSetAttribute(ws_gemm_test_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    WsTestMaps tm;
    memset(&tm, 0, sizeof(tm));
    tm.flush = (flush && !B_lo) ? 1 : 0;
    if (B_lo) {
        const int rows = (int)grid.x * tile_n;
        tm.use_tma = 1;
        if (vk_make_tmap_2d(&tm.hi, B, ldb, rows, tile_n) || vk_make_tmap_2d(&tm.lo, B_lo, ldb, rows, tile_n)) return 1;
    }
    ws_gemm_test_kernel<<<grid, tc::WS_THREADS, smem, s>>>(A_lane, lda, B, ldb, C, M, N, tile_n, kt0, nk, tm);
    VK_LAUNCH_CHECK();
    return 0;
}

extern "C" int64_t vk_lane_major_index(int r, int k, int ld) { return (int64_t)tc::lane_major_index(r, k, ld); }

"""GPU suite: the PRODUCTION wgmma 3xTF32 main loop (tc::ws_mainloop in vk_tc.cuh -- the loop inside
fwd_layer_tc_kernel / bwd_layer_tc_kernel: A operand in registers from the lane-major staging layout, B operand
through the shared-memory ring) against an fp64 reference, for every tile width, ragged shapes and split-K offsets.
Near-fp32 accuracy is the contract: the relative error of the result matrix stays below 1e-6 + 1.2e-8 * K (plain TF32
would sit at ~5e-4 for every K)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

# M, N, K, tile_n
SHAPES = [(128, 128, 32, 128), (128, 128, 64, 64), (256, 512, 512, 16), (256, 512, 512, 32), (4096, 512, 512, 128),
          (300, 154, 154, 32), (77, 48, 70, 48), (512, 513, 1024, 32), (154, 512, 256, 64), (256, 32, 512, 16),
          (200, 512, 32, 32), (1000, 155, 512, 96), (8192, 512, 154, 128)]


def lane_major(a: torch.Tensor, ld: int) -> torch.Tensor:
    """[rows (multiple of 128), ld] row-major -> the lane-major staging layout (vk_tc.cuh: tc::lane_major_index)."""
    rows = a.shape[0]
    r = torch.arange(rows, device=a.device).view(-1, 1)
    k = torch.arange(ld, device=a.device).view(1, -1)
    idx = (r >> 7) * 128 * ld + (k >> 5) * 4096 + ((k & 31) >> 2) * 512 + (r & 127) * 4 + (k & 3)
    out = torch.empty(rows * ld, device=a.device, dtype=a.dtype)
    out[idx.reshape(-1)] = a.reshape(-1)
    return out


def run(A, B, tile_n, kt0=0, nk=None, tma=False, flush=False):
    from vamb_b200 import _lib

    _lib.require_device()
    M, K = A.shape
    N = B.shape[0]
    ld = (K + 31) // 32 * 32
    Mp, Np = (M + 127) // 128 * 128, (N + tile_n - 1) // tile_n * tile_n
    Ap = torch.zeros(Mp, ld, device="cuda")
    Ap[:M, :K] = A
    Bp = torch.zeros(Np, ld, device="cuda")
    Bp[:N, :K] = B
    Al = lane_major(Ap, ld)
    C = torch.full((M, N), float("nan"), device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    nk = ld // 32 - kt0 if nk is None else nk
    b_lo = None
    if tma:  # the tf32 remainder the tensor core does not see: x - (x with the low 13 mantissa bits cleared)
        b_lo = Bp - (Bp.view(torch.int32) & -8192).view(torch.float32)
    _lib.check(_lib.lib.vk_tc_gemm_test(Al.data_ptr(), ld, Bp.data_ptr(), b_lo.data_ptr() if tma else None, ld, C.data_ptr(),
                                        M, N, tile_n, kt0, nk, 1 if flush else 0, s))
    torch.cuda.synchronize()
    return C


@pytest.mark.parametrize("tma", [False, True], ids=["cp.async-B", "tma-B"])
@pytest.mark.parametrize("M,N,K,tile_n", SHAPES)
def test_ws_mainloop_matches_fp64(M, N, K, tile_n, tma):
    g = torch.Generator(device="cuda").manual_seed(M * 7 + N * 3 + K)
    A = torch.randn(M, K, device="cuda", generator=g)
    B = torch.randn(N, K, device="cuda", generator=g)
    C = run(A, B, tile_n, tma=tma)
    ref = A.double() @ B.double().t()
    assert torch.isfinite(C).all()
    err = float((C.double() - ref).norm() / ref.norm())
    assert err < 1e-6 + 1.2e-8 * K, err


@pytest.mark.parametrize("kt0,nk", [(0, 4), (4, 4), (12, 4), (3, 1), (0, 0), (2, 13)])
def test_ws_mainloop_split_k_slices(kt0, nk):
    """k-tile ranges as the wgrad split-K slices use them (an empty slice yields zeros)."""
    g = torch.Generator(device="cuda").manual_seed(kt0 * 31 + nk)
    M, N, K = 384, 100, 512
    A = torch.randn(M, K, device="cuda", generator=g)
    B = torch.randn(N, K, device="cuda", generator=g)
    C = run(A, B, 32, kt0, nk)
    sl = slice(kt0 * 32, (kt0 + nk) * 32)
    ref = A[:, sl].double() @ B[:, sl].double().t()
    if nk == 0:
        assert float(C.abs().max()) == 0.0
    else:
        assert float((C.double() - ref).norm() / ref.norm()) < 1e-6 + 1.2e-8 * 32 * nk


def test_lane_major_helper_matches_the_c_abi():
    from vamb_b200 import _lib

    for r, k, ld in [(0, 0, 32), (5, 7, 64), (127, 31, 32), (128, 0, 96), (300, 95, 96), (8191, 511, 512)]:
        a = torch.zeros((r // 128 + 1) * 128, ld)
        a[r, k] = 1.0
        assert int(lane_major(a, ld).argmax()) == int(_lib.lib.vk_lane_major_index(r, k, ld))


@pytest.mark.parametrize("M,N,K,tile_n", [(512, 513, 512, 32), (154, 512, 4096, 64), (300, 100, 1000, 128), (128, 64, 96, 16),
                                          (128, 48, 160, 48), (256, 128, 8192, 128)])
def test_ws_mainloop_flush_variant_matches_fp64(M, N, K, tile_n):
    """The wgrad variant: the tensor-core accumulation chain cut every 4 k-tiles and summed into fp32 registers.  The
    error no longer grows with the chain length: below 1e-6 + 1.2e-8 * 128 for every K, and not above the plain loop."""
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = torch.randn(M, K, device="cuda", generator=g)
    B = torch.randn(N, K, device="cuda", generator=g)
    ref = A.double() @ B.double().t()
    err_f = float((run(A, B, tile_n, flush=True).double() - ref).norm() / ref.norm())
    err_p = float((run(A, B, tile_n).double() - ref).norm() / ref.norm())
    assert err_f < 1e-6 + 1.2e-8 * 128 + 2e-8 * (K // 128), (err_f, err_p)
    assert err_f <= err_p * 1.05 + 3e-7

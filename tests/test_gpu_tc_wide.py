"""Tensor-core layer kernel at the widths where its column tiling changes: 2-plane layers wider than 128 columns run one
128 x 256 tile per row block, 3-plane layers and narrower 2-plane layers 128 x 128 tiles.  The output has a row stride
of N + 8 and two rows past M, all pre-filled with NaN: every element outside [M, N] must stay NaN (weight rows past the
image tile, N = 217 -> 224 and N = 257 -> 272, never reach the output)."""
import pytest
import torch

from tests.gpu_util import err_inf, scale_inf

pytestmark = pytest.mark.gpu
DEV = "cuda"
K = 256
BOUND = {2: 5e-5, 3: 2e-6}          # the bounds of test_gpu_tc.py::test_dense_forward_tc_vs_fp64


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _lib():
    from neuraludf_b200 import _lib as L
    return L, L.lib()


@pytest.mark.parametrize("N", [256, 217, 257, 128])
@pytest.mark.parametrize("M", [65536, 1000, 77])
def test_dense_forward_tc_tiles(M, N):
    L, lib = _lib()
    g = torch.Generator().manual_seed(7 * M + N)
    X = torch.randn(M, K, generator=g, dtype=torch.float64).to(DEV)
    W = (torch.randn(N, K, generator=g, dtype=torch.float64) / K ** 0.5).to(DEV)
    b = torch.randn(N, generator=g, dtype=torch.float64).to(DEV)
    ref = X @ W.t() + b
    Xd, bd = X.float().contiguous(), b.float().contiguous()
    ldy = N + 8
    for transposed in (0, 1):
        # transposed == 1: the image of the [K, N] matrix W^T, read as B(n, k) = W^T[k, n]
        Wd = (W.t() if transposed else W).float().contiguous()
        for planes in (2, 3):
            img = torch.zeros(lib.nudf_tc_image_elems(N, K, planes), dtype=torch.int16, device=DEV)
            L.check(lib.nudf_tc_prepare_weights(L.ptr(Wd), Wd.stride(0), N, K, transposed, planes, L.ptr(img), L.stream_ptr()),
                    "prep")
            Y = torch.full((M + 2, ldy), float("nan"), device=DEV)
            L.check(lib.nudf_dense_forward_tc(L.ptr(Xd), K, L.ptr(img), planes, L.ptr(bd), L.ptr(Y), ldy, M, N, K, 0,
                                              L.stream_ptr()), "dense_tc")
            torch.cuda.synchronize()
            tag = (M, N, transposed, planes)
            outside = torch.ones_like(Y, dtype=torch.bool)
            outside[:M, :N] = False
            assert torch.isnan(Y[outside]).all(), ("write outside [M, N]", tag)
            inside = Y[:M, :N]
            assert torch.isfinite(inside).all(), ("non-finite output", tag)
            e = err_inf(inside, ref) / scale_inf(ref)
            assert e < BOUND[planes], (e, tag)

"""GPU tests of the 2-plane tensor-core layer kernel (nudf_dense_forward_tc, planes = 2) on operands on and off
alignment.  The kernel reads activations through a 2-D tensor map (a row stride that is a multiple of 4 floats and a
16-byte-aligned base); nudf_dense_forward_tc copies any other operand into an aligned temporary first.  The kernel never
reads the padding columns, so an operand off alignment must give the bits of the aligned one; each is also checked
against fp64."""
import pytest
import torch

from tests.gpu_util import err_inf, report, scale_inf

pytestmark = pytest.mark.gpu
DEV = "cuda"

SHAPES = [(256, 256), (256, 39), (217, 256), (256, 217), (128, 128), (128, 259)]   # (N, K)
BOUND = 5e-5                        # the 2-plane bound of test_gpu_tc.py::test_dense_forward_tc_vs_fp64


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _ld4(n):
    return (n + 3) // 4 * 4


def _operand(P, width, ld, offset, g):
    """[P, width] view with row stride ld, starting `offset` floats into its buffer; the columns from width to ld are NaN"""
    buf = torch.full((P * ld + offset,), float("nan"), device=DEV)
    x = buf[offset:].view(P, ld)
    x[:, :width] = torch.randn(P, width, generator=g, device=DEV)
    return x


def _layer(X, img, b, N, K, P):
    from neuraludf_b200 import _lib as L
    lib = L.lib()
    Y = torch.full((P, N), float("nan"), device=DEV)
    L.check(lib.nudf_dense_forward_tc(L.ptr(X), X.stride(0), L.ptr(img), 2, L.ptr(b), L.ptr(Y), N, P, N, K, 0,
                                      L.stream_ptr()), "dense_forward_tc")
    torch.cuda.synchronize()
    return Y


def _image(W, N, K, transposed):
    from neuraludf_b200 import _lib as L
    lib = L.lib()
    img = torch.zeros(lib.nudf_tc_image_elems(N, K, 2), dtype=torch.int16, device=DEV)
    L.check(lib.nudf_tc_prepare_weights(L.ptr(W), W.stride(0), N, K, transposed, 2, L.ptr(img), L.stream_ptr()), "prep")
    return img


@pytest.mark.parametrize("transposed", [0, 1])
@pytest.mark.parametrize("N,K", SHAPES)
@pytest.mark.parametrize("P", [65499, 1000, 40])
def test_layer_offset_operand_matches_aligned(P, N, K, transposed):
    """The row stride rounded up to 4 floats with NaN in the padding columns: the kernel's tensor map must stop at K (a
    ragged last K slice arrives zero-filled) and at P (a ragged last row block).  The same values one float into a
    buffer are repacked, and the two results must be the same bits.  P = 40 is one partial row block."""
    g = torch.Generator(device=DEV).manual_seed(P * 7 + N * 3 + K + transposed)
    W = torch.randn(N, K, generator=g, device=DEV) / K ** 0.5
    b = torch.randn(N, generator=g, device=DEV)
    # transposed == 1: the image of the [K, N] matrix W^T, read as B(n, k) = W^T[k, n]
    img = _image(W.t().contiguous() if transposed else W, N, K, transposed)
    X = _operand(P, K, _ld4(K), 0, g)
    X1 = _operand(P, K, _ld4(K), 1, g)
    X1[:, :K] = X[:, :K]
    aligned = _layer(X, img, b, N, K, P)
    offset = _layer(X1, img, b, N, K, P)
    assert torch.isfinite(aligned).all()
    assert torch.equal(aligned, offset)
    assert torch.equal(aligned, _layer(X, img, b, N, K, P))
    ref = X[:, :K].double() @ W.double().t() + b.double()
    tag = "layer[%d,%d,%d,t%d]" % (P, N, K, transposed)
    for name, Y in (("aligned", aligned), ("offset", offset)):
        e = err_inf(Y, ref) / scale_inf(ref)
        report("%s.%s" % (tag, name), rel=e)
        assert e < BOUND, (name, e)


@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("N", [256, 128])
def test_layer_k0_gives_bias(N, offset):
    """K = 0: no copy and no product, the epilogue on zero accumulators gives the bias on every row, for an operand on
    or off alignment."""
    P = 1000
    g = torch.Generator(device=DEV).manual_seed(N + offset)
    b = torch.randn(N, generator=g, device=DEV)
    img = torch.zeros(8, dtype=torch.int16, device=DEV)     # the image of a K = 0 layer is empty and never read
    Y = _layer(_operand(P, 0, 4, offset, g), img, b, N, 0, P)
    assert torch.equal(Y, b.expand(P, N))

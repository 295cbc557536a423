"""GPU tests of the two activation paths of the 3-plane tensor-core layer (nudf_dense_forward_tc, planes = 3).  A row
stride that is a multiple of 4 floats with a 16-byte-aligned base takes the persistent TMA-fed kernel (producer
warpgroup splitting 2-D TMA boxes into planes, two consumer warpgroups, epilogue from registers); any other operand
takes the register-staged kernel.  Both split the same bf16 planes, issue the same products and add them in the same
order, so they must give the same bits: the meshing paths rely on a point getting the same bits in any batch, and a
batch offset can change an operand's alignment.  Each is also checked against fp64."""
import pytest
import torch

from tests.gpu_util import err_inf, report, scale_inf

pytestmark = pytest.mark.gpu
DEV = "cuda"

SHAPES = [(256, 256), (256, 39), (217, 256), (256, 217), (128, 128), (128, 259)]   # (N, K)
# 38 417 points are 301 row blocks: 301 or 602 tiles, not a multiple of the persistent grid (one CTA per SM), so some
# CTAs run three or more tiles and others fewer; 65 499 ends in a partial row block; 40 is one partial row block
POINTS = [65499, 38417, 1000, 40]
ACT_NONE, ACT_SOFTPLUS100 = 0, 2
BOUND = 5e-5                        # the bound of test_gpu_tc.py::test_dense_forward_tc_vs_fp64


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


def _layer(X, img, b, N, K, P, act):
    from neuraludf_b200 import _lib as L
    lib = L.lib()
    Y = torch.full((P, N), float("nan"), device=DEV)
    L.check(lib.nudf_dense_forward_tc(L.ptr(X), X.stride(0), L.ptr(img), 3, L.ptr(b), L.ptr(Y), N, P, N, K, act,
                                      L.stream_ptr()), "dense_forward_tc")
    torch.cuda.synchronize()
    return Y


def _image(W, N, K, transposed):
    from neuraludf_b200 import _lib as L
    lib = L.lib()
    img = torch.zeros(lib.nudf_tc_image_elems(N, K, 3), dtype=torch.int16, device=DEV)
    L.check(lib.nudf_tc_prepare_weights(L.ptr(W), W.stride(0), N, K, transposed, 3, L.ptr(img), L.stream_ptr()), "prep")
    return img


@pytest.mark.parametrize("act", [ACT_NONE, ACT_SOFTPLUS100])
@pytest.mark.parametrize("transposed", [0, 1])
@pytest.mark.parametrize("N,K", SHAPES)
@pytest.mark.parametrize("P", POINTS)
def test_layer3_tma_matches_register_path(P, N, K, transposed, act):
    """The row stride rounded up to 4 floats with NaN in the padding columns: the TMA path, whose tensor map must stop
    at K (a ragged last K slice arrives zero-filled) and at P (a ragged last row block, landing quarters past P split as
    zeros).  The same values one float into a buffer take the register path, and the two results must be the same
    bits, on every call."""
    g = torch.Generator(device=DEV).manual_seed(P * 7 + N * 3 + K + transposed + 11 * act)
    W = torch.randn(N, K, generator=g, device=DEV) / K ** 0.5
    b = torch.randn(N, generator=g, device=DEV)
    # transposed == 1: the image of the [K, N] matrix W^T, read as B(n, k) = W^T[k, n]
    img = _image(W.t().contiguous() if transposed else W, N, K, transposed)
    X = _operand(P, K, _ld4(K), 0, g)
    X1 = _operand(P, K, _ld4(K), 1, g)
    X1[:, :K] = X[:, :K]
    tma = _layer(X, img, b, N, K, P, act)
    regs = _layer(X1, img, b, N, K, P, act)
    assert torch.isfinite(tma).all()
    assert torch.equal(tma, regs)
    assert torch.equal(tma, _layer(X, img, b, N, K, P, act))
    ref = X[:, :K].double() @ W.double().t() + b.double()
    if act == ACT_SOFTPLUS100:
        ref = torch.nn.functional.softplus(ref, beta=100.0)
    tag = "layer3[%d,%d,%d,t%d,a%d]" % (P, N, K, transposed, act)
    for name, Y in (("tma", tma), ("regs", regs)):
        e = err_inf(Y, ref) / scale_inf(ref)
        report("%s.%s" % (tag, name), rel=e)
        assert e < BOUND, (name, e)

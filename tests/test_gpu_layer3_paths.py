"""GPU tests of the 3-plane tensor-core layer (nudf_dense_forward_tc, planes = 3) on operands on and off alignment.  The
persistent kernel (a producer warpgroup splitting 2-D TMA boxes into planes, two consumer warpgroups, epilogue from
registers) reads activations through a tensor map (a row stride that is a multiple of 4 floats and a 16-byte-aligned
base); nudf_dense_forward_tc copies any other operand into an aligned temporary first.  The padding columns are never
read, so an operand off alignment must give the bits of the aligned one: the meshing paths rely on a point getting the
same bits in any batch, and a batch offset can change an operand's alignment.  Each is also checked against fp64."""
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
BOUND = 2e-6                        # the 3-plane bound of test_gpu_tc.py::test_dense_forward_tc_vs_fp64 and test_gpu_tc_wide.py


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
def test_layer3_offset_operand_matches_aligned(P, N, K, transposed, act):
    """The row stride rounded up to 4 floats with NaN in the padding columns: the kernel's tensor map must stop at K (a
    ragged last K slice arrives zero-filled) and at P (a ragged last row block, landing quarters past P split as zeros).
    The same values one float into a buffer are repacked, and the two results must be the same bits, on every call."""
    g = torch.Generator(device=DEV).manual_seed(P * 7 + N * 3 + K + transposed + 11 * act)
    W = torch.randn(N, K, generator=g, device=DEV) / K ** 0.5
    b = torch.randn(N, generator=g, device=DEV)
    # transposed == 1: the image of the [K, N] matrix W^T, read as B(n, k) = W^T[k, n]
    img = _image(W.t().contiguous() if transposed else W, N, K, transposed)
    X = _operand(P, K, _ld4(K), 0, g)
    X1 = _operand(P, K, _ld4(K), 1, g)
    X1[:, :K] = X[:, :K]
    aligned = _layer(X, img, b, N, K, P, act)
    offset = _layer(X1, img, b, N, K, P, act)
    assert torch.isfinite(aligned).all()
    assert torch.equal(aligned, offset)
    assert torch.equal(aligned, _layer(X, img, b, N, K, P, act))
    ref = X[:, :K].double() @ W.double().t() + b.double()
    if act == ACT_SOFTPLUS100:
        ref = torch.nn.functional.softplus(ref, beta=100.0)
    tag = "layer3[%d,%d,%d,t%d,a%d]" % (P, N, K, transposed, act)
    for name, Y in (("aligned", aligned), ("offset", offset)):
        e = err_inf(Y, ref) / scale_inf(ref)
        report("%s.%s" % (tag, name), rel=e)
        assert e < BOUND, (name, e)


@pytest.mark.parametrize("act", [ACT_NONE, ACT_SOFTPLUS100])
@pytest.mark.parametrize("offset", [0, 1])
@pytest.mark.parametrize("N", [256, 128])
def test_layer3_k0_gives_act_bias(N, offset, act):
    """K = 0: no copy and no product, the epilogue on zero accumulators gives act(bias) on every row, for an operand on
    or off alignment."""
    P = 1000
    g = torch.Generator(device=DEV).manual_seed(N + offset + 11 * act)
    b = torch.randn(N, generator=g, device=DEV)
    img = torch.zeros(8, dtype=torch.int16, device=DEV)     # the image of a K = 0 layer is empty and never read
    Y = _layer(_operand(P, 0, 4, offset, g), img, b, N, 0, P, act)
    assert torch.equal(Y, Y[:1].expand(P, N))
    if act == ACT_NONE:
        assert torch.equal(Y[0], b)
    else:
        ref = torch.nn.functional.softplus(b.double(), beta=100.0)
        assert (Y[0].double() - ref).abs().max().item() < 1e-6

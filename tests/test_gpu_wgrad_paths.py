"""GPU tests of the tensor-core weight-gradient contraction (nudf_wgrad, engine 1) on operands on and off alignment.
The kernel reads both operands through 2-D tensor maps (row strides that are a multiple of 4 floats and 16-byte-aligned
bases; an fp32 ring split into MN-major planes); nudf_wgrad copies any other operand into an aligned temporary first.
The padding columns are never read, so operands off alignment must give the bits of aligned ones; each is also checked
against fp64."""
import pytest
import torch

from tests.gpu_util import err_inf, report, scale_inf

pytestmark = pytest.mark.gpu
DEV = "cuda"

SHAPES = [(256, 256), (256, 39), (217, 256), (128, 128), (128, 158), (128, 259)]


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


def _wgrad(dZ, X, n_out, n_in, P):
    from neuraludf_b200 import _lib as L
    lib = L.lib()
    dW = torch.zeros(n_out, n_in, device=DEV)
    L.check(lib.nudf_wgrad(L.ptr(dZ), dZ.stride(0), L.ptr(X), X.stride(0), n_out, n_in, P, L.ptr(dW), n_in, 1,
                           L.stream_ptr()), "wgrad")
    torch.cuda.synchronize()
    return dW


def _vs_fp64(dW, dZ, X, n_out, n_in, tag, P):
    ref = dZ[:, :n_out].double().t() @ X[:, :n_in].double()
    e = err_inf(dW, ref) / scale_inf(ref)
    report("wgrad.%s[%d,%d,%d]" % (tag, P, n_out, n_in), rel=e)
    assert e < 5e-5, e


@pytest.mark.parametrize("n_out,n_in", SHAPES)
@pytest.mark.parametrize("P", [65499, 1000, 40])
def test_wgrad_offset_operands_match_aligned(P, n_out, n_in):
    """Strides rounded up to 4 floats with NaN in the padding columns: the kernel's tensor maps must stop at the width
    (a ragged last column tile arrives zero-filled).  The same values one float into a buffer are repacked, and the two
    results must be the same bits.  P = 40 is a single split of one full and one 8-point slice."""
    g = torch.Generator(device=DEV).manual_seed(P * 5 + n_out + n_in)
    ldz, ldx = _ld4(n_out), _ld4(n_in)
    dZ = _operand(P, n_out, ldz, 0, g)
    X = _operand(P, n_in, ldx, 0, g)
    dZ1 = _operand(P, n_out, ldz, 1, g)
    X1 = _operand(P, n_in, ldx, 1, g)
    dZ1[:, :n_out] = dZ[:, :n_out]
    X1[:, :n_in] = X[:, :n_in]
    aligned = _wgrad(dZ, X, n_out, n_in, P)
    offset = _wgrad(dZ1, X1, n_out, n_in, P)
    assert torch.isfinite(aligned).all()
    assert torch.equal(aligned, offset)
    assert torch.equal(aligned, _wgrad(dZ, X, n_out, n_in, P))
    _vs_fp64(aligned, dZ, X, n_out, n_in, "aligned", P)


@pytest.mark.parametrize("P", [65499, 40])
@pytest.mark.parametrize("misaligned", ["dZ", "X"])
def test_wgrad_misaligned_base_vs_fp64(P, misaligned):
    """Row strides a multiple of 4, but one base pointer one float past a 16-byte boundary: that operand is repacked."""
    n_out, n_in = 256, 256
    g = torch.Generator(device=DEV).manual_seed(P + (misaligned == "X"))
    dZ = _operand(P, n_out, n_out, 1 if misaligned == "dZ" else 0, g)
    X = _operand(P, n_in, n_in, 1 if misaligned == "X" else 0, g)
    _vs_fp64(_wgrad(dZ, X, n_out, n_in, P), dZ, X, n_out, n_in, "misaligned_" + misaligned, P)

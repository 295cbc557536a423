"""GPU tests of the tensor-core weight-gradient contraction (nudf_wgrad, engine 1: gemm_tn_kernel with its split over the
points) at the shapes of the C2 step and at ragged point counts: against fp64, bitwise reproducible, and writing nothing
outside the [n_out, n_in] block of dW."""
import pytest
import torch

from tests.gpu_util import err_inf, report, scale_inf

pytestmark = pytest.mark.gpu
DEV = "cuda"

# (n_out, n_in): UDF hidden layers, UDF layer 0 (39 positional-encoding inputs), the layer before the skip (217 outputs),
# the colour hidden layers and the first layers of the colour network's main (158 inputs) and base (259 inputs) stacks
SHAPES = [(256, 256), (256, 39), (217, 256), (128, 128), (128, 158), (128, 259)]
POINTS = [65536, 65499, 1000, 77]
SENTINEL = 7.0


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _wgrad(dZ, X, n_out, n_in, P, ldw):
    """dW [n_out, ldw] with the columns beyond n_in set to SENTINEL, += dZ^T X on the tensor cores"""
    from neuraludf_b200 import _lib as L
    lib = L.lib()
    dW = torch.zeros(n_out, ldw, device=DEV)
    dW[:, n_in:] = SENTINEL
    L.check(lib.nudf_wgrad(L.ptr(dZ), dZ.stride(0), L.ptr(X), X.stride(0), n_out, n_in, P, L.ptr(dW), ldw, 1,
                           L.stream_ptr()), "wgrad")
    torch.cuda.synchronize()
    return dW


def _check(P, n_out, n_in, ldz, ldx, tag):
    g = torch.Generator(device=DEV).manual_seed(P * 7 + n_out * 3 + n_in + ldz + ldx)
    dZ = torch.randn(P, ldz, generator=g, device=DEV)
    X = torch.randn(P, ldx, generator=g, device=DEV)
    ref = dZ[:, :n_out].double().t() @ X[:, :n_in].double()
    ldw = n_in + 3
    runs = [_wgrad(dZ, X, n_out, n_in, P, ldw) for _ in range(2)]
    assert torch.equal(runs[0], runs[1])                      # fixed-order split-K sum: the same bits on every run
    assert bool((runs[0][:, n_in:] == SENTINEL).all())        # nothing written beyond n_in
    e = err_inf(runs[0][:, :n_in], ref) / scale_inf(ref)
    report("wgrad.%s[%d,%d,%d]" % (tag, P, n_out, n_in), rel=e)
    assert e < 5e-5, e


@pytest.mark.parametrize("n_out,n_in", SHAPES)
@pytest.mark.parametrize("P", POINTS)
def test_wgrad_vs_fp64(P, n_out, n_in):
    """Dense row-major operands (row stride = width): the float4 staging path wherever the width allows it."""
    _check(P, n_out, n_in, n_out, n_in, "dense")


@pytest.mark.parametrize("n_out,n_in", SHAPES)
@pytest.mark.parametrize("P", [65499, 77])
def test_wgrad_strided_vs_fp64(P, n_out, n_in):
    """Row strides above the width and not a multiple of 4: every operand load takes the scalar path."""
    _check(P, n_out, n_in, n_out + 5, n_in + 3, "strided")


def _param_grads(engine, mask, run):
    from neuraludf_b200 import _lib as L
    lib = L.lib()
    old_engine, old_mask = lib.nudf_get_engine(), lib.nudf_get_tc_mask()
    lib.nudf_set_engine(engine)
    lib.nudf_set_tc_mask(mask)
    try:
        return run()
    finally:
        lib.nudf_set_engine(old_engine)
        lib.nudf_set_tc_mask(old_mask)


@pytest.mark.parametrize("P", [65499, 1000])
def test_fused_bias_gradients_match_ffma(P):
    """The bias gradients that gemm_tn_kernel sums from its staged activations (the backward layers of the UDF and colour
    networks), against the separate column-sum kernel of the FFMA path.  Only the weight gradients run on the tensor
    cores (chain mask TC_WGRAD); every other contraction is the same FFMA kernel in both runs, so both sum the same
    upstream gradients and differ only in the order of the fp32 additions."""
    from neuraludf_b200 import synthetic as S
    from neuraludf_b200.models import fields as F
    dev = torch.device(DEV)
    udf = F.UDFNetwork(d_in=3, d_out=257, d_hidden=256, n_layers=8, skip_in=(4,), multires=6, bias=0.5, scale=1.0,
                       geometric_init=True, weight_norm=True, udf_type="abs")
    udf.load_state_dict(S.make_udf_params(S.udf_cfg(), 0))
    col = F.ResidualRenderingNetwork(d_feature=256, mode="no_normal", d_in=6, d_out=3, d_hidden=128, n_layers=4,
                                     weight_norm=True, multires_view=4, squeeze_out=True, blending_cand_views=10)
    col.load_state_dict(S.make_color_params(S.color_cfg(), 1))
    udf, col = udf.to(dev), col.to(dev)
    g = torch.Generator(device=DEV).manual_seed(P)
    x = torch.rand(P, 3, generator=g, device=DEV) - 0.5
    r_out = torch.randn(P, 257, generator=g, device=DEV)
    r_grad = torch.randn(P, 3, generator=g, device=DEV)
    dirs = torch.nn.functional.normalize(torch.randn(P, 3, generator=g, device=DEV), dim=1)
    feat = torch.randn(P, 256, generator=g, device=DEV)

    def run():
        for p in list(udf.parameters()) + list(col.parameters()):
            p.grad = None
        out, grad = udf.value_and_gradient(x)
        loss = (out * r_out).sum() + (grad * r_grad).sum()
        gc = torch.Generator(device=DEV).manual_seed(P + 1)    # the same colour-output weights in every run
        loss = loss + sum((y * torch.randn(y.shape, generator=gc, device=DEV)).sum() for y in col(x, None, dirs, feat))
        loss.backward()
        torch.cuda.synchronize()
        return {"%s.%s" % (mn, k): p.grad.clone() for mn, m in (("udf", udf), ("color", col))
                for k, p in m.named_parameters() if k.endswith("bias")}

    tc = _param_grads(1, 16, run)
    ffma = _param_grads(0, 0, run)
    assert len(tc) >= 8
    worst = 0.0
    for k, ref in ffma.items():
        assert torch.isfinite(tc[k]).all(), k
        e = err_inf(tc[k], ref) / scale_inf(ref)
        worst = max(worst, e)
        assert e < 1e-4, (k, e)
    report("wgrad.fused_bias[%d]" % P, rel_worst=worst)

"""Pins oracle/oracle_torch.py at the shapes of the configuration sweep (tests/test_gpu_net_shapes.py) against outputs of
the UNMODIFIED reference's networks (tests/golden/net_shapes.*.npz, written by oracle/make_golden_shapes.py).

Same tolerances as tests/test_oracle_pinned.py: the fp64 oracle agrees with the fp64 reference run to round-off and the fp32
oracle with the fp32 run to fp32 noise.  Outputs and the gradients with respect to every input are compared."""
import pytest
import torch

from oracle import oracle_torch as O
from tests.golden_util import Fixtures, rel_err
from tests.test_gpu_net_shapes import COLOR_CFGS, NERF_CFGS, UDF_CFGS, _color_params, _nerf_params, _udf_params

TOL = {torch.float64: 1e-8, torch.float32: 2e-5}
TAGS = [(torch.float32, "f32"), (torch.float64, "f64")]


@pytest.fixture(scope="module")
def fx():
    return Fixtures("net_shapes")


def _t(fx, key, dtype, grad=False):
    return torch.from_numpy(fx[key]).to(dtype).requires_grad_(grad)


def _pin(fx, name, got, tag, dtype):
    for k, t in got.items():
        t = t.detach()
        ref = torch.from_numpy(fx["%s_%s_%s" % (name, k, tag)])
        assert t.shape == ref.shape, (name, k, tuple(t.shape), tuple(ref.shape))
        if t.numel():
            assert rel_err(t, ref) < TOL[dtype], (name, k, rel_err(t, ref))


@pytest.mark.parametrize("dtype,tag", TAGS)
@pytest.mark.parametrize("name", list(UDF_CFGS))
def test_udf_shapes(fx, name, dtype, tag):
    cfg, p = _udf_params(name)
    p = O.to_dtype(p, dtype)
    x = _t(fx, name + "_x", dtype)
    _pin(fx, name, {"out": O.udf_mlp(p, cfg, x), "grad": O.udf_gradient_autograd(p, cfg, x, create_graph=False)}, tag, dtype)


@pytest.mark.parametrize("dtype,tag", TAGS)
@pytest.mark.parametrize("name", list(COLOR_CFGS))
def test_color_shapes(fx, name, dtype, tag):
    cc, p = _color_params(name)
    pts, dirs, feat = (_t(fx, "%s_%s" % (name, k), dtype, True) for k in ("pts", "dirs", "feat"))
    bars = [_t(fx, "%s_%s" % (name, k), dtype) for k in ("bar_cb", "bar_c", "bar_bl")]
    out = O.color_mlp(O.to_dtype(p, dtype), cc, pts, dirs, feat)
    got = dict(zip(("base", "color"), out[:2]))
    if cc["blending_cand_views"] > 0:          # without views the reference returns (color_base, color) only
        got["blend"] = out[2]
    loss = sum((t * b).sum() for t, b in zip(out, bars))
    got.update(zip(("dpts", "ddirs", "dfeat"), torch.autograd.grad(loss, [pts, dirs, feat])))
    _pin(fx, name, got, tag, dtype)


@pytest.mark.parametrize("dtype,tag", TAGS)
@pytest.mark.parametrize("name", list(NERF_CFGS))
def test_nerf_shapes(fx, name, dtype, tag):
    nc, p = _nerf_params(name)
    pts, dirs = (_t(fx, "%s_%s" % (name, k), dtype, True) for k in ("pts", "dirs"))
    alpha, rgb = O.nerf_mlp(O.to_dtype(p, dtype), nc, pts, dirs)
    loss = (alpha * _t(fx, name + "_bar_alpha", dtype)).sum() + (rgb * _t(fx, name + "_bar_rgb", dtype)).sum()
    got = {"alpha": alpha, "rgb": rgb}
    got.update(zip(("dpts", "ddirs"), torch.autograd.grad(loss, [pts, dirs])))
    _pin(fx, name, got, tag, dtype)


def test_fixture_covers_the_sweep(fx):
    for name in list(UDF_CFGS) + list(COLOR_CFGS) + list(NERF_CFGS):
        assert any(k.startswith(name + "_") and k.endswith("_f64") for k in fx.files), name

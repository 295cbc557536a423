"""Generate golden fixtures of the networks at the shapes of the configuration sweep (dev container only).

    python oracle/make_golden_shapes.py     # writes tests/golden/net_shapes.NN.npz

tests/test_gpu_net_shapes.py judges the CUDA networks against the oracle (oracle/oracle_torch.py) at shapes no shipped conf
uses: UDF networks with scale != 1, multires 0 or 16, no skip or a skip on the first or last layer, 2..16 layers; colour networks
of 3..16 layers per stack with 0..29 blending views; NeRF++ networks of 2..16 layers with and without a skip.  This script
runs the UNMODIFIED reference's UDFNetwork, ResidualRenderingNetwork and NeRF (imported through oracle/refshim.py) at each of
those configurations, with the same seeded parameters, in fp32 and fp64, on a few dozen points, and stores the outputs and
the gradients with respect to the inputs.  tests/test_oracle_shapes_pinned.py pins the oracle to them, so the arbiter of the
sweep is pinned at the shapes it judges.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle_torch as O  # noqa: E402
from oracle import refshim  # noqa: E402
from tests.golden_util import save_fixtures  # noqa: E402
from tests.test_gpu_net_shapes import (COLOR_CFGS, NERF_CFGS, UDF_CFGS, _color_params, _nerf_params,  # noqa: E402
                                       _udf_params)

NAME = "net_shapes"
N_POINTS = 48


def np_(t):
    return t.detach().cpu().numpy()


def inputs(kind, name, cfg):
    """the seeded float32 inputs of one configuration: UDF (x,), colour (pts, dirs, feat, bars), NeRF++ (pts, dirs, bars)"""
    gen = torch.Generator().manual_seed(sum(map(ord, name)) + 1000 * "ucn".index(kind))
    f = lambda *shape: torch.randn(*shape, generator=gen, dtype=torch.float64)
    unit = lambda t: t / t.norm(dim=1, keepdim=True)
    if kind == "u":
        return ((torch.rand(N_POINTS, 3, generator=gen, dtype=torch.float64) * 2 - 1) * 0.9,)
    if kind == "c":
        pts = torch.rand(N_POINTS, 3, generator=gen, dtype=torch.float64) * 2 - 1
        return (pts, unit(f(N_POINTS, 3)), 0.3 * f(N_POINTS, cfg["d_feature"]), f(N_POINTS, cfg["d_out"]),
                f(N_POINTS, cfg["d_out"]), f(N_POINTS, cfg["blending_cand_views"]))
    pts = f(N_POINTS, 4)
    pts = (pts / pts[:, :3].norm(dim=1, keepdim=True))[:, :cfg["d_in"]]
    return pts, unit(f(N_POINTS, 3)), f(N_POINTS, 1), f(N_POINTS, 3)


def main():
    F, _ = refshim.load()
    fx = {}
    for name in UDF_CFGS:
        cfg, p = _udf_params(name)
        (x,) = inputs("u", name, cfg)
        fx[name + "_x"] = np_(x.float())
        for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
            torch.set_default_dtype(dtype)
            net = F.UDFNetwork(d_in=3, d_out=cfg["d_out"], d_hidden=cfg["d_hidden"], n_layers=cfg["n_layers"],
                               skip_in=cfg["skip_in"], multires=cfg["multires"], scale=cfg["scale"], bias=cfg["bias"],
                               geometric_init=False, weight_norm=True, udf_type="abs")
            net.load_state_dict(O.to_dtype(p, dtype))
            xx = x.float().to(dtype)
            fx["%s_out_%s" % (name, tag)] = np_(net(xx))
            fx["%s_grad_%s" % (name, tag)] = np_(net.gradient(xx.clone())[:, 0])
    for name in COLOR_CFGS:
        cc, p = _color_params(name)
        ins = inputs("c", name, cc)
        for k, t in zip(("pts", "dirs", "feat", "bar_cb", "bar_c", "bar_bl"), ins):
            fx["%s_%s" % (name, k)] = np_(t.float())
        for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
            torch.set_default_dtype(dtype)
            net = F.ResidualRenderingNetwork(d_feature=cc["d_feature"], mode="no_normal", d_in=6, d_out=cc["d_out"],
                                             d_hidden=cc["d_hidden"], n_layers=cc["n_layers"], weight_norm=True,
                                             multires_view=cc["multires_view"], squeeze_out=True,
                                             blending_cand_views=cc["blending_cand_views"])
            net.load_state_dict(O.to_dtype(p, dtype))
            pts, dirs, feat, *bars = [t.float().to(dtype).requires_grad_(i < 3) for i, t in enumerate(ins)]
            out = net(pts, None, dirs, feat)
            for k, t in zip(("base", "color", "blend"), out):
                fx["%s_%s_%s" % (name, k, tag)] = np_(t)
            loss = sum((t * b).sum() for t, b in zip(out, bars))
            for k, gr in zip(("pts", "dirs", "feat"), torch.autograd.grad(loss, [pts, dirs, feat])):
                fx["%s_d%s_%s" % (name, k, tag)] = np_(gr)
    for name in NERF_CFGS:
        nc, p = _nerf_params(name)
        ins = inputs("n", name, nc)
        for k, t in zip(("pts", "dirs", "bar_alpha", "bar_rgb"), ins):
            fx["%s_%s" % (name, k)] = np_(t.float())
        for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
            torch.set_default_dtype(dtype)
            net = F.NeRF(D=nc["D"], W=nc["W"], d_in=nc["d_in"], d_in_view=3, multires=nc["multires"],
                         multires_view=nc["multires_view"], output_ch=4, skips=list(nc["skips"]), use_viewdirs=True)
            net.load_state_dict(O.to_dtype(p, dtype))
            pts, dirs, *bars = [t.float().to(dtype).requires_grad_(i < 2) for i, t in enumerate(ins)]
            alpha, rgb = net(pts, dirs)
            fx["%s_alpha_%s" % (name, tag)], fx["%s_rgb_%s" % (name, tag)] = np_(alpha), np_(rgb)
            loss = (alpha * bars[0]).sum() + (rgb * bars[1]).sum()
            for k, gr in zip(("pts", "dirs"), torch.autograd.grad(loss, [pts, dirs])):
                fx["%s_d%s_%s" % (name, k, tag)] = np_(gr)
    torch.set_default_dtype(torch.float32)
    save_fixtures(NAME, fx)
    print("wrote", len(fx), "arrays;", sum(v.nbytes for v in fx.values()) / 1e6, "MB raw")


if __name__ == "__main__":
    main()

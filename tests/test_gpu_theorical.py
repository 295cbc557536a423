"""The 'theorical' sdf2alpha rule on the device (reference models/udf_renderer_blending.py:321-323): nudf_up_sample mode 2,
the compositing forward / backward and the view renderer under alpha_rule 1, against the UNMODIFIED reference's outputs
(tests/golden/theorical_outputs.*.npz) and the oracle's fp64 autograd, with the bounds of SURVEY.md 8(c); the view renderer
keeps the compositing forward's bits under either rule; and the unmodified runner trains under the rule."""
import ctypes
import glob
import math
import os
import re

import pytest
import torch

from oracle import oracle_theorical as OT
from oracle import oracle_torch as O
from oracle import refshim
from tests.golden_util import Fixtures
from tests.gpu_util import build_modules, err_inf, parity, report, scale_inf

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def th():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return Fixtures("theorical_outputs")


def T(fx, key):
    return torch.from_numpy(fx[key])


def _renderer(g, **kw):
    from neuraludf_b200.models.udf_renderer_blending import UDFRendererBlending
    udf, col, nerf, var, beta = build_modules(g, DEV)
    args = dict(n_samples=64, n_importance=50, n_outside=32, up_sample_steps=5, perturb=0.0, sdf2alpha_type="theorical")
    args.update(kw)
    return UDFRendererBlending(nerf, udf, var, col, beta, **args), (udf, col, nerf, var, beta)


# ---------------------------------------------------------------------------------------------------------------
# up-sampling: nudf_up_sample mode 2 and both importance schedules
# ---------------------------------------------------------------------------------------------------------------
def test_up_sampling_rounds_vs_reference(golden, th):
    from neuraludf_b200 import ops
    g = golden
    o, d = g.t("rays_o").to(DEV), g.t("rays_d").to(DEV)
    near, far = g.t("near"), g.t("far")
    z, udf = g.t("up_z_f32").to(DEV), g.t("up_udf_f32").to(DEV)
    sd = ((far - near) / 64).mean().item()
    total_mism = 0
    for i in range(5):
        gamma = float(min(max(20 * 2 ** (5 - i), 20), 320))
        nz, inds = ops.up_sample(2, o, d, z, udf, sd, 10, 64 * 2 ** i, 64 * 2 ** (i + 1), gamma, return_inds=True)
        nz1, inds1 = ops.up_sample(0, o, d, z, udf, sd, 10, 64 * 2 ** i, 64 * 2 ** (i + 1), gamma, return_inds=True,
                                   alpha_rule=1)
        assert torch.equal(nz, nz1) and torch.equal(inds, inds1)
        mism = inds.cpu() != T(th, "up_inds_r%d_f32" % i)
        total_mism += int(mism.sum())
        report("theorical.up_sample.round%d.index_mismatches" % i, count=int(mism.sum()), total=int(mism.numel()))
        parity("theorical.up_sample.round%d.new_z" % i, nz, T(th, "up_newz_r%d_f64" % i), T(th, "up_newz_r%d_f32" % i),
               tol=1e-5, noise_mult=4.0)
    assert total_mism <= 2, "more index flips than near-ties can explain"


def _z_vs(name, z, ref64, ref32):
    assert z.shape == ref64.shape
    assert bool((z[:, 1:] >= z[:, :-1]).all()), "merged z must be sorted"
    diff = (z.cpu().double() - ref64).abs()
    frac_bad = float((diff > 1e-4).float().mean())
    ref_bad = float(((ref32.double() - ref64).abs() > 1e-4).float().mean())
    report(name, frac_gt_1e4=frac_bad, ref32_frac_gt_1e4=ref_bad, max_abs=float(diff.max()))
    assert frac_bad <= max(2e-3, 3 * ref_bad)
    assert float(diff.max()) <= 3 * float((ref32.double() - ref64).abs().max()) + 1e-4


def test_importance_sampling_schedules_vs_reference(golden, th):
    g = golden
    ren, _ = _renderer(g)
    o, d = g.t("rays_o").to(DEV), g.t("rays_d").to(DEV)
    near, far = g.t("near").to(DEV), g.t("far").to(DEV)
    sd = ((far - near) / 64).mean().item()
    z0 = (near + (far - near) * torch.linspace(0.0, 1.0, 64, device=DEV)[None, :]).contiguous()
    _z_vs("theorical.importance_sample", ren.importance_sample(o, d, z0, sd), T(th, "imp_z_f64"), T(th, "imp_z_f32"))
    ren2, _ = _renderer(g, n_importance=78, n_outside=0, upsampling_type="mix")
    _z_vs("theorical.importance_sample_mix", ren2.importance_sample_mix(o, d, z0, sd), T(th, "impmix_z_f64"),
          T(th, "impmix_z_f32"))


# ---------------------------------------------------------------------------------------------------------------
# compositing alone against the oracle's fp64 / fp32 autograd
# ---------------------------------------------------------------------------------------------------------------
def _oracle_composite(c, dt, S, Oo, has_r, use_norm, bg_rgb, consts):
    inv_s, beta, gamma, r, fs, ssf, bgv = consts
    leaves = {k: c[k].to(dt).clone().requires_grad_(True) for k in ("udf", "grads", "scb", "sc", "bga", "bgc")}
    heads = [torch.tensor(v, dtype=dt, requires_grad=True) for v in (inv_s, beta, gamma)]
    ret = OT.composite(c["d"].to(dt), c["pts"].to(dt), c["mid"].to(dt), c["dists"].to(dt), leaves["udf"], leaves["grads"],
                       leaves["scb"], leaves["sc"], heads[0], heads[1], heads[2], cos_anneal_ratio=r if has_r else None,
                       flip_saturation=fs, background_rgb=bgv.to(dt) if bg_rgb else None,
                       background_alpha=leaves["bga"] if Oo else None,
                       background_sampled_color=leaves["bgc"] if Oo else None, sparse_scale_factor=ssf,
                       use_norm_grad_for_cosine=bool(use_norm), sdf2alpha_type="theorical")
    gen = torch.Generator().manual_seed(99)
    keys = ("color_base", "color", "depth", "weight_sum", "weight_sum_fg_bg")
    bars = {k: torch.randn(ret[k].shape, generator=gen, dtype=torch.float64) for k in keys}
    sb = torch.randn(3, generator=gen, dtype=torch.float64)
    loss = sum((ret[k] * bars[k].to(dt)).sum() for k in keys) + sb[0] * ret["gradient_error"] \
        + sb[1] * ret["gradient_error_near_surface"] + sb[2] * ret["sparse_error"]
    wanted = [leaves["udf"], leaves["grads"], leaves["scb"], leaves["sc"]] + heads + \
        ([leaves["bga"], leaves["bgc"]] if Oo else [])
    gr = torch.autograd.grad(loss, wanted)
    return {k: v.detach() for k, v in ret.items() if torch.is_tensor(v)}, gr, bars, sb


def _bound(new, r64, r32, name):
    """SURVEY 8(c): max(1e-4 max|ref64|, 2 |ref32 - ref64|)"""
    r64 = r64.double()
    e = err_inf(new, r64)
    b = max(1e-4 * scale_inf(r64), 2.0 * err_inf(r32, r64))
    report(name, err=e, bound=b)
    assert e <= b + 1e-30, (name, e, b)


@pytest.mark.parametrize("S,Oo,has_r,use_norm,bg_rgb", [(40, 0, 1, 0, 0), (70, 9, 1, 0, 1), (33, 5, 0, 1, 0),
                                                        (128, 32, 1, 0, 0), (128, 0, 0, 0, 1), (64, 32, 0, 1, 1)])
def test_composite_forward_backward_vs_oracle(S, Oo, has_r, use_norm, bg_rgb):
    from neuraludf_b200 import ops
    from tests.test_raymath_host import make_case
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    c = make_case(3 + S, S, Oo, True)
    N = c["udf"].shape[0]
    consts = (403.4, 148.4, 20.1, 0.35, 0.4, 300.0, torch.tensor([0.2, 0.5, 0.9]))
    inv_s, beta, gamma, r, fs, ssf, bgv = consts
    ret64, gr64, bars, sb = _oracle_composite(c, torch.float64, S, Oo, has_r, use_norm, bg_rgb, consts)
    ret32, gr32, _, _ = _oracle_composite(c, torch.float32, S, Oo, has_r, use_norm, bg_rgb, consts)
    P = N * S
    dev = lambda t: t.float().to(DEV).contiguous()
    udf_t = dev(c["udf"]).reshape(P).requires_grad_(True)
    grads_t = dev(c["grads"]).reshape(P, 3).requires_grad_(True)
    scb_t = dev(c["scb"]).reshape(P, 3).requires_grad_(True)
    sc_t = dev(c["sc"]).reshape(P, 3).requires_grad_(True)
    bga_t = dev(c["bga"]).requires_grad_(True) if Oo else None
    bgc_t = dev(c["bgc"]).requires_grad_(True) if Oo else None
    heads_t = torch.tensor([inv_s, beta, gamma], device=DEV, requires_grad=True)
    cfg = ops._make_cfg(N, S, Oo, float(c["dists"][0, -1]), r if has_r else None, fs, ssf, bool(use_norm),
                        bgv if bg_rgb else None, 1)
    geom = (dev(c["d"]), dev(c["pts"]).reshape(P, 3), dev(c["mid"]), dev(c["dists"]))
    comp = ops.composite(udf_t, grads_t, scb_t, sc_t, bga_t, bgc_t, heads_t, geom, cfg, want_diag=True)
    tag = "theorical.composite[S%d,O%d,r%d,n%d,bg%d]." % (S, Oo, has_r, use_norm, bg_rgb)
    keys = ("color_base", "color", "depth", "weight_sum", "weight_sum_fg_bg")
    for k in keys + ("weights", "normals", "alpha", "alpha_plus", "alpha_minus", "vis_prob"):
        _bound(comp[k].reshape(ret64[k].shape), ret64[k], ret32[k], tag + k)
    # where the reference's alpha is exactly 0, the device's is too
    assert bool((comp["alpha_plus"].cpu()[ret32["alpha_plus"] == 0] == 0).all())
    rs = comp["ray_sums"]
    ge = rs[:, 0].sum() / (rs[:, 1].sum().detach() + 1e-5)
    gens = rs[:, 2].sum() / (rs[:, 3].sum().detach() + 1e-5)
    sp = rs[:, 4].sum() / N
    loss_t = sum((comp[k] * bars[k].float().to(DEV)).sum() for k in keys) + float(sb[0]) * ge + float(sb[1]) * gens \
        + float(sb[2]) * sp
    loss_t.backward()
    _bound(udf_t.grad.reshape(N, S), gr64[0], gr32[0], tag + "udf_bar")
    _bound(grads_t.grad.reshape(N, S, 3), gr64[1], gr32[1], tag + "grads_bar")
    _bound(scb_t.grad.reshape(N, S, 3), gr64[2], gr32[2], tag + "scb_bar")
    _bound(sc_t.grad.reshape(N, S, 3), gr64[3], gr32[3], tag + "sc_bar")
    _bound(heads_t.grad[:1], gr64[4].reshape(1), gr32[4].reshape(1), tag + "inv_s_bar")
    _bound(heads_t.grad[1:], torch.stack([gr64[5], gr64[6]]), torch.stack([gr32[5], gr32[6]]), tag + "beta_gamma_bar")
    if Oo:
        floor = 1e-6 * scale_inf(gr64[2])
        for t, k in ((bga_t, 7), (bgc_t, 8)):
            e = err_inf(t.grad[:, S:], gr64[k][:, S:])
            b = max(1e-4 * scale_inf(gr64[k][:, S:]), 2.0 * err_inf(gr32[k][:, S:], gr64[k][:, S:])) + floor
            assert e <= b, (k, e, b)


# ---------------------------------------------------------------------------------------------------------------
# render_core and whole render() against the reference's goldens, on both engines
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(params=[0, 1], ids=["ffma", "tcgen05"])
def engine(request):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from neuraludf_b200 import _lib
    L = _lib.lib()
    old, old_mask = L.nudf_get_engine(), L.nudf_get_tc_mask()
    L.nudf_set_engine(request.param)
    L.nudf_set_tc_mask(L.nudf_default_tc_mask())
    yield request.param
    L.nudf_set_engine(old)
    L.nudf_set_tc_mask(old_mask)


RC_KEYS = ["color_base", "color", "weights", "depth", "gradient_error", "gradient_error_near_surface", "normals",
           "alpha", "alpha_plus", "alpha_minus", "sparse_error"]


@pytest.mark.parametrize("case", ["rc", "rc_na", "rc_bg"])
def test_render_core_vs_reference(golden, th, engine, case):
    from oracle.make_golden import GRAD_STRIDE
    from oracle.make_golden_theorical import rc_loss
    g = golden
    ren, (udf, col, nerf, var, beta) = _renderer(g)
    kw = dict(cos_anneal_ratio=None, flip_saturation=0.0) if case == "rc_na" else dict(cos_anneal_ratio=0.5,
                                                                                       flip_saturation=0.3)
    if case == "rc_bg":
        kw.update(background_alpha=T(th, "rc_bg_alpha_in_f32").to(DEV),
                  background_sampled_color=T(th, "rc_bg_color_in_f32").to(DEV))
    o, d = g.t("rays_o").to(DEV), g.t("rays_d").to(DEV)
    near, far = g.t("near").to(DEV), g.t("far").to(DEV)
    S = 128
    z = (near + (far - near) * torch.linspace(0.0, 1.0, S, device=DEV)[None, :]).contiguous()
    sd = ((far - near) / S).mean().item()
    ret = ren.render_core(o, d, z, sd, udf, var, col, beta_network=beta, **kw)
    for k in RC_KEYS:
        r64, r32 = T(th, "%s_%s_f64" % (case, k)), T(th, "%s_%s_f32" % (case, k))
        parity("theorical.%s.%s" % (case, k), ret[k].reshape(r64.shape), r64, r32, tol=2e-4,
               noise_mult=4.0 if k == "sparse_error" else 2.0)
    loss = rc_loss(ret, S, torch.float32)
    parity("theorical.%s.loss" % case, loss, T(th, case + "_loss_f64"), T(th, case + "_loss_f32"), tol=2e-4)
    loss.backward()
    n = 0
    for mn, m in (("udf", udf), ("color", col)):
        for pn, p in m.named_parameters():
            key = "%s_grad.%s.%s_f64" % (case, mn, pn)
            if key in th:
                ref, new = T(th, key), p.grad.cpu()
            else:
                ref, new = T(th, key + "_sub"), p.grad.reshape(-1)[::GRAD_STRIDE].cpu()
            e = err_inf(new, ref) / scale_inf(ref)
            n += 1
            assert e < 5e-3, (key, e)
    assert n >= 50
    for mn, m, pn in (("var", var, "variance"), ("beta", beta, "beta")):
        ref64 = T(th, "%s_grad.%s.%s_f64" % (case, mn, pn))
        ref32 = T(th, "%s_grad.%s.%s_f32" % (case, mn, pn))
        parity("theorical.%s.dparam.%s" % (case, pn), getattr(m, pn).grad, ref64, ref32, tol=2e-3, noise_mult=6.0)


def test_whole_render_gradients_with_reference_samples(golden, th, engine):
    """render()'s fine pass on the reference's own samples: every UDF / colour parameter gradient within 5e-3 of max"""
    from oracle.make_golden import GRAD_STRIDE
    g = golden
    ren, (udf, col, nerf, var, beta) = _renderer(g)
    o, d = g.t("rays_o")[:32].to(DEV), g.t("rays_d")[:32].to(DEV)
    near, far = g.t("near")[:32], g.t("far")[:32]
    _, z_out, sd = O.coarse_z(near, far, 64, 32)
    z = T(th, "render_z_vals_f64").float().to(DEV).contiguous()
    ret = ren._render_from_z(o, d, z, z_out.to(DEV), sd, cos_anneal_ratio=0.7, flip_saturation=0.2)
    for k in ("color", "color_base", "depth", "weight_sum", "weight_sum_fg_bg", "normals", "gradient_error", "weights"):
        r64 = T(th, "render_%s_f64" % k)
        parity("theorical.render_fixed_z." + k, ret[k].cpu().reshape(r64.shape), r64, None, tol=3e-4)
    tgt = torch.full((32, 3), 0.4, device=DEV)
    loss = ((ret["color"] - tgt).abs().mean() + 0.01 * (ret["color_base"] - tgt).abs().mean() + 0.1 * ret["gradient_error"])
    loss.backward()
    bad, n = [], 0
    for mn, m in (("udf", udf), ("color", col)):
        for pn, p in m.named_parameters():
            key = "render_grad.%s.%s_f64" % (mn, pn)
            if key in th:
                ref, new = T(th, key), p.grad.cpu()
            elif key + "_sub" in th:
                ref, new = T(th, key + "_sub"), p.grad.reshape(-1)[::GRAD_STRIDE].cpu()
            else:
                continue
            e = err_inf(new, ref) / scale_inf(ref)
            n += 1
            if not e < 5e-3:
                bad.append((key, e))
    assert not bad, bad
    assert n >= 40


def test_whole_render_vs_reference(golden, th):
    g = golden
    ren, _ = _renderer(g)
    o, d = g.t("rays_o")[:32].to(DEV), g.t("rays_d")[:32].to(DEV)
    near, far = g.t("near")[:32].to(DEV), g.t("far")[:32].to(DEV)
    ret = ren.render(o, d, near, far, cos_anneal_ratio=0.7, perturb_overwrite=0, flip_saturation=0.2)
    _z_vs("theorical.render.z_vals", ret["z_vals"], T(th, "render_z_vals_f64"), T(th, "render_z_vals_f32"))
    for k in ("color", "color_base", "depth", "weight_sum", "normals"):
        r64, r32 = T(th, "render_%s_f64" % k), T(th, "render_%s_f32" % k)
        parity("theorical.render." + k, ret[k].cpu().reshape(r64.shape), r64, r32, tol=3e-4, noise_mult=4.0)


# ---------------------------------------------------------------------------------------------------------------
# view renderer, numerical path unchanged, status flag, graph capture
# ---------------------------------------------------------------------------------------------------------------
def test_render_view_bits_match_render(golden, th):
    from neuraludf_b200 import render as R
    g = golden
    ren, _ = _renderer(g, n_outside=32)
    o, d = g.t("rays_o")[:32].to(DEV), g.t("rays_d")[:32].to(DEV)
    near, far = g.t("near")[:32].to(DEV), g.t("far")[:32].to(DEV)
    ren.want_diagnostics = True
    with torch.no_grad():
        ref = ren.render(o, d, near, far, cos_anneal_ratio=0.4, perturb_overwrite=0)
    out = R.render_view(ren, o.reshape(4, 8, 3), d.reshape(4, 8, 3), near.reshape(4, 8, 1), far.reshape(4, 8, 1),
                        cos_anneal_ratio=0.4)
    assert torch.equal(out["color"].reshape(32, 3), ref["color"])
    assert torch.equal(out["depth"].reshape(32, 1), ref["depth"])
    # and the rule matters: the numerical renderer's image differs
    ren.sdf2alpha_type, ren.alpha_rule = "numerical", 0
    out_num = R.render_view(ren, o.reshape(4, 8, 3), d.reshape(4, 8, 3), near.reshape(4, 8, 1), far.reshape(4, 8, 1),
                            cos_anneal_ratio=0.4)
    assert not torch.equal(out_num["color"], out["color"])


def _composite_args(S=96, Oo=16, seed=5):
    from tests.test_raymath_host import make_case
    c = make_case(seed, S, Oo, True)
    N = c["udf"].shape[0]
    P = N * S
    dev = lambda t: t.float().to(DEV).contiguous()
    args = dict(udf=dev(c["udf"]).reshape(P), grads=dev(c["grads"]).reshape(P, 3), scb=dev(c["scb"]).reshape(P, 3),
                sc=dev(c["sc"]).reshape(P, 3), bga=dev(c["bga"]), bgc=dev(c["bgc"]),
                heads=torch.tensor([403.4, 148.4, 20.1], device=DEV))
    geom = (dev(c["d"]), dev(c["pts"]).reshape(P, 3), dev(c["mid"]), dev(c["dists"]))
    return N, S, Oo, float(c["dists"][0, -1]), args, geom


def _forward_and_view(N, S, Oo, sd, a, geom, rule):
    """every output of the compositing forward and of the view renderer on the same inputs under alpha_rule = rule"""
    from neuraludf_b200 import _lib as L
    from neuraludf_b200 import ops
    lib = L.lib()
    cfg = ops._make_cfg(N, S, Oo, sd, 0.35, 0.4, 300.0, False, torch.tensor([0.2, 0.5, 0.9]), rule)
    rays_d, pts, mid, dists = geom
    f = lambda *shape: torch.full(shape, float("nan"), device=DEV)
    outs = {"color_base": f(N, 3), "color": f(N, 3), "depth": f(N, 1), "normals": f(N, 3), "weights": f(N, S + Oo),
            "weight_sum": f(N, 1), "weight_sum_fg_bg": f(N, 1), "ray_sums": f(N, 5)}
    for k in ops.DIAG_KEYS:
        outs[k] = f(N, S)
    outs["gradients_flip"] = f(N, S, 3)
    ro = L.RenderOut()
    for k in L.RENDER_OUT_FIELDS:
        setattr(ro, k, outs[k].data_ptr() if k in outs else None)
    ro.status = None
    L.check(lib.nudf_render_composite_forward(ctypes.byref(cfg), L.ptr(a["heads"]), L.ptr(rays_d), L.ptr(pts), L.ptr(mid),
                                              L.ptr(dists), L.ptr(a["udf"]), 1, L.ptr(a["grads"]), L.ptr(a["scb"]),
                                              L.ptr(a["sc"]), L.ptr(a["bga"]), L.ptr(a["bgc"]), ctypes.byref(ro), None), "fwd")
    vo = {k: f(N, 3 if k in ("color", "color_pixel", "normal") else 1) for k in L.VIEW_OUT_FIELDS}
    ro2 = L.ViewOut()
    for k in L.VIEW_OUT_FIELDS:
        setattr(ro2, k, vo[k].data_ptr())
    r9 = (ctypes.c_float * 9)(1, 0, 0, 0, 1, 0, 0, 0, 1)
    L.check(lib.nudf_render_view_forward(ctypes.byref(cfg), L.ptr(a["heads"]), L.ptr(rays_d), L.ptr(pts), L.ptr(mid),
                                         L.ptr(dists), L.ptr(a["udf"]), 1, L.ptr(a["grads"]), L.ptr(a["sc"]), L.ptr(a["sc"]),
                                         L.ptr(a["bga"]), L.ptr(a["bgc"]), r9, ctypes.byref(ro2), None), "view")
    torch.cuda.synchronize()
    res = {"fwd." + k: v for k, v in outs.items()}
    res.update({"view." + k: v for k, v in vo.items()})
    return res


def test_view_forward_matches_forward_under_both_rules():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    N, S, Oo, sd, a, geom = _composite_args()
    num = _forward_and_view(N, S, Oo, sd, a, geom, 0)
    th_ = _forward_and_view(N, S, Oo, sd, a, geom, 1)
    assert not torch.equal(num["fwd.alpha"], th_["fwd.alpha"])
    for r in (num, th_):
        assert torch.equal(r["view.color"], r["fwd.color"]) and torch.equal(r["view.depth"], r["fwd.depth"])


def test_non_finite_results_raise_under_the_rule():
    from neuraludf_b200 import ops
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    N, S, Oo, sd, a, geom = _composite_args()
    dev = a["udf"].device                              # the status word is kept per device as the kernels see it
    ops.check_status(dev)
    cfg = ops._make_cfg(N, S, Oo, sd, 0.35, 0.4, 300.0, False, None, 1)
    ops.composite(a["udf"], a["grads"], a["scb"], a["sc"], a["bga"], a["bgc"], a["heads"], geom, cfg)
    ops.check_status(dev)                              # a healthy composite raises nothing
    sc = a["sc"].clone()
    sc[7, 1] = float("nan")
    ops.composite(a["udf"], a["grads"], a["scb"], sc, a["bga"], a["bgc"], a["heads"], geom, cfg)
    with pytest.raises(RuntimeError, match="non-finite"):
        ops.check_status(dev)


def test_cuda_graph_capture_under_the_rule():
    from neuraludf_b200 import ops
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    N, S, Oo, sd, a, geom = _composite_args()
    cfg = ops._make_cfg(N, S, Oo, sd, 0.35, 0.4, 300.0, False, None, 1)
    leaves = {k: a[k].clone().requires_grad_(True) for k in ("udf", "grads", "scb", "sc", "bga", "bgc", "heads")}

    def step():
        comp = ops.composite(leaves["udf"], leaves["grads"], leaves["scb"], leaves["sc"], leaves["bga"], leaves["bgc"],
                             leaves["heads"], geom, cfg, want_diag=False)
        loss = comp["color"].sum() + comp["depth"].sum() + comp["ray_sums"][:, 4].sum()
        return torch.autograd.grad(loss, [leaves["udf"], leaves["heads"]])

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        eager = step()
    torch.cuda.current_stream().wait_stream(s)
    gph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gph):
        out = step()
    gph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])


# ---------------------------------------------------------------------------------------------------------------
# the unmodified runner under the launcher, with sdf2alpha_type = theorical
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(not refshim.available(), reason="no staged reference copy (oracle/make_ref.py)")
def test_unmodified_runner_trains_and_validates_theorical(tmp_path):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from tests import runner_env
    from tests.test_runner_e2e import _run
    ref = refshim.REFERENCE_ROOT
    runner = os.path.join(ref, "exp_runner_blending.py")
    tmp = str(tmp_path)
    runner_env.write_synthetic_dtu(os.path.join(tmp, "data", "synth"), n_images=12, width=96, height=72)
    exp = os.path.join(tmp, "exp", "CASE_NAME") + "/"
    conf = runner_env.write_conf(ref, os.path.join(tmp, "synth.conf"), os.path.join(tmp, "data", "CASE_NAME") + "/", exp,
                                 end_iter=4, batch_size=256, save_freq=2, val_freq=3,
                                 extra_replace=(("sdf2alpha_type", "theorical"),))
    assert re.search(r"(?m)^\s*sdf2alpha_type\s*=\s*theorical", open(conf).read())
    r = _run(tmp, [runner, "--mode", "train", "--conf", conf, "--case", "synth", "--gpu", "0"])
    tail = (r.stdout[-3000:] + "\n---- stderr ----\n" + r.stderr[-3000:])
    assert r.returncode == 0, tail
    exp_dir = os.path.join(tmp, "exp", "synth", "udf_dtu")
    ck = sorted(glob.glob(os.path.join(exp_dir, "checkpoints", "ckpt_*.pth")))
    assert [os.path.basename(c) for c in ck] == ["ckpt_000002.pth", "ckpt_000004.pth"], tail
    assert glob.glob(os.path.join(exp_dir, "**", "*.png"), recursive=True), tail
    losses = [float(v) for v in re.findall(r"loss\s*=\s*([-+0-9.eEnaif]+)", r.stdout)]
    assert losses, tail
    assert all(math.isfinite(v) for v in losses), losses
    report("theorical.runner", losses=losses[:8])

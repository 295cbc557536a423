"""GPU tests of the fused blending kernel (csrc/blend.cu) at every patch size it takes, h_patch_size 0..5 (up to the
fine-tuning conf's 11 x 11 patches): render_core at h = 5 against fixtures of the UNMODIFIED reference
(oracle/make_golden_blend_h5.py), ops.blend_views against the op-by-op path over patch sizes, view counts and odd sizes,
the refusal of larger patches by the C entry points, and whole render() calls at the fine-tuning conf's renderer settings.
"""
import ctypes

import pytest
import torch

from neuraludf_b200.synthetic import make_blend_views
from tests.golden_util import Fixtures
from tests.gpu_util import build_modules, err_inf, parity, report, scale_inf

pytestmark = pytest.mark.gpu
DEV = "cuda"
H_PATCH = 5
N_RAYS, S, N_OUT, N_VIEWS = 16, 32, 8, 6
IMG_H, IMG_W = 96, 128


@pytest.fixture(scope="module")
def fx():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return Fixtures("blend_h5_outputs")


def _loss(ret):
    """the fine-tuning loss's shape (exp_runner_blending.py:318-371) with plain L1 terms"""
    n = ret["color"].shape[0]
    tgt = torch.full((n, 3), 0.4, device=DEV)
    loss = (ret["color"] - tgt).abs().mean() + 0.5 * (ret["color_pixel"] - tgt).abs().mean()
    loss = loss + 0.01 * (ret["color_base"] - tgt).abs().mean() + 0.1 * ret["gradient_error"]
    if ret["patch_colors"] is None:
        return loss
    pm = ret["patch_mask"].detach()
    return loss + 0.5 * ((ret["patch_colors"] - 0.4).abs().mean(dim=(1, 2)) * pm).sum() / (pm.sum() + 1e-5)


@pytest.mark.parametrize("engine", [0, 1])
def test_render_core_blending_h5_vs_reference(golden, fx, engine):
    """engine 0: exact fp32; 1: tensor engine (default chains)"""
    from neuraludf_b200 import _lib
    from neuraludf_b200.models.udf_renderer_blending import UDFRendererBlending
    from oracle.make_golden import GRAD_STRIDE
    L = _lib.lib()
    old = L.nudf_get_engine()
    L.nudf_set_engine(engine)
    try:
        udf, col, nerf, var, beta = build_modules(golden, DEV)
        ren = UDFRendererBlending(nerf, udf, var, col, beta, n_samples=S, n_importance=0, n_outside=N_OUT,
                                  up_sample_steps=0, perturb=0.0, h_patch_size=H_PATCH)
        v = {k: t.to(DEV) for k, t in make_blend_views(N_RAYS, n_views=N_VIEWS, height=IMG_H, width=IMG_W,
                                                       seed=0).items()}
        o, d = v["rays_o"], v["rays_d"]
        z = torch.from_numpy(fx["blend_z"]).to(DEV).contiguous()
        z_feed = torch.from_numpy(fx["blend_z_feed"]).to(DEV).contiguous()
        sd = float(fx["blend_sample_dist"])
        bg = ren.render_core_outside(o, d, z_feed, sd, nerf)
        ret = ren.render_core(o, d, z, sd, udf, var, col, beta_network=beta, cos_anneal_ratio=0.8,
                              background_alpha=bg["alpha"], background_sampled_color=bg["sampled_color"],
                              flip_saturation=0.1, color_maps=v["color_maps"], w2cs=v["w2cs"],
                              intrinsics=v["intrinsics"], query_c2w=v["query_c2w"], img_index=None,
                              rays_uv=v["rays_uv"])
        assert ret["patch_colors"].shape == (N_RAYS, 121, 3)
        tag = "blend_h5.e%d." % engine
        tol = 2e-4 if engine == 0 else 5e-4
        for k in ("color_base", "color", "color_pixel", "patch_colors", "patch_mask", "weights", "depth"):
            r64 = torch.from_numpy(fx["blend_%s_f64" % k])
            r32 = torch.from_numpy(fx["blend_%s_f32" % k])
            parity(tag + k, ret[k].reshape(r64.shape), r64, r32, tol=tol)
        loss = _loss(ret)
        parity(tag + "loss", loss, torch.from_numpy(fx["blend_loss_f64"]), torch.from_numpy(fx["blend_loss_f32"]),
               tol=tol)
        loss.backward()
        worst, n = 0.0, 0
        for mn, m in (("udf", udf), ("color", col), ("nerf", nerf)):
            for pn, p in m.named_parameters():
                key = "blend_grad.%s.%s_f64" % (mn, pn)
                if key in fx.files:
                    ref, new = torch.from_numpy(fx[key]), p.grad.cpu()
                elif key + "_sub" in fx.files:
                    ref, new = torch.from_numpy(fx[key + "_sub"]), p.grad.reshape(-1)[::GRAD_STRIDE].cpu()
                else:
                    assert p.grad is None or float(p.grad.abs().max()) == 0.0, key
                    continue
                e = err_inf(new, ref) / scale_inf(ref)
                worst = max(worst, e)
                n += 1
                report(tag + "dparam.%s.%s" % (mn, pn), rel=e)
                assert e < 2e-3, (key, e)
        assert n >= 60
        report(tag + "dparam.worst_rel", rel=worst)
        # the blending logits (10 output rows of the colour head) must receive a gradient
        assert float(col.lin4.weight_v.grad[3:].abs().max()) > 0
    finally:
        L.nudf_set_engine(old)


# point counts N x S that do not fill whole 256-thread blocks (8 points per block)
SHAPES = {1: (37, 19), 8: (13, 7), 32: (5, 3)}


@pytest.mark.parametrize("with_patch", [True, False])
@pytest.mark.parametrize("n_views", [1, 8, 32])
@pytest.mark.parametrize("h", [0, 1, 2, 3, 4, 5])
def test_fused_blend_sweep_vs_op_by_op(h, n_views, with_patch):
    """ops.blend_views against PatchProjector.pixel_warp / patch_warp + color_blend + autograd on the same device, for
    every patch size of the kernel (2 pixels per lane up to h = 3, 4 from h = 4): blended colours, patch mask and the
    gradient w.r.t. the blending logits; some patches lie partly outside the source images."""
    from neuraludf_b200 import ops
    from neuraludf_b200.models.fields import color_blend
    from neuraludf_b200.models.patch_projector import PatchProjector
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    N, S_ = SHAPES[n_views]
    V, npx, n_logits = n_views, (2 * h + 1) ** 2, max(10, n_views + 2)      # columns past V get no gradient
    v = {k: t.to(DEV) for k, t in make_blend_views(N, n_views=V, height=IMG_H, width=IMG_W, seed=9 + h).items()}
    g = torch.Generator().manual_seed(3 + 7 * h + n_views)
    z = v["near"] + (v["far"] - v["near"]) * torch.linspace(0.0, 1.0, S_, device=DEV)[None, :]
    pts = (v["rays_o"][:, None, :] + v["rays_d"][:, None, :] * z[..., None]).contiguous()
    nrm = -v["rays_d"][:, None, :] + 0.6 * torch.randn(N, S_, 3, generator=g).to(DEV)
    nrm = nrm / nrm.norm(dim=-1, keepdim=True)
    logits = (torch.randn(N, S_, n_logits, generator=g) * 1.5).to(DEV).requires_grad_(True)
    pp = PatchProjector(h)
    pix_col, pix_mask = pp.pixel_warp(pts, v["color_maps"], v["intrinsics"], v["w2cs"])
    pat_col = pat_mask = None
    if with_patch:
        pat_col, pat_mask = pp.patch_warp(pts, v["rays_uv"], nrm, v["color_maps"], v["intrinsics"][0], v["intrinsics"],
                                          v["query_c2w"], torch.inverse(v["w2cs"]))
        if h > 0:      # (point, view) patches that are whole, and ones cut by an image border, both occur
            whole, some = pat_mask.all(-1), pat_mask.any(-1)
            assert bool((some & ~whole).any()) and bool(whole.any())
    c_pix, _, c_pat, m_pat = color_blend(logits, None, pix_col, pix_mask, pat_col, pat_mask)
    g_pix = torch.randn(N, S_, 3, generator=g).to(DEV)
    g_pat = torch.randn(N, S_, npx, 3, generator=g).to(DEV)
    loss = (c_pix * g_pix).sum() + ((c_pat * g_pat).sum() if with_patch else 0.0)
    loss.backward()
    ref_grad = logits.grad.clone()
    logits.grad = None

    proj = (v["intrinsics"][:, :3, :3] @ v["w2cs"][:, :3, :]).reshape(V, 12)
    hom = px = None
    if with_patch:
        hom, px = pp.homographies(pts, v["rays_uv"], nrm, (IMG_H, IMG_W), v["intrinsics"][0], v["intrinsics"],
                                  v["query_c2w"], torch.inverse(v["w2cs"]))
        hom = hom.reshape(V, -1, 9)
    f_pix, f_pat, f_m = ops.blend_views(logits.reshape(N * S_, n_logits), pts.reshape(-1, 3), proj, hom, px,
                                        v["color_maps"], N, S_, h)
    loss2 = (f_pix.view(N, S_, 3) * g_pix).sum() + ((f_pat.view(N, S_, npx, 3) * g_pat).sum() if with_patch else 0.0)
    loss2.backward()
    e_pix = float((f_pix.view(N, S_, 3) - c_pix).abs().max())
    e_grad = float((logits.grad - ref_grad).abs().max()) / max(1.0, float(ref_grad.abs().max()))
    tag = "blend.sweep.h%d.v%d.%s" % (h, V, "patch" if with_patch else "pixel")
    report(tag, pix=e_pix, grad_rel=e_grad)
    assert e_pix < 5e-6 and e_grad < 5e-5
    assert float(logits.grad[..., V:].abs().max()) == 0.0
    if with_patch:
        ref_m = m_pat.reshape(-1).float()
        same = f_m == ref_m
        assert float((~same).float().mean()) < 2e-3
        e_pat = float((f_pat.view(N, S_, npx, 3) - c_pat).abs().reshape(N * S_, -1).max(-1).values[same].max())
        report(tag + ".patch_colors", err=e_pat, mask_mismatch=float((~same).float().mean()))
        assert e_pat < 1e-5
    else:
        assert f_pat is None and f_m is None


@pytest.mark.parametrize("backward", [False, True])
def test_blend_refuses_patches_larger_than_11x11(backward):
    """h_patch = 6 (13 x 13 pixels) is refused by the C entry points with -1 and an error message, and nothing runs"""
    from neuraludf_b200 import _lib
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    L = _lib.lib()
    N, S_, V = 2, 3, 2
    P = N * S_
    cfg = _lib.BlendCfg(N, S_, V, IMG_H, IMG_W, 6)
    f = lambda *s: torch.zeros(*s, device=DEV)
    pts, proj, hom, px, imgs, logits = f(P, 3), f(V, 12), f(V, P, 9), f(N, 2), f(V, 3, IMG_H, IMG_W), f(P, V)
    out = torch.full((P, V), 7.0, device=DEV)
    torch.cuda.synchronize()
    n0 = L.nudf_launch_count()
    p = _lib.ptr
    if backward:
        rc = L.nudf_blend_backward(ctypes.byref(cfg), p(pts), p(proj), p(hom), p(px), p(imgs), p(logits), V, p(f(P, 3)),
                                   p(f(P, 169, 3)), p(out), _lib.stream_ptr())
    else:
        rc = L.nudf_blend_forward(ctypes.byref(cfg), p(pts), p(proj), p(hom), p(px), p(imgs), p(logits), V, p(out),
                                  p(f(P, 169, 3)), p(f(P)), _lib.stream_ptr())
    assert rc == -1
    assert b"h_patch" in L.nudf_last_error()
    assert L.nudf_launch_count() == n0
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())


# the renderer settings of confs/udf_dtu_blending_ft.conf
FT = dict(n_samples=64, n_importance=50, n_outside=32, up_sample_steps=5, perturb=1.0, h_patch_size=H_PATCH)
FT_RAYS, FT_VIEWS = 128, 8


@pytest.fixture
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _forbid_op_by_op(monkeypatch):
    from neuraludf_b200.models.patch_projector import PatchProjector

    def refuse(*a, **k):
        raise AssertionError("the op-by-op blending path was taken")
    monkeypatch.setattr(PatchProjector, "pixel_warp", refuse)
    monkeypatch.setattr(PatchProjector, "patch_warp", refuse)


def _render_ft(golden, v, with_patch, perturb_overwrite=-1, seed=0):
    from neuraludf_b200.models.udf_renderer_blending import UDFRendererBlending
    udf, col, nerf, var, beta = build_modules(golden, DEV)
    ren = UDFRendererBlending(nerf, udf, var, col, beta, **FT)
    torch.manual_seed(seed)
    ret = ren.render(v["rays_o"], v["rays_d"], v["near"], v["far"], cos_anneal_ratio=1.0, perturb_overwrite=perturb_overwrite,
                     color_maps=v["color_maps"], w2cs=v["w2cs"], intrinsics=v["intrinsics"], query_c2w=v["query_c2w"],
                     img_index=None, rays_uv=v["rays_uv"] if with_patch else None)
    _loss(ret).backward()
    grads = {"%s.%s" % (mn, pn): p.grad.detach().clone()
             for mn, m in (("udf", udf), ("color", col), ("nerf", nerf)) for pn, p in m.named_parameters()
             if p.grad is not None}
    return ret, grads


def _compare_with_op_by_op(golden, monkeypatch, v, with_patch):
    """perturb 0: the fused path, then the op-by-op branch (reached by lowering the fused view limit) on the same inputs"""
    from neuraludf_b200.models import udf_renderer_blending as urb
    with monkeypatch.context() as mp:
        _forbid_op_by_op(mp)
        fused, g_f = _render_ft(golden, v, with_patch, perturb_overwrite=0)
    with monkeypatch.context() as mp:
        mp.setattr(urb, "FUSED_MAX_VIEWS", 0)
        obo, g_o = _render_ft(golden, v, with_patch, perturb_overwrite=0)
    tag = "blend_h5.render.%s" % ("patch" if with_patch else "pixel")
    e_pix = float((fused["color_pixel"] - obo["color_pixel"]).abs().max())
    report(tag + ".color_pixel", err=e_pix)
    assert e_pix < 1e-5
    if with_patch:
        # a patch whose outermost pixel lies within rounding of the border margin can count a view as whole on one path
        # only (the sweep test bounds that at 2e-3 of the points); such a ray is allowed to differ
        e_ray = (fused["patch_colors"] - obo["patch_colors"]).abs().reshape(FT_RAYS, -1).max(-1).values
        off = e_ray >= 1e-5
        report(tag + ".patch_colors", err_agreeing=float(e_ray[~off].max()), rays_off=int(off.sum()),
               err_max=float(e_ray.max()))
        assert float(e_ray[~off].max()) < 1e-5 and int(off.sum()) <= FT_RAYS // 64
    assert g_f.keys() == g_o.keys() and len(g_f) >= 60
    worst = max(err_inf(g_f[k], g_o[k]) / scale_inf(g_o[k]) for k in g_f)
    report(tag + ".dparam.worst_rel", rel=worst)
    assert worst < 2e-3


def test_render_finetune_conf_fused(cuda, golden, monkeypatch):
    """render() forward + backward at the fine-tuning conf's renderer settings with pixel and patch blending: the fused
    kernel is taken, the outputs have the 11 x 11 shape and are finite, and they match the op-by-op branch"""
    v = {k: t.to(DEV) for k, t in make_blend_views(FT_RAYS, n_views=FT_VIEWS, height=IMG_H, width=IMG_W,
                                                   seed=4).items()}
    with monkeypatch.context() as mp:
        _forbid_op_by_op(mp)
        ret, grads = _render_ft(golden, v, True)                    # perturb 1, as in training
    assert ret["patch_colors"].shape == (FT_RAYS, 121, 3) and ret["patch_mask"].shape == (FT_RAYS,)
    assert ret["z_vals"].shape == (FT_RAYS, FT["n_samples"] + FT["n_importance"])
    for k in ("color", "color_pixel", "patch_colors", "patch_mask"):
        assert torch.isfinite(ret[k]).all(), k
    assert 0.0 < float((ret["patch_mask"] > 0).float().mean())
    assert all(torch.isfinite(g_).all() for g_ in grads.values())
    assert float(grads["color.lin4.weight_v"][3:].abs().max()) > 0
    _compare_with_op_by_op(golden, monkeypatch, v, True)


def test_render_finetune_conf_pixel_only_fused(cuda, golden, monkeypatch):
    """pixel-only blending (colour maps without uv, as validate() renders) at h_patch_size = 5 runs on the fused kernel
    with h_patch = 0 and matches the op-by-op branch"""
    v = {k: t.to(DEV) for k, t in make_blend_views(FT_RAYS, n_views=FT_VIEWS, height=IMG_H, width=IMG_W,
                                                   seed=5).items()}
    with monkeypatch.context() as mp:
        _forbid_op_by_op(mp)
        ret, _ = _render_ft(golden, v, False)
    assert ret["color_pixel"].shape == (FT_RAYS, 3) and ret["patch_colors"] is None
    _compare_with_op_by_op(golden, monkeypatch, v, False)

"""GPU parity of the pixel / patch blending stage (config C3; SURVEY 8(f) rank 1): render_core with colour maps, uv and
a NeRF++ background against fixtures of the UNMODIFIED reference (oracle/make_golden_blend.py), fp64 reference = arbiter.
"""
import os

import numpy as np
import pytest
import torch

from neuraludf_b200.synthetic import make_blend_views
from tests.golden_util import Fixtures
from tests.gpu_util import build_modules, err_inf, parity, report, scale_inf

pytestmark = pytest.mark.gpu
DEV = "cuda"
N_RAYS, S, N_OUT, N_VIEWS = 16, 32, 8, 6


@pytest.fixture(scope="module")
def fx():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return Fixtures("blend_outputs")


def _loss(ret):
    n = ret["color"].shape[0]
    tgt = torch.full((n, 3), 0.4, device=DEV)
    loss = (ret["color"] - tgt).abs().mean() + 0.5 * (ret["color_pixel"] - tgt).abs().mean()
    loss = loss + 0.01 * (ret["color_base"] - tgt).abs().mean() + 0.1 * ret["gradient_error"]
    pm = ret["patch_mask"].detach()
    return loss + 0.5 * ((ret["patch_colors"] - 0.4).abs().mean(dim=(1, 2)) * pm).sum() / (pm.sum() + 1e-5)


@pytest.mark.parametrize("engine", [0, 1])
def test_render_core_blending_vs_reference(golden, fx, engine):
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
                                  up_sample_steps=0, perturb=0.0)
        v = {k: t.to(DEV) for k, t in make_blend_views(N_RAYS, n_views=N_VIEWS, seed=0).items()}
        o, d = v["rays_o"], v["rays_d"]
        z = torch.from_numpy(fx["blend_z"]).to(DEV).contiguous()
        z_feed = torch.from_numpy(fx["blend_z_feed"]).to(DEV).contiguous()
        sd = float(fx["blend_sample_dist"])
        bg = ren.render_core_outside(o, d, z_feed, sd, nerf)
        uv0 = v["rays_uv"].clone()
        ret = ren.render_core(o, d, z, sd, udf, var, col, beta_network=beta, cos_anneal_ratio=0.8,
                              background_alpha=bg["alpha"], background_sampled_color=bg["sampled_color"],
                              flip_saturation=0.1, color_maps=v["color_maps"], w2cs=v["w2cs"],
                              intrinsics=v["intrinsics"], query_c2w=v["query_c2w"], img_index=None,
                              rays_uv=v["rays_uv"])
        assert torch.equal(uv0, v["rays_uv"])
        tag = "blend.e%d." % engine
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
                assert e < 2e-3, (key, e)     # measured worst: 2.7e-4 (all engines); the reference's own fp32 noise is ~2e-3
        assert n >= 60
        report(tag + "dparam.worst_rel", rel=worst)
        # the blending logits (10 output rows of the colour head) must receive a gradient
        assert float(col.lin4.weight_v.grad[3:].abs().max()) > 0
    finally:
        L.nudf_set_engine(old)


def test_whole_render_with_blending_runs_and_trains_all_networks(golden):
    from neuraludf_b200.models.udf_renderer_blending import UDFRendererBlending
    udf, col, nerf, var, beta = build_modules(golden, DEV)
    ren = UDFRendererBlending(nerf, udf, var, col, beta, n_samples=32, n_importance=24, n_outside=8, up_sample_steps=2,
                              perturb=1.0)
    v = {k: t.to(DEV) for k, t in make_blend_views(64, n_views=N_VIEWS, seed=3).items()}
    ret = ren.render(v["rays_o"], v["rays_d"], v["near"], v["far"], cos_anneal_ratio=1.0, flip_saturation=0.0,
                     color_maps=v["color_maps"], w2cs=v["w2cs"], intrinsics=v["intrinsics"], query_c2w=v["query_c2w"],
                     img_index=None, rays_uv=v["rays_uv"])
    assert ret["color_pixel"].shape == (64, 3) and ret["patch_colors"].shape == (64, 49, 3)
    assert ret["patch_mask"].shape == (64,)
    for k in ("color", "color_pixel", "patch_colors", "patch_mask"):
        assert torch.isfinite(ret[k]).all(), k
    _loss(ret).backward()
    for m in (udf, col, nerf):
        gs = [p.grad for p in m.parameters() if p.grad is not None]
        assert gs and all(torch.isfinite(g_).all() for g_ in gs) and sum(float(g_.abs().sum()) for g_ in gs) > 0
    # pixel-only blending (colour maps without uv) is a valid configuration of the trainer as well
    ret2 = ren.render(v["rays_o"], v["rays_d"], v["near"], v["far"], cos_anneal_ratio=1.0, perturb_overwrite=0,
                      color_maps=v["color_maps"], w2cs=v["w2cs"], intrinsics=v["intrinsics"], query_c2w=v["query_c2w"])
    assert ret2["color_pixel"] is not None and ret2["patch_colors"] is None and ret2["patch_mask"] is None


@pytest.mark.parametrize("with_patch", [True, False])
def test_fused_blend_kernel_vs_op_by_op(with_patch):
    """ops.blend_views (csrc/blend.cu) against PatchProjector.pixel_warp / patch_warp + color_blend on the same device:
    blended colours, patch mask and the gradient w.r.t. the blending logits; a size that does not divide the block."""
    from neuraludf_b200 import ops
    from neuraludf_b200.models.fields import color_blend
    from neuraludf_b200.models.patch_projector import PatchProjector
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    N, S, V, h = 37, 19, 5, 3
    v = {k: t.to(DEV) for k, t in make_blend_views(N, n_views=V, height=96, width=128, seed=9).items()}
    g = torch.Generator().manual_seed(3)
    z = v["near"] + (v["far"] - v["near"]) * torch.linspace(0.0, 1.0, S, device=DEV)[None, :]
    pts = (v["rays_o"][:, None, :] + v["rays_d"][:, None, :] * z[..., None]).contiguous()
    nrm = -v["rays_d"][:, None, :] + 0.6 * torch.randn(N, S, 3, generator=g).to(DEV)
    nrm = nrm / nrm.norm(dim=-1, keepdim=True)
    logits = (torch.randn(N, S, 10, generator=g) * 1.5).to(DEV).requires_grad_(True)
    pp = PatchProjector(h)
    pix_col, pix_mask = pp.pixel_warp(pts, v["color_maps"], v["intrinsics"], v["w2cs"])
    pat_col = pat_mask = None
    if with_patch:
        pat_col, pat_mask = pp.patch_warp(pts, v["rays_uv"], nrm, v["color_maps"], v["intrinsics"][0], v["intrinsics"],
                                          v["query_c2w"], torch.inverse(v["w2cs"]))
    c_pix, _, c_pat, m_pat = color_blend(logits, None, pix_col, pix_mask, pat_col, pat_mask)
    g_pix = torch.randn(N, S, 3, generator=g).to(DEV)
    g_pat = torch.randn(N, S, 49, 3, generator=g).to(DEV)
    loss = (c_pix * g_pix).sum() + ((c_pat * g_pat).sum() if with_patch else 0.0)
    loss.backward()
    ref_grad = logits.grad.clone()
    logits.grad = None

    proj = (v["intrinsics"][:, :3, :3] @ v["w2cs"][:, :3, :]).reshape(V, 12)
    hom = px = None
    if with_patch:
        hom, px = pp.homographies(pts, v["rays_uv"], nrm, (96, 128), v["intrinsics"][0], v["intrinsics"], v["query_c2w"],
                                  torch.inverse(v["w2cs"]))
        hom = hom.reshape(V, -1, 9)
    f_pix, f_pat, f_m = ops.blend_views(logits.reshape(N * S, 10), pts.reshape(-1, 3), proj, hom, px, v["color_maps"], N, S, h)
    loss2 = (f_pix.view(N, S, 3) * g_pix).sum() + ((f_pat.view(N, S, 49, 3) * g_pat).sum() if with_patch else 0.0)
    loss2.backward()
    e_pix = float((f_pix.view(N, S, 3) - c_pix).abs().max())
    e_grad = float((logits.grad - ref_grad).abs().max()) / max(1.0, float(ref_grad.abs().max()))
    report("blend.fused.%s" % ("patch" if with_patch else "pixel"), pix=e_pix, grad_rel=e_grad)
    assert e_pix < 5e-6 and e_grad < 5e-5
    assert float(logits.grad[..., V:].abs().max()) == 0.0
    if with_patch:
        ref_m = m_pat.reshape(-1).float()
        same = f_m == ref_m
        assert float((~same).float().mean()) < 2e-3 and 0.2 < float(ref_m.mean()) < 1.0
        e_pat = float((f_pat.view(N, S, 49, 3) - c_pat).abs().reshape(N * S, -1).max(-1).values[same].max())
        report("blend.fused.patch_colors", err=e_pat)
        assert e_pat < 1e-5
    else:
        assert f_pat is None and f_m is None

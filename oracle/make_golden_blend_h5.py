"""Golden fixtures for pixel / patch blending with 11 x 11 patches (h_patch_size = 5, the fine-tuning conf's
udf_dtu_blending_ft.conf), from the UNMODIFIED reference (dev container only).

    python oracle/make_golden_blend_h5.py      # writes tests/golden/blend_h5_outputs.NN.npz

The same two groups as make_golden_blend.py (h_patch_size = 3), on source images of 96 x 128 pixels so that an 11 x 11
patch fits well inside them:
  * proj_*: PatchProjector(5).pixel_warp / patch_warp of the reference on fixed points and normals (fp32);
  * blend_*: render_core with h_patch_size = 5, colour maps, uv and a NeRF++ background produced by the reference's
    render_core_outside, in fp32 and fp64, with the gradients of the same trainer-like loss.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle_torch as O  # noqa: E402
from oracle import refshim  # noqa: E402
from oracle.make_golden import GRAD_STRIDE, build_ref_nets, np_  # noqa: E402
from oracle.make_golden_blend import blend_loss  # noqa: E402
from tests.golden_util import save_fixtures  # noqa: E402

H_PATCH = 5
N_RAYS, S, N_OUT, N_VIEWS = 16, 32, 8, 6
IMG_H, IMG_W = 96, 128
N_PROJ, S_PROJ = 8, 12        # projector points: [8, 12] x 6 views x 121 pixels keeps the fixture small


def main():
    F, R = refshim.load()
    udf_c, col_c, nerf_c = O.udf_cfg(), O.color_cfg(), O.nerf_cfg()
    udf_p, col_p = O.make_udf_params(udf_c, seed=0), O.make_color_params(col_c, seed=1)
    nerf_p, sc = O.make_nerf_params(nerf_c, seed=2), O.make_scalars()
    fx = {}

    # ---- projector alone (fp32, CPU) ----
    torch.set_default_dtype(torch.float32)
    from models.patch_projector import PatchProjector
    pp = PatchProjector(H_PATCH)
    pv = O.make_blend_views(N_PROJ, n_views=N_VIEWS, height=IMG_H, width=IMG_W, seed=0)
    z = pv["near"] + (pv["far"] - pv["near"]) * torch.linspace(0.0, 1.0, S_PROJ)[None, :]
    pts = pv["rays_o"][:, None, :] + pv["rays_d"][:, None, :] * z[..., None]
    gg = torch.Generator().manual_seed(21)
    nrm = -pv["rays_d"][:, None, :] + 0.5 * torch.randn(N_PROJ, S_PROJ, 3, generator=gg)
    nrm = nrm / nrm.norm(dim=-1, keepdim=True)
    fx["proj_pts"], fx["proj_normals"] = np_(pts), np_(nrm)
    c, m = pp.pixel_warp(pts, pv["color_maps"], pv["intrinsics"], pv["w2cs"])
    fx["proj_pixel_color"], fx["proj_pixel_mask"] = np_(c), np_(m)
    c, m = pp.patch_warp(pts, pv["rays_uv"].clone(), nrm, pv["color_maps"], pv["intrinsics"][0],
                         pv["intrinsics"], pv["query_c2w"], torch.inverse(pv["w2cs"]))
    fx["proj_patch_color"], fx["proj_patch_mask"] = np_(c), np_(m)
    visible = float(m.all(dim=-1).float().mean())          # (point, view) pairs that see the whole patch
    print("projector: whole-patch visible fraction %.3f" % visible)
    assert 0.2 < visible < 1.0, visible

    # ---- render_core with blending, h_patch_size = 5 ----
    views = O.make_blend_views(N_RAYS, n_views=N_VIEWS, height=IMG_H, width=IMG_W, seed=0)
    for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        udf, col, nerf, var, beta = build_ref_nets(F, udf_c, col_c, nerf_c, udf_p, col_p, nerf_p, sc, dtype)
        ren = R.UDFRendererBlending(nerf, udf, var, col, beta, n_samples=S, n_importance=0, n_outside=N_OUT,
                                    up_sample_steps=0, perturb=0.0, h_patch_size=H_PATCH)
        ren.patch_projector.z_axis = ren.patch_projector.z_axis.to(dtype)
        v = {k: t.to(dtype) for k, t in views.items()}
        o, d, near, far = v["rays_o"], v["rays_d"], v["near"], v["far"]
        z = near + (far - near) * torch.linspace(0.0, 1.0, S)[None, :]
        sd = ((far - near) / S).mean().item()
        z_out = torch.linspace(1e-3, 1.0 - 1.0 / (N_OUT + 1.0), N_OUT)
        z_out = far / torch.flip(z_out, dims=[-1]) + 1.0 / S
        z_feed, _ = torch.sort(torch.cat([z, z_out], dim=-1), dim=-1)
        if tag == "f32":
            fx["blend_z"], fx["blend_z_feed"], fx["blend_sample_dist"] = np_(z), np_(z_feed), np.array(sd)
        for m_ in (udf, col, var, beta, nerf):
            m_.zero_grad(set_to_none=True)
        bg = ren.render_core_outside(o, d, z_feed, sd, nerf)
        ret = ren.render_core(o, d, z, sd, udf, var, col, beta_network=beta, cos_anneal_ratio=0.8,
                              background_alpha=bg["alpha"], background_sampled_color=bg["sampled_color"],
                              flip_saturation=0.1, color_maps=v["color_maps"], w2cs=v["w2cs"],
                              intrinsics=v["intrinsics"], query_c2w=v["query_c2w"], img_index=None,
                              rays_uv=v["rays_uv"].clone())
        assert ret["patch_colors"].shape == (N_RAYS, (2 * H_PATCH + 1) ** 2, 3)
        loss = blend_loss(ret, dtype)
        loss.backward()
        for k in ("color_base", "color", "color_pixel", "patch_colors", "patch_mask", "weights", "depth"):
            fx["blend_%s_%s" % (k, tag)] = np_(ret[k])
        fx["blend_loss_" + tag] = np_(loss)
        for mn, m_ in (("udf", udf), ("color", col), ("var", var), ("beta", beta), ("nerf", nerf)):
            for pn, p in m_.named_parameters():
                if p.grad is not None:
                    fx["blend_grad.%s.%s_%s" % (mn, pn, tag)] = np_(p.grad)

    torch.set_default_dtype(torch.float32)
    for k in list(fx):
        if "_grad." in k and fx[k].size > 4096:
            if k.endswith("_f32"):
                del fx[k]
                continue
            full = fx.pop(k).astype(np.float64).reshape(-1)
            fx[k + "_sub"] = full[::GRAD_STRIDE].copy()
            fx[k + "_norm"] = np.array(np.sqrt((full ** 2).sum()))
    save_fixtures("blend_h5_outputs", fx)
    print("wrote", len(fx), "arrays;", sum(a.nbytes for a in fx.values()) / 1e6, "MB raw")


if __name__ == "__main__":
    main()

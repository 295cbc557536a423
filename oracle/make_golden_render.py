"""Golden fixtures for whole-view rendering (neuraludf_b200/render.py), from the UNMODIFIED reference (dev container only).

    python oracle/make_golden_render.py      # writes tests/golden/render_view.NN.npz

Scene networks of make_golden.py (same seeds); a synthetic DTU-layout scan written by tests/runner_env.write_synthetic_dtu
(9 cameras, 96 x 72), one view at resolution level 3 (32 x 24 rays) with its 8 source views.  The reference's `Dataset`
methods run unbound on a small CPU stand-in object holding the tensors its __init__ builds (`load_K_Rt_from_P` of
world_mat @ scale_mat, images BGR / 256): gen_rays_at, near_far_from_sphere, prepare_ref_src_pairs, get_ref_src_info and
gen_rays_between (ratios 0.25 and 0.6); `.cuda()` is the identity in this CPU-only process.  Then:
  * e2e_*:    one render() call per dtype (fp32, fp64) with the source views, perturb_overwrite = 0 (its own sampling);
  * strict_*: render_core_outside + render_core on the fp32 call's z_vals, as render() runs them (:645-680), fp32 and fp64;
each with color, color_pixel, depth and validate()'s normal map (exp_runner_blending.py:660-683 restated:
sum(gradients_flip * weights[:, :S] * inside_sphere) rotated by inv(pose[:3, :3])).
"""
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle_torch as O  # noqa: E402
from oracle import refshim  # noqa: E402
from oracle.make_golden import build_ref_nets, np_  # noqa: E402
from tests.golden_util import save_fixtures  # noqa: E402
from tests.runner_env import write_synthetic_dtu  # noqa: E402

N_IMAGES, WIDTH, HEIGHT, LEVEL, IDX = 9, 96, 72, 3, 2
COS_ANNEAL = 0.7
RATIOS = (0.25, 0.6)
RENDERER = dict(n_samples=64, n_importance=50, n_outside=32, up_sample_steps=5, perturb=0.0)


def scan_standin(data_dir, load_K_Rt_from_P):
    """the tensors Dataset.__init__ builds (dataset/dataset.py:41-127, downsample_factor 1), on the CPU"""
    import cv2
    from glob import glob
    ds = types.SimpleNamespace()
    ds.images_lis = sorted(glob(os.path.join(data_dir, "image/*.png")))
    ds.n_images = len(ds.images_lis)
    cams = np.load(os.path.join(data_dir, "cameras.npz"))
    ds.images_np = np.stack([cv2.imread(f) for f in ds.images_lis]) / 256.0
    intr, poses = [], []
    for i in range(ds.n_images):
        P = cams["world_mat_%d" % i].astype(np.float32) @ cams["scale_mat_%d" % i].astype(np.float32)
        k, p = load_K_Rt_from_P(None, P[:3, :4])
        intr.append(torch.from_numpy(k).float())
        poses.append(torch.from_numpy(p).float())
    ds.images = torch.from_numpy(ds.images_np.astype(np.float32))
    ds.intrinsics_all = torch.stack(intr)
    ds.intrinsics_all_inv = torch.inverse(ds.intrinsics_all)
    ds.pose_all = torch.stack(poses)
    ds.H, ds.W = ds.images.shape[1], ds.images.shape[2]
    return ds


def normal_map(ret, rot):
    S = ret["gradients_flip"].shape[1]
    n = (ret["gradients_flip"] * ret["weights"][:, :S, None] * ret["inside_sphere"][..., None]).sum(dim=1)
    return torch.matmul(rot.to(n.dtype)[None], n[:, :, None])[:, :, 0]


def main():
    F, R = refshim.load()
    from dataset.dataset import Dataset, load_K_Rt_from_P
    torch.Tensor.cuda = lambda self, *a, **k: self            # CPU-only process: the reference's .cuda() calls are no-ops
    tmp = tempfile.mkdtemp()
    data = write_synthetic_dtu(tmp, n_images=N_IMAGES, width=WIDTH, height=HEIGHT)
    torch.set_default_dtype(torch.float32)
    ds = scan_standin(data, load_K_Rt_from_P)
    fx = {"intrinsics": np_(ds.intrinsics_all), "pose": np_(ds.pose_all)}
    ds.ref_src_pair = Dataset.prepare_ref_src_pairs(ds)
    fx["src_pairs"] = np.stack([np_(ds.ref_src_pair[i][:8]) for i in range(ds.n_images)])
    rays_o, rays_d = Dataset.gen_rays_at(ds, IDX, resolution_level=LEVEL)
    H, W = rays_o.shape[:2]
    o, d = rays_o.reshape(-1, 3).contiguous(), rays_d.reshape(-1, 3).contiguous()
    near, far = Dataset.near_far_from_sphere(ds, o, d)
    fx.update(rays_o=np_(o), rays_d=np_(d), near=np_(near), far=np_(far), hw=np.array([H, W]))
    ref_c2w, src_c2ws, src_intr, src_images, _ = Dataset.get_ref_src_info(ds, IDX)
    rot = torch.from_numpy(np.linalg.inv(np_(ds.pose_all[IDX, :3, :3])))
    for k, r in enumerate(RATIOS):
        bo, bd = Dataset.gen_rays_between(ds, 0, 1, r, resolution_level=LEVEL)
        fx["between%d_ratio" % k], fx["between%d_rays_o" % k], fx["between%d_rays_d" % k] = np.array(r), np_(bo), np_(bd)

    udf_c, col_c, nerf_c = O.udf_cfg(), O.color_cfg(), O.nerf_cfg()
    udf_p, col_p = O.make_udf_params(udf_c, seed=0), O.make_color_params(col_c, seed=1)
    nerf_p, sc = O.make_nerf_params(nerf_c, seed=2), O.make_scalars()
    z32 = None
    for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        udf, col, nerf, var, beta = build_ref_nets(F, udf_c, col_c, nerf_c, udf_p, col_p, nerf_p, sc, dtype)
        ren = R.UDFRendererBlending(nerf, udf, var, col, beta, **RENDERER)
        ren.patch_projector.z_axis = ren.patch_projector.z_axis.to(dtype)
        # render()'s sparse_random_error draws fp32 points (`.float()`, :683); in the fp64 run they are cast on the way in
        # (the value is not stored)
        udf.udf = lambda x, f=udf.udf: f(x.to(dtype))
        c = lambda t: t.to(dtype)
        blend = dict(color_maps=c(src_images), w2cs=torch.inverse(c(src_c2ws)), intrinsics=c(src_intr),
                     query_c2w=c(ref_c2w))
        ret = ren.render(c(o), c(d), c(near), c(far), cos_anneal_ratio=COS_ANNEAL, perturb_overwrite=0, **blend)
        if tag == "f32":
            z32 = ret["z_vals"].detach().clone()
            fx["z_vals"] = np_(z32)
        for k in ("color", "color_pixel", "depth"):
            fx["e2e_%s_%s" % (k, tag)] = np_(ret[k])
        fx["e2e_normal_" + tag] = np_(normal_map(ret, rot))
        # the same passes on the fp32 call's samples (reference render(), :645-680)
        z = c(z32)
        sd = ((c(far) - c(near)) / RENDERER["n_samples"]).mean()
        zo = torch.linspace(1e-3, 1.0 - 1.0 / (RENDERER["n_outside"] + 1.0), RENDERER["n_outside"])
        zo = c(far) / torch.flip(zo, dims=[-1]) + 1.0 / RENDERER["n_samples"]
        z_feed, _ = torch.sort(torch.cat([z, zo], dim=-1), dim=-1)
        bg = ren.render_core_outside(c(o), c(d), z_feed, sd, nerf)
        ret = ren.render_core(c(o), c(d), z, sd, udf, var, col, beta_network=beta, cos_anneal_ratio=COS_ANNEAL,
                              background_alpha=bg["alpha"], background_sampled_color=bg["sampled_color"], **blend)
        for k in ("color", "color_pixel", "depth"):
            fx["strict_%s_%s" % (k, tag)] = np_(ret[k])
        fx["strict_normal_" + tag] = np_(normal_map(ret, rot))
    torch.set_default_dtype(torch.float32)
    save_fixtures("render_view", fx)
    print("wrote", len(fx), "arrays;", sum(a.nbytes for a in fx.values()) / 1e6, "MB raw")


if __name__ == "__main__":
    main()

"""Times pixel / patch blending at the fine-tuning conf's sizes (confs/udf_dtu_blending_ft.conf: 512 rays, 64 + 50
samples, 8 source views of 1600 x 1200, 10 blending logits, h_patch_size 5), on the fused kernel (csrc/blend.cu) and on the
op-by-op path (PatchProjector.pixel_warp / patch_warp + fields.color_blend + autograd), at h = 3 and h = 5.

    python tools/blend_bench.py [--iters 20] [--warmup 3] [--out result.json]
    python tools/blend_bench.py --dump DIR      # only writes the h = 3 fused outputs (blend_h3.npz) and exits

Two measurements, each a median of --iters calls (CUDA events) after --warmup calls:
  * the blend stage alone, forward + backward to the logits, on seeded synthetic points, normals and logits; both paths
    include their homographies; also the fused kernels alone (homographies precomputed).  The op-by-op path's bytes are
    counted from shapes as a lower bound: its [N, S, V, Npx, 3] fp32 patch-colour tensor written once, read once by the
    blend and once by the backward.  Peak memory is torch.cuda.max_memory_allocated over one call.  At the timed size
    the two paths' outputs are compared with each other (against the bounds of tests/test_gpu_blend_h5.py) and with the
    op-by-op path evaluated in fp64;
  * a whole render() forward + backward (golden-scene-sized networks of neuraludf_b200.synthetic, a loss of the runner's
    shape), fused against the op-by-op branch of UDFRendererBlending._blend.
The card name, power limit and SM clocks are read with nvidia-smi in the same run.  --dump writes the h = 3 fused outputs
of the blend stage, so that two builds of the library (NUDF_LIB_PATH) can be compared bit for bit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

N_RAYS, N_SAMPLES, N_VIEWS, N_LOGITS = 512, 64 + 50, 8, 10
IMG_H, IMG_W = 1200, 1600
FT_RENDERER = dict(n_samples=64, n_importance=50, n_outside=32, up_sample_steps=5, perturb=1.0)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn, iters, warmup):
    """median and min of per-call device time (CUDA events), ms"""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts), min(ts)


def peak_bytes(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def blend_inputs(dev, seed=0):
    """seeded points along the rays of a query view, surface normals near the ray direction, logits, upstream gradients"""
    from neuraludf_b200.synthetic import make_blend_views
    v = {k: t.to(dev) for k, t in make_blend_views(N_RAYS, n_views=N_VIEWS, height=IMG_H, width=IMG_W, seed=seed).items()}
    g = torch.Generator().manual_seed(100 + seed)
    z = v["near"] + (v["far"] - v["near"]) * torch.linspace(0.0, 1.0, N_SAMPLES, device=dev)[None, :]
    pts = (v["rays_o"][:, None, :] + v["rays_d"][:, None, :] * z[..., None]).contiguous()
    nrm = -v["rays_d"][:, None, :] + 0.6 * torch.randn(N_RAYS, N_SAMPLES, 3, generator=g).to(dev)
    v["pts"], v["normals"] = pts, nrm / nrm.norm(dim=-1, keepdim=True)
    v["logits"] = (torch.randn(N_RAYS, N_SAMPLES, N_LOGITS, generator=g) * 1.5).to(dev)
    v["g_pix"] = torch.randn(N_RAYS, N_SAMPLES, 3, generator=g).to(dev)
    v["g_pat"] = {h: torch.randn(N_RAYS, N_SAMPLES, (2 * h + 1) ** 2, 3, generator=g).to(dev) for h in (3, 5)}
    return v


def fused_blend(v, h, hom=None):
    """forward + backward to the logits on the fused kernel; returns (c_pix, c_pat, m_pat, d logits).  hom: precomputed
    (homographies [V, P, 9], query pixels), or None to build them as UDFRendererBlending._blend does"""
    from neuraludf_b200 import ops
    from neuraludf_b200.models.patch_projector import PatchProjector
    N, S = N_RAYS, N_SAMPLES
    proj = (v["intrinsics"][:, :3, :3] @ v["w2cs"][:, :3, :]).reshape(N_VIEWS, 12)
    if hom is None:
        hom, px = PatchProjector(h).homographies(v["pts"], v["rays_uv"], v["normals"], (IMG_H, IMG_W), v["intrinsics"][0],
                                                 v["intrinsics"], v["query_c2w"], torch.inverse(v["w2cs"]))
        hom = (hom.reshape(N_VIEWS, -1, 9), px)
    logits = v["logits"].clone().requires_grad_(True)
    c_pix, c_pat, m_pat = ops.blend_views(logits.reshape(N * S, N_LOGITS), v["pts"].reshape(-1, 3), proj, hom[0], hom[1],
                                          v["color_maps"], N, S, h)
    loss = (c_pix.view(N, S, 3) * v["g_pix"]).sum() + (c_pat.view(N, S, -1, 3) * v["g_pat"][h]).sum()
    loss.backward()
    return c_pix.view(N, S, 3), c_pat.view(N, S, -1, 3), m_pat.view(N, S), logits.grad


def op_by_op_blend(v, h):
    from neuraludf_b200.models.fields import color_blend
    from neuraludf_b200.models.patch_projector import PatchProjector
    pp = PatchProjector(h)
    logits = v["logits"].clone().requires_grad_(True)
    pix_col, pix_mask = pp.pixel_warp(v["pts"], v["color_maps"], v["intrinsics"], v["w2cs"])
    pat_col, pat_mask = pp.patch_warp(v["pts"], v["rays_uv"], v["normals"], v["color_maps"], v["intrinsics"][0],
                                      v["intrinsics"], v["query_c2w"], torch.inverse(v["w2cs"]))
    c_pix, _, c_pat, m_pat = color_blend(logits, None, pix_col, pix_mask, pat_col, pat_mask)
    loss = (c_pix * v["g_pix"]).sum() + (c_pat * v["g_pat"][h]).sum()
    loss.backward()
    return c_pix, c_pat, m_pat.view(N_RAYS, N_SAMPLES), logits.grad


def agreement(f, o, r64):
    """fused (f) against op by op (o), with the bounds of tests/test_gpu_blend_h5.py::test_fused_blend_sweep_vs_op_by_op,
    and each of them against the op-by-op path evaluated in fp64 (r64), where the patch masks of all three agree"""
    f, o, r64 = [t.detach() for t in f], [t.detach() for t in o], [t.detach() for t in r64]
    same = (f[2] == o[2].float()) & (f[2] == r64[2].float())
    pat = lambda a, b: float((a - b).abs().reshape(same.numel(), -1).max(-1).values[same.reshape(-1)].max())  # noqa: E731
    rel = lambda a, b: float((a - b).abs().max()) / max(1.0, float(r64[3].abs().max()))  # noqa: E731
    out = {"fused_vs_op_by_op": {"pix": float((f[0] - o[0]).abs().max()), "grad_rel": rel(f[3], o[3]),
                                 "patch_where_masks_agree": pat(f[1], o[1]),
                                 "mask_mismatch": float((f[2] != o[2].float()).float().mean())},
           "visible_fraction": float(o[2].float().mean())}
    for name, x in (("fused", f), ("op_by_op", o)):
        out[name + "_vs_fp64"] = {"pix": float((x[0].double() - r64[0]).abs().max()), "grad_rel": rel(x[3].double(), r64[3]),
                                  "patch_where_masks_agree": pat(x[1].double(), r64[1])}
    a = out["fused_vs_op_by_op"]
    a["within_test_bounds"] = (a["pix"] < 5e-6 and a["grad_rel"] < 5e-5 and a["patch_where_masks_agree"] < 1e-5
                               and a["mask_mismatch"] < 2e-3)
    return out


def bench_blend(args, dev):
    from neuraludf_b200.models.patch_projector import PatchProjector
    v = blend_inputs(dev)
    res = {}
    for h in (3, 5):
        npx = (2 * h + 1) ** 2
        t_bytes = N_RAYS * N_SAMPLES * N_VIEWS * npx * 3 * 4
        hp = PatchProjector(h).homographies(v["pts"], v["rays_uv"], v["normals"], (IMG_H, IMG_W), v["intrinsics"][0],
                                            v["intrinsics"], v["query_c2w"], torch.inverse(v["w2cs"]))
        hom = (hp[0].reshape(N_VIEWS, -1, 9).contiguous(), hp[1])
        r = {"patch_pixels": npx}
        r["fused_ms"], r["fused_min_ms"] = timed(lambda: fused_blend(v, h), args.iters, args.warmup)
        r["fused_kernels_only_ms"], _ = timed(lambda: fused_blend(v, h, hom=hom), args.iters, args.warmup)
        r["op_by_op_ms"], r["op_by_op_min_ms"] = timed(lambda: op_by_op_blend(v, h), args.iters, args.warmup)
        r["speedup"] = r["op_by_op_ms"] / r["fused_ms"]
        r["fused_peak_MB"] = peak_bytes(lambda: fused_blend(v, h)) / 1e6
        r["op_by_op_peak_MB"] = peak_bytes(lambda: op_by_op_blend(v, h)) / 1e6
        r["op_by_op_patch_tensor_MB"] = t_bytes / 1e6
        r["op_by_op_bytes_lower_bound_GB"] = 3 * t_bytes / 1e9
        r["op_by_op_lower_bound_rate_TBps"] = 3 * t_bytes / (r["op_by_op_ms"] * 1e-3) / 1e12
        v64 = {k: (t.double() if torch.is_tensor(t) and t.is_floating_point() else t) for k, t in v.items()}
        v64["g_pat"] = {k: t.double() for k, t in v["g_pat"].items()}
        r["agreement"] = agreement(fused_blend(v, h), op_by_op_blend(v, h), op_by_op_blend(v64, h))
        del v64
        res["h%d" % h] = r
        print("blend h=%d:" % h, json.dumps(r), flush=True)
    return res


def networks(dev):
    from neuraludf_b200 import synthetic as O
    from neuraludf_b200.models import fields as F
    udf = F.UDFNetwork(d_in=3, d_out=257, d_hidden=256, n_layers=8, skip_in=(4,), multires=6, bias=0.5, scale=1.0,
                       geometric_init=True, weight_norm=True, udf_type="abs")
    udf.load_state_dict(O.make_udf_params(O.udf_cfg(), seed=0))
    col = F.ResidualRenderingNetwork(d_feature=256, mode="no_normal", d_in=6, d_out=3, d_hidden=128, n_layers=4,
                                     weight_norm=True, multires_view=4, squeeze_out=True, blending_cand_views=N_LOGITS)
    col.load_state_dict(O.make_color_params(O.color_cfg(), seed=1))
    nerf = F.NeRF(D=8, d_in=4, d_in_view=3, W=256, multires=10, multires_view=4, output_ch=4, skips=[4], use_viewdirs=True)
    nerf.load_state_dict(O.make_nerf_params(O.nerf_cfg(), seed=2))
    var = F.SingleVarianceNetwork(0.6)
    beta = F.BetaNetwork(init_var_beta=0.5, init_var_gamma=0.3, init_var_zeta=0.3, beta_min=5e-5,
                         requires_grad_beta=True, requires_grad_gamma=False, requires_grad_zeta=False)
    return [m.to(dev) for m in (udf, col, nerf, var, beta)]


def bench_render(args, dev):
    """render() fwd + bwd at the fine-tuning conf's settings, pixel + patch blending, h = 3 and 5"""
    from neuraludf_b200.models import udf_renderer_blending as urb
    from neuraludf_b200.synthetic import make_blend_views
    udf, col, nerf, var, beta = networks(dev)
    mods = (udf, col, nerf, var, beta)
    v = {k: t.to(dev) for k, t in make_blend_views(N_RAYS, n_views=N_VIEWS, height=IMG_H, width=IMG_W, seed=1).items()}
    tgt = torch.full((N_RAYS, 3), 0.4, device=dev)
    res = {}
    for h in (3, 5):
        ren = urb.UDFRendererBlending(nerf, udf, var, col, beta, h_patch_size=h, **FT_RENDERER)
        ren.want_diagnostics = False

        def step():
            for m in mods:
                m.zero_grad(set_to_none=True)
            ret = ren.render(v["rays_o"], v["rays_d"], v["near"], v["far"], cos_anneal_ratio=1.0, flip_saturation=0.0,
                             color_maps=v["color_maps"], w2cs=v["w2cs"], intrinsics=v["intrinsics"],
                             query_c2w=v["query_c2w"], rays_uv=v["rays_uv"])
            pm = ret["patch_mask"].detach()
            loss = ((ret["color"] - tgt).abs().mean() + 0.01 * (ret["color_base"] - tgt).abs().mean()
                    + 0.1 * ret["gradient_error"] + 0.1 * (ret["color_pixel"] - tgt).abs().mean()
                    + 0.1 * ((ret["patch_colors"] - 0.4).abs().mean(dim=(1, 2)) * pm).sum() / (pm.sum() + 1e-5))
            loss.backward()
            return loss

        r = {}
        r["fused_ms"], r["fused_min_ms"] = timed(step, args.iters, args.warmup)
        r["fused_peak_MB"] = peak_bytes(step) / 1e6
        old = urb.FUSED_MAX_VIEWS
        urb.FUSED_MAX_VIEWS = 0                   # every blend takes the op-by-op branch
        try:
            r["op_by_op_ms"], r["op_by_op_min_ms"] = timed(step, args.iters, args.warmup)
            r["op_by_op_peak_MB"] = peak_bytes(step) / 1e6
        finally:
            urb.FUSED_MAX_VIEWS = old
        r["speedup"] = r["op_by_op_ms"] / r["fused_ms"]
        res["h%d" % h] = r
        print("render h=%d:" % h, json.dumps(r), flush=True)
    return res


def dump(out_dir, dev):
    os.makedirs(out_dir, exist_ok=True)
    v = blend_inputs(dev)
    c_pix, c_pat, m_pat, g = fused_blend(v, 3)
    arrays = {"c_pix": c_pix, "c_pat": c_pat, "m_pat": m_pat, "g_logits": g}
    np.savez(os.path.join(out_dir, "blend_h3.npz"), **{k: t.detach().cpu().numpy() for k, t in arrays.items()})
    from neuraludf_b200 import _lib
    print("dumped h = 3 fused outputs of", _lib.LIB_PATH, "to", out_dir)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--dump", default=None, metavar="DIR")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("blend_bench needs a CUDA device")
    dev = torch.device("cuda", 0)
    if args.dump:
        dump(args.dump, dev)
        return
    from neuraludf_b200 import _lib
    out = {"gpu_before": gpu_info(), "library": _lib.LIB_PATH, "iters": args.iters, "warmup": args.warmup,
           "shapes": {"rays": N_RAYS, "samples": N_SAMPLES, "views": N_VIEWS, "image_hw": [IMG_H, IMG_W],
                      "logits": N_LOGITS}}
    out["blend_stage"] = bench_blend(args, dev)
    out["render"] = bench_render(args, dev)
    out["gpu_after"] = gpu_info()
    s = json.dumps(out)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()

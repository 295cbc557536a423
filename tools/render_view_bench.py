"""Time per view of render.render_view against the runner's validate() loop (render() on 512-ray chunks plus its normal
expression), alternating in one process; peak memory, launches per view and the time of nudf_render_view_forward.

The golden scene's networks (DTU shapes), the DTU conf's sampling, a synthetic 1600 x 1200 scan
with 8 source views; one view at level 4 and at level 1.  Prints one JSON line per level and writes them to --out."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def modules(dev):
    """the golden scene's networks (tests/golden: UDF 8 x 256, colour 2 x (4 x 128), NeRF++ 8 x 256, the scalar heads)"""
    from tests.golden_util import load_golden
    from tests.gpu_util import build_modules
    return build_modules(load_golden(), dev)


def runner_loop(ren, scan, idx, level, kw, ratio):
    """validate()'s loop (exp_runner_blending.py:621-668): render() per 512 rays, host copies of its outputs"""
    rays_o, rays_d, near, far = scan.rays_at(idx, level)
    o, d = rays_o.reshape(-1, 3).split(512), rays_d.reshape(-1, 3).split(512)
    nr, fr = near.reshape(-1, 1).split(512), far.reshape(-1, 1).split(512)
    outs = []
    with torch.no_grad():
        for ob, db, nb, fb in zip(o, d, nr, fr):
            r = ren.render(ob, db, nb, fb, color_maps=kw["color_maps"], w2cs=kw["w2cs"], intrinsics=kw["intrinsics"],
                           query_c2w=scan.pose_all[idx], cos_anneal_ratio=ratio)
            S = r["gradients_flip"].shape[1]
            outs.append([r["color"].cpu().numpy(), r["color_pixel"].cpu().numpy(), r["depth"].cpu().numpy(),
                         (r["gradients_flip"] * r["weights"][:, :S, None] * r["inside_sphere"][..., None]).sum(1).cpu().numpy()])
    return outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", type=int, nargs="+", default=[4, 1])
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    from neuraludf_b200 import _lib, render as R
    from neuraludf_b200.models.udf_renderer_blending import UDFRendererBlending
    from tests.runner_env import write_synthetic_dtu
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    dev = torch.device("cuda", 0)
    udf, col, nerf, var, beta = modules(dev)
    ren = UDFRendererBlending(nerf, udf, var, col, beta, n_samples=64, n_importance=50, n_outside=32, up_sample_steps=5,
                              perturb=0.0)
    tmp = tempfile.mkdtemp()
    scan = R.load_scan(write_synthetic_dtu(tmp, n_images=9, width=1600, height=1200), device=dev)
    idx, ratio = 0, 0.5
    cm, w2, it = scan.source_info(idx)
    kw = dict(color_maps=cm, w2cs=w2, intrinsics=it)
    rot = np.linalg.inv(scan.pose_all[idx, :3, :3].cpu().numpy())
    L = _lib.lib()
    results = []
    for level in a.levels:
        rays_o, rays_d, near, far = scan.rays_at(idx, level)
        view = lambda: {k: v.cpu() for k, v in R.render_view(ren, rays_o, rays_d, near, far, rot=rot,
                                                                cos_anneal_ratio=ratio, **kw).items()}
        view()
        runner_loop(ren, scan, idx, level, kw, ratio)                       # warm-up of both
        tv, tr = [], []
        for _ in range(a.reps):                                              # alternating
            torch.cuda.synchronize(); t0 = time.perf_counter(); view(); torch.cuda.synchronize()
            tv.append(time.perf_counter() - t0)
            torch.cuda.synchronize(); t0 = time.perf_counter(); runner_loop(ren, scan, idx, level, kw, ratio)
            torch.cuda.synchronize(); tr.append(time.perf_counter() - t0)
        n_rays = rays_o.shape[0] * rays_o.shape[1]
        torch.cuda.reset_peak_memory_stats(); base = torch.cuda.memory_allocated()
        c0 = L.nudf_launch_count(); view(); torch.cuda.synchronize(); launches = L.nudf_launch_count() - c0
        peak_view = torch.cuda.max_memory_allocated() - base
        torch.cuda.reset_peak_memory_stats(); base = torch.cuda.memory_allocated()
        c0 = L.nudf_launch_count(); runner_loop(ren, scan, idx, level, kw, ratio); launches_r = L.nudf_launch_count() - c0
        peak_runner = torch.cuda.max_memory_allocated() - base
        # kernel time of nudf_render_view_forward, from a profiled view of its own
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            view(); torch.cuda.synchronize()
        kt = sum(e.device_time_total for e in prof.key_averages() if "view_forward_kernel" in e.key)
        res = dict(level=level, rays=n_rays, gpu=smi, render_view_s=min(tv), runner_loop_s=min(tr),
                   render_view_rays_per_s=n_rays / min(tv), runner_rays_per_s=n_rays / min(tr), speedup=min(tr) / min(tv),
                   render_view_s_all=tv, runner_loop_s_all=tr, peak_bytes_render_view=peak_view,
                   peak_bytes_runner=peak_runner, libnudf_launches_render_view=launches,
                   libnudf_launches_runner=launches_r, view_kernel_us=kt)
        print(json.dumps(res), flush=True)
        results.append(res)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()

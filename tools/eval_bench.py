"""Point-cloud evaluation timing at DTU scale: one JSON line.

    python tools/eval_bench.py [--faces 770000] [--gt 2000000] [--repeats 3] [--no-reference]

Inputs: a UV sphere of radius 100 mm with ~770 k faces (a 512^3 reconstruction's face count), sampled at the DTU density
0.2 mm, and a 2 M-point GT cloud around it (noisy surface, 5 % off-surface, 1 % beyond max_dist).  Reported: the device
name and power limit read in the same run, milliseconds per stage (CUDA events, median of the repeats after one warm-up:
sample = sample_mesh, downsample, d2s / s2d = nearest_distance of the DTU protocol's two directions, eval_dtu = the whole
protocol), point counts and the downsampling rounds; and -- unless --no-reference, when the reference's scripts are staged
(oracle/ref_eval.py) -- the wall time of the reference's `eval_cloud` on the host for the same inputs.  Writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30)
        return out.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--faces", type=int, default=770_000)
    ap.add_argument("--gt", type=int, default=2_000_000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("eval_bench needs a CUDA device")
    from neuraludf_b200 import evaluate as E
    from oracle import ref_eval
    from tests.proto import eval_cases as C
    dev = torch.device("cuda", 0)
    n = int(round((args.faces / 2) ** 0.5))
    v, f = C.uv_sphere(100.0, n, n)
    rng = np.random.default_rng(0)
    m = args.gt
    gt = np.concatenate([C.sphere_points(rng, m - m // 20 - m // 100, 100.0, noise=0.2),
                         C.sphere_points(rng, m // 20, 104.0), C.sphere_points(rng, m // 100, 140.0)])
    bb = np.array([[-110.0, -110.0, -110.0], [110.0, 110.0, 110.0]])
    res = np.array([[2.0]])
    obs = np.ones((111, 111, 111), np.uint8)
    plane = np.array([[0.0, 0.0, 1.0, 80.0]])
    vd, fd, gd = (torch.from_numpy(a).to(dev) for a in (v, f, gt))
    out = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "faces": int(len(f)), "gt_points": int(m),
           "density_mm": 0.2, "max_dist_mm": 20.0}
    runs = []
    for rep in range(args.repeats + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
        ev[0].record()
        pcd = E.sample_mesh(vd, fd, 0.2)
        ev[1].record()
        down, info = E.downsample(pcd, 0.2, seed=0)
        ev[2].record()
        d2s = E.nearest_distance(down, gd, 20.0)
        ev[3].record()
        s2d = E.nearest_distance(gd, down, 20.0)
        ev[4].record()
        r = E.eval_dtu(vd, fd, gd, obs, bb, res, plane, seed=0)
        ev[5].record()
        torch.cuda.synchronize()
        if rep:
            runs.append([ev[i].elapsed_time(ev[i + 1]) for i in range(5)])
    ms = np.median(np.array(runs), axis=0)
    out["ms"] = dict(zip(["sample", "downsample", "d2s", "s2d", "eval_dtu"], [round(float(x), 2) for x in ms]))
    out.update(points=int(pcd.shape[0]), kept=int(down.shape[0]), downsample_rounds=info["rounds"], edges=info["edges"],
               s2d_beyond_max=int(torch.isinf(s2d).sum()), over_all=r["over_all"])
    if not args.no_reference and (ref_eval.verify() or ref_eval.stage(verbose=False) is not None):
        t = time.perf_counter()
        rec = ref_eval.run_dtu(v, f, gt, obs, bb, res, plane, seed=0)
        out["reference_eval_cloud_s"] = round(time.perf_counter() - t, 1)
        out["reference_cpu_count"] = os.cpu_count()
        out["reference_over_all"] = rec["over_all"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()

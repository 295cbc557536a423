"""Timing of camera visibility and colour (paint.surface_views / point_colors) on the C5 test network: clouds of 10^6 and
4 10^6 points from 512^3 / 1024^3 lattices (cloud.udf_point_cloud), 49 cameras on a DTU-like cap.  Reports ms per stage,
udf evaluations per point, the histogram of trace lengths, pairs traced per second, the unseen / undecided counts and
peak memory.  Prints one JSON line per case; with --out it also writes them, with the card's name and limits, to a file.

    python tools/paint_bench.py [--cases 512:1000000 1024:4000000] [--out path]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

H, W, FOCAL = 1200, 1600, 2900.0             # DTU's image size and roughly its focal length in pixels


def c5():
    from neuraludf_b200 import synthetic as S
    from neuraludf_b200.models import fields as F
    udf = F.UDFNetwork(d_in=3, d_out=257, d_hidden=256, n_layers=8, skip_in=(4,), multires=6, bias=0.5, scale=1.0,
                       geometric_init=True, weight_norm=True, udf_type="abs")
    udf.load_state_dict(S.make_udf_params(S.udf_cfg(), 0))
    col = F.ResidualRenderingNetwork(d_feature=256, mode="no_normal", d_in=6, d_out=3, d_hidden=128, n_layers=4,
                                     weight_norm=True, multires_view=4, squeeze_out=True, blending_cand_views=10)
    col.load_state_dict(S.make_color_params(S.color_cfg(), 1))
    return udf.cuda(), col.cuda()


def cameras(n=49):
    """n cameras 2.5 units from the origin on a cap of polar angle up to 60 degrees, looking at it (tests/proto/udf_paint)"""
    from tests.proto import udf_paint as P
    intr, poses = P.cameras(P.cap_centres(n, max_polar=np.pi / 3, seed=0), H, W, FOCAL)
    return intr, poses


def run(udf, col, N, n_points):
    from neuraludf_b200 import cloud, paint
    intr, poses = cameras()
    mats, centres = paint.camera_matrices(torch.from_numpy(intr), torch.from_numpy(poses), torch.device("cuda"))
    pts = cloud.udf_point_cloud(udf, N, n_points)
    images = torch.rand(len(poses), H, W, 3, device="cuda")
    voxel = 2.0 / (N - 1)
    out = dict(N=N, points=int(pts.shape[0]), cameras=len(poses))
    for rep in range(2):                    # the first pass warms up every shape
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
        ev[0].record()
        ninfo, vinfo = {}, {}
        n = paint.point_normals(udf, pts, info=ninfo)
        ev[1].record()
        view, n = paint.surface_views(udf, pts, n, mats, centres, H, W, voxel, info=vinfo)
        ev[2].record()
        paint.point_colors(pts, view, n, "image", images=images, mats=mats)
        ev[3].record()
        paint.point_colors(pts, view, n, "network", centres=centres, udf_network=udf, color_network=col)
        ev[4].record()
        torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in zip(ev, ev[1:])]
    lengths = {}
    for r in vinfo["rounds"]:
        prev = r["traced"]
        for s, a in enumerate(r["active"], 1):
            lengths[s] = lengths.get(s, 0) + prev - a      # pairs that ended at step s
            prev = a
    pairs = sum(r["traced"] for r in vinfo["rounds"])
    stages = dict(normals=ms[0], views=ms[1], image_colors=ms[2], network_colors=ms[3])
    stages.update({"views." + k: v for k, v in vinfo["ms"].items()})
    out.update(ms=stages,
               zero_normals=ninfo["zero"], no_candidate=vinfo["no_candidate"], seen=vinfo["seen"],
               unseen=out["points"] - vinfo["seen"], undecided=vinfo["undecided"],
               rounds=[dict(traced=r["traced"], visible=r["visible"], steps=len(r["active"])) for r in vinfo["rounds"]],
               pairs=pairs, evaluations=vinfo["evaluations"],
               evaluations_per_point=vinfo["evaluations"] / max(out["points"], 1),
               trace_length_histogram=dict(sorted(lengths.items())), pairs_per_s=pairs / (ms[1] / 1e3),
               evaluations_per_s=vinfo["evaluations"] / (vinfo["ms"]["trace"] / 1e3),
               peak_gb_over_cloud=(torch.cuda.max_memory_allocated() - base) / 2 ** 30)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", nargs="*", default=["512:1000000", "1024:4000000"])
    ap.add_argument("--out", default=None, help="also write the results to this JSON file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("paint_bench measures on a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    udf, col = c5()
    res = dict(gpu=gpu, cases=[])
    for c in a.cases:
        N, n = (int(x) for x in c.split(":"))
        r = run(udf, col, N, n)
        print(json.dumps(r))
        res["cases"].append(r)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(gpu)


if __name__ == "__main__":
    main()

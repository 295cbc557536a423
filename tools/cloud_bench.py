"""Surface point cloud timing, counts and memory on the C5 synthetic UDF network: one JSON line.

    python tools/cloud_bench.py [--sizes 512 1024 2048] [--points 1048576 4194304] [--repeats 2] [--residual 512 1024]

Reported with the device name and power limit read in the same run.  Per lattice size N and target count, for
cloud.udf_point_cloud with its defaults (5 steps, ratio 1, Lipschitz 2, batches of 2^20): milliseconds per stage (band,
seeds, projection, filter, densify; CUDA events, median of the repeats after one warm-up), point-steps (value_gradient
evaluations) per second over the projection stage, seeds, survivors after each step, kept after the filter, densify
rounds, and the peak torch.cuda.max_memory_allocated of the call beside N^3 bytes.  With --residual: the udf at the
projected seeds after each of 0 .. 8 steps (median, 99th percentile, max, in voxels, and the share below one voxel) and
the points each step drops, by reason (non-finite u or g; |g| = 0 with u = 0; |g| = 0 with u > 0; leaving the box): what
the default step count is chosen from.  Requires a CUDA device; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def c5_network():
    from neuraludf_b200 import synthetic as S
    from neuraludf_b200.models.fields import UDFNetwork
    net = UDFNetwork(d_in=3, d_out=257, d_hidden=256, n_layers=8, skip_in=(4,), multires=6, bias=0.5, scale=1.0,
                     geometric_init=True, weight_norm=True, udf_type="abs")
    net.load_state_dict(S.make_udf_params(S.udf_cfg(), 0))
    return net.cuda()


def run(net, N, n_points):
    """one udf_point_cloud call: (info, peak bytes above what was allocated before it)"""
    import torch
    from neuraludf_b200 import cloud
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    info = {}
    pts = cloud.udf_point_cloud(net, N, n_points, info=info)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    del pts
    return info, peak


def dropped(net, pts, max_batch):
    """the points one projection step drops, by reason, restated in torch from the chain's (u, g) (the kernel's order)"""
    import torch
    out = dict(nonfinite=0, zero_grad_zero_u=0, zero_grad=0, box=0)
    for i in range(0, pts.shape[0], max_batch):
        p = pts[i:i + max_batch]
        u, g = net.value_gradient(p)
        fin = torch.isfinite(u) & torch.isfinite(g).all(1)
        n = torch.sqrt((g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]) + g[:, 2] * g[:, 2])
        q = p - (u / n)[:, None] * g
        out["nonfinite"] += int((~fin).sum())
        out["zero_grad_zero_u"] += int((fin & (n == 0) & (u == 0)).sum())
        out["zero_grad"] += int((fin & (n == 0) & (u != 0)).sum())
        out["box"] += int((fin & (n != 0) & ~((q >= -1) & (q <= 1)).all(1)).sum())
    return out


def residual(net, N, max_steps=8, max_batch=1 << 20):
    """udf statistics (in voxels) at the projected seeds after 0 .. max_steps steps"""
    import torch
    from neuraludf_b200 import cloud, grid
    h = 2.0 / (N - 1)
    with torch.no_grad():
        band, _ = grid.udf_band_sparse(net, N, max_batch=max_batch)
        pts = grid._index_points(grid.near_surface_indices_sparse(band), N)
        del band
        rows = []
        for k in range(max_steps + 1):
            drops = None
            if k:
                drops = dropped(net, pts, max_batch)
                pts, _ = cloud._project(net, pts, 1, max_batch)
            u = torch.cat([net.udf_values(pts[i:i + max_batch]) for i in range(0, pts.shape[0], max_batch)]).double() / h
            q = torch.quantile(u[torch.randperm(u.numel(), device=u.device)[:1 << 24]], torch.tensor(
                [0.5, 0.99], dtype=torch.float64, device=u.device)).tolist()
            rows.append(dict(steps=k, points=int(u.numel()), median=round(q[0], 4), p99=round(q[1], 4),
                             max=round(float(u.max()), 4), below_1=round(float((u < 1.0).double().mean()), 5),
                             dropped=drops))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[512, 1024, 2048])
    ap.add_argument("--points", type=int, nargs="+", default=[1 << 20, 1 << 22])
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--residual", type=int, nargs="*", default=[512, 1024])
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("cloud_bench needs a CUDA device")
    from tools.eval_bench import power_limit
    net = c5_network()
    out = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "scene": "C5 synthetic UDF network",
           "sizes": {}, "residual": {}}
    r3 = lambda x: round(float(x), 3)
    for N in args.residual:
        out["residual"][str(N)] = residual(net, N)
        print(json.dumps({"residual": {str(N): out["residual"][str(N)]}}), file=sys.stderr, flush=True)
    for N in args.sizes:
        rec = {}
        for n in args.points:
            runs, peaks = [], []
            for rep in range(args.repeats + 1):
                info, peak = run(net, N, n)
                if rep:
                    runs.append([info["ms"][k] for k in ("band", "seeds", "projection", "filter", "densify")])
                peaks.append(peak)
            med = np.median(np.array(runs), axis=0)
            point_steps = info["seeds"] + sum(info["steps"][:-1])
            rec[str(n)] = {"ms": dict(zip(["band", "seeds", "projection", "filter", "densify"], [r3(x) for x in med])),
                           "total_ms": r3(med.sum()), "projection_point_steps_per_s": r3(point_steps / (med[2] / 1e3)),
                           "seeds": info["seeds"], "steps": info["steps"], "filtered": info["filtered"],
                           "rounds": info["rounds"], "points": info["points"], "truncated": info["truncated"],
                           "peak_gb": r3(max(peaks) / 1e9), "n3_bytes_gb": r3(N ** 3 / 1e9),
                           "band_points": info["band"]["points"], "bricks": info["band"]["bricks"]}
            print(json.dumps({str(N): {str(n): rec[str(n)]}}), file=sys.stderr, flush=True)
        out["sizes"][str(N)] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Narrow-band meshing timing on the C5 scene (the golden UDF network): one JSON line.

    python tools/mesh_band_bench.py [--sizes 256 512 1024] [--dense 256 512] [--repeats 3]

Reported with the device name and power limit read in the same run.  Per lattice size, for the default stride schedule
(grid.default_strides) and a few alternatives: milliseconds per level of grid.udf_band (level 0 = the coarsest
sub-lattice; level k = the block test at the previous stride, point emission and evaluation), points evaluated per level
and in total as a fraction of N^3, kept blocks per level, and max_edge_slope.  For the default schedule also: normals
(grid.near_surface_cells), MC and filter milliseconds, the whole udf_mesh_band, and, at the --dense sizes, the whole dense
udf_mesh with a check that both give the same mesh.  CUDA events, median of the repeats after one warm-up.  Requires a CUDA
device; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def schedules(N):
    from neuraludf_b200 import grid
    d = grid.default_strides(N)
    out = {"default": d, "halving_from_2x": [2 * d[0]] + d, "halving_from_half": d[1:] or d}
    s, q = 1, []
    while 4 * s <= d[0]:
        s *= 4
    while s >= 1:
        q.append(s)
        s //= 4
    out["quartering"] = q
    return out


def timed(fn, repeats):
    import numpy as np
    import torch
    runs, res = [], None
    for rep in range(repeats + 1):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        res = fn()
        b.record()
        torch.cuda.synchronize()
        if rep:
            runs.append(a.elapsed_time(b))
    return float(np.median(runs)), res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[256, 512, 1024])
    ap.add_argument("--dense", type=int, nargs="*", default=[256, 512])
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("mesh_band_bench needs a CUDA device")
    from neuraludf_b200 import grid, mesh
    from tests.golden_util import load_golden
    from tests.gpu_util import build_modules
    from tools.eval_bench import power_limit
    udf = build_modules(load_golden(), "cuda")[0]
    out = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "scene": "C5 golden UDF network",
           "sizes": {}}
    r3 = lambda x: round(float(x), 3)
    for N in args.sizes:
        rec = {"schedules": {}}
        for name, strides in schedules(N).items():
            level_runs = []
            for rep in range(args.repeats + 1):
                df, info = grid.udf_band(udf, N, strides=strides)
                if rep:
                    level_runs.append(info["level_ms"] + [info["slope_ms"]])
                del df
            lv = np.median(np.array(level_runs), axis=0)
            whole = np.median(np.array(level_runs).sum(1))
            rec["schedules"][name] = {
                "strides": strides, "udf_band_ms": r3(whole), "level_ms": [r3(x) for x in lv[:-1]],
                "slope_pass_ms": r3(lv[-1]), "points": info["points"], "fraction": float("%.5f" % (sum(info["points"]) / N ** 3)),
                "kept_blocks": info["kept_blocks"], "max_edge_slope": r3(info["max_edge_slope"])}
        torch.cuda.empty_cache()
        # stages after the band, default schedule
        voxel = 2.0 / (N - 1)
        df, _ = grid.udf_band(udf, N)
        stage = []
        for rep in range(args.repeats + 1):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            ev[0].record()
            idx, nrm = grid.near_surface_cells(udf, N, df)
            ev[1].record()
            v, f, _ = mesh.marching_cubes_index(df, (N, N, N), nrm, idx)
            v = v * voxel - 1.0
            ev[2].record()
            vd = udf.udf_values(v).reshape(-1)
            vf, ff = mesh._compact(v, f[vd[f].max(dim=1).values < voxel])
            ev[3].record()
            torch.cuda.synchronize()
            if rep:
                stage.append([ev[i].elapsed_time(ev[i + 1]) for i in range(3)])
        rec["ms"] = dict(zip(["normals", "mc", "filter"], [r3(x) for x in np.median(np.array(stage), axis=0)]))
        rec.update(raw_faces=int(f.shape[0]), faces=int(ff.shape[0]), vertices=int(vf.shape[0]))
        del df, idx, nrm, v, f, vd, vf, ff
        torch.cuda.empty_cache()
        ms, (vb, fb) = timed(lambda: mesh.udf_mesh_band(udf, N), args.repeats)
        rec["udf_mesh_band_ms"] = r3(ms)
        if N in args.dense:
            ms, (vd_, fd_) = timed(lambda: mesh.udf_mesh(udf, N), args.repeats)
            rec["udf_mesh_dense_ms"] = r3(ms)
            rec["same_mesh_as_dense"] = bool(torch.equal(vb, vd_) and torch.equal(fb, fd_))
            del vd_, fd_
        del vb, fb
        torch.cuda.empty_cache()
        out["sizes"][str(N)] = rec
        print(json.dumps({str(N): rec}), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Block-sparse narrow-band meshing timing and memory on the C5 scene (the golden UDF network): one JSON line.

    python tools/mesh_sparse_bench.py [--sizes 512 1024 2048] [--band 512 1024] [--repeats 2]

Reported with the device name and power limit read in the same run.  Per lattice size, for udf_mesh_sparse's stages
(grid.udf_band_sparse, grid.near_surface_cells_sparse, mesh.marching_cubes_sparse, the vertex filter) and, at the --band
sizes, udf_mesh_band's (grid.udf_band, grid.near_surface_cells, mesh.marching_cubes_index, the filter): milliseconds per
stage (CUDA events, median of the repeats after one warm-up) and the peak torch.cuda.max_memory_allocated of the whole
run, split into the value chain's batch workspace (the peak a 2^21-point udf_values batch or a 2^20-point gradient batch
adds on its own) and everything else.  Also the store's bytes (coarse array, brick directory, bricks, the largest
block-test flags) and its brick count.  Requires a CUDA device; writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

MAX_BATCH = 1 << 21


def workspace(udf):
    import torch
    g = torch.Generator(device="cpu").manual_seed(0)
    ws = 0
    for fn, n in ((udf.udf_values, MAX_BATCH), (udf.gradient, MAX_BATCH // 2)):
        pts = (torch.rand(n, 3, generator=g) * 2 - 1).cuda()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        with torch.no_grad():
            out = fn(pts)
        torch.cuda.synchronize()
        ws = max(ws, torch.cuda.max_memory_allocated() - base)
        del pts, out
    return ws


def run(udf, N, sparse):
    """one udf_mesh_sparse (or udf_mesh_band) run by stages: (ms per stage, peak bytes, faces, band info)"""
    import torch
    from neuraludf_b200 import grid, mesh
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    ev[0].record()
    if sparse:
        band, info = grid.udf_band_sparse(udf, N, max_batch=MAX_BATCH)
        ev[1].record()
        idx, nrm = grid.near_surface_cells_sparse(udf, band, max_batch=MAX_BATCH // 2)
        ev[2].record()
        v, f, _ = mesh.marching_cubes_sparse(band, nrm, idx)
        del band
    else:
        df, info = grid.udf_band(udf, N, max_batch=MAX_BATCH)
        ev[1].record()
        idx, nrm = grid.near_surface_cells(udf, N, df, max_batch=MAX_BATCH // 2)
        ev[2].record()
        v, f, _ = mesh.marching_cubes_index(df, (N, N, N), nrm, idx)
        del df
    del idx, nrm
    ev[3].record()
    vf, ff = mesh._vertex_filter(udf, N, v, f, 1.0, 0, MAX_BATCH if sparse else None)   # as udf_mesh_sparse / udf_mesh_band
    ev[4].record()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    ms = [ev[i].elapsed_time(ev[i + 1]) for i in range(4)]
    return ms, peak, int(ff.shape[0]), info


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[512, 1024, 2048])
    ap.add_argument("--band", type=int, nargs="*", default=[512, 1024])
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("mesh_sparse_bench needs a CUDA device")
    from tests.golden_util import load_golden
    from tests.gpu_util import build_modules
    from tools.eval_bench import power_limit
    udf = build_modules(load_golden(), "cuda")[0]
    ws = workspace(udf)
    out = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "scene": "C5 golden UDF network",
           "workspace_gb": round(ws / 1e9, 3), "sizes": {}}
    r3 = lambda x: round(float(x), 3)
    for N in args.sizes:
        rec = {}
        for name, sparse in (("udf_mesh_sparse", True), ("udf_mesh_band", False)):
            if not sparse and N not in args.band:
                continue
            runs, peaks = [], []
            for rep in range(args.repeats + 1):
                ms, peak, faces, info = run(udf, N, sparse)
                if rep:
                    runs.append(ms)
                peaks.append(peak)
            med = np.median(np.array(runs), axis=0)
            r = {"ms": dict(zip(["band", "normals", "mc", "filter"], [r3(x) for x in med])), "total_ms": r3(med.sum()),
                 "peak_gb": r3(max(peaks) / 1e9), "rest_gb": r3((max(peaks) - ws) / 1e9), "faces": faces,
                 "points": info["points"]}
            if sparse:
                r.update(bricks=info["bricks"], store_gb={k: r3(v / 1e9) for k, v in info["bytes"].items()},
                         rest_below_n3_bytes=bool(max(peaks) - ws < N ** 3))
            rec[name] = r
            torch.cuda.empty_cache()
        out["sizes"][str(N)] = rec
        print(json.dumps({str(N): rec}), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

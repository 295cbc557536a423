"""Block-sparse threshold meshing timing and memory on the C5 scene (the golden UDF network), as the runner's
validate_mesh runs it with NUDF_BAND_MESH=sparse: one JSON line.

    python tools/iso_sparse_bench.py [--sizes 512 1024 2048] [--band-sizes 512 1024] [--level 0.005] [--repeats 3]

Per lattice size on the box +-1.01: milliseconds of each band level (grid.iso_band_sparse's level_ms) and the points
evaluated; of the stages of mesh.iso_marching_cubes_sparse (CUDA events): the active-cell enumeration from the store
(count, scan, emit, sort), count + scan, emit, weld (unique) and vertices; the whole mesh.iso_mesh_sparse (host clock
after a synchronise); its peak max_memory_allocated above the start; the store's bytes and bricks.  For --band-sizes the
whole mesh.iso_mesh_band and its peak in the same run, and whether the two meshes are bit-identical.  Median of the
repeats after one warm-up.  Also the GPU name, power limit and SM clocks, read in one nvidia-smi call in the same run.
Requires a CUDA device; writes nothing.
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


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _timed(fn):
    import torch
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, 1e3 * (time.perf_counter() - t), torch.cuda.max_memory_allocated() - base


def _stages(band, level):
    """iso_marching_cubes_sparse's stages, CUDA-event milliseconds: (ms dict, faces)"""
    import torch
    from neuraludf_b200 import _lib, mesh
    from neuraludf_b200._lib import check, ptr
    L, st, dev = _lib.lib(), _lib.stream_ptr(), band.device
    ev = []

    def mark():
        ev.append(torch.cuda.Event(enable_timing=True))
        ev[-1].record()
    lat = band.lattice()
    mark()
    cells = mesh.iso_active_cells(band, level)
    mark()
    n = cells.numel()
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    check(L.nudf_iso_lat_count(lat, level, ptr(cells), n, ptr(counts), st), "nudf_iso_lat_count")
    csum = torch.cumsum(counts, 0, dtype=torch.int64)
    offsets = (csum - counts).contiguous()
    n_faces = int(csum[-1])
    mark()
    keys = torch.empty(3 * n_faces, dtype=torch.int64, device=dev)
    check(L.nudf_iso_lat_emit(lat, level, ptr(cells), n, ptr(offsets), ptr(keys), st), "nudf_iso_lat_emit")
    mark()
    ukeys, inv = torch.unique(keys, sorted=True, return_inverse=True)
    ukeys = ukeys.contiguous()
    mark()
    verts = torch.empty(ukeys.numel(), 3, dtype=torch.float64, device=dev)
    check(L.nudf_iso_lat_vertices(lat, level, ptr(cells), n, ptr(ukeys), ukeys.numel(), ptr(verts), st),
          "nudf_iso_lat_vertices")
    mark()
    torch.cuda.synchronize()
    names = ("enumerate", "count", "emit", "weld", "vertices")
    return {k: ev[i].elapsed_time(ev[i + 1]) for i, k in enumerate(names)}, n_faces, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[512, 1024, 2048])
    ap.add_argument("--band-sizes", type=int, nargs="*", default=[512, 1024])
    ap.add_argument("--level", type=float, default=0.005)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("iso_sparse_bench needs a CUDA device")
    from neuraludf_b200 import grid, mesh
    from tests.golden_util import load_golden
    from tests.gpu_util import build_modules
    udf = build_modules(load_golden(), "cuda")[0]
    query = lambda p: udf.udf_values(p)     # noqa: E731  (the renderer's extract_geometry query)
    bmin, bmax = torch.tensor([-1.01] * 3), torch.tensor([1.01] * 3)
    level = float(np.float32(args.level))
    out = {"device": torch.cuda.get_device_name(0), "gpu": _gpu_info(), "scene": "C5 golden UDF network", "level": level,
           "runs": []}
    for N in args.sizes:
        reps = []
        for _ in range(args.repeats + 1):
            (v, f, info), ms, peak = _timed(lambda: mesh.iso_mesh_sparse(query, bmin, bmax, N, level))
            reps.append((ms, peak, info["band"]))
            del v, f, info
        reps = reps[1:]
        b = reps[-1][2]
        band, _ = grid.iso_band_sparse(query, bmin, bmax, N, level)
        st = [_stages(band, level) for _ in range(args.repeats + 1)][1:]
        del band
        run = {"N": N, "sparse_ms": float(np.median([r[0] for r in reps])), "sparse_peak_gb": max(r[1] for r in reps) / 1e9,
               "level_ms": [float(np.median([r[2]["level_ms"][k] for r in reps])) for k in range(len(b["level_ms"]))],
               "points": b["points"], "evaluated": sum(b["points"]) / N ** 3, "bricks": b["bricks"],
               "store_gb": sum(b["bytes"].values()) / 1e9, "bytes": b["bytes"],
               "stage_ms": {k: float(np.median([s[0][k] for s in st])) for k in st[0][0]},
               "active_cells": st[0][2], "faces": st[0][1], "r3_gb": N ** 3 / 1e9}
        if N in args.band_sizes:
            breps = [_timed(lambda: mesh.iso_mesh_band(query, bmin, bmax, N, level)) for _ in range(args.repeats + 1)][1:]
            (v0, f0, _), _, _ = breps[-1]
            v1, f1, _ = mesh.iso_mesh_sparse(query, bmin, bmax, N, level)
            run.update(band_ms=float(np.median([r[1] for r in breps])), band_peak_gb=max(r[2] for r in breps) / 1e9,
                       same_mesh=bool(torch.equal(f0, f1) and torch.equal(v0.view(torch.int64), v1.view(torch.int64))))
            del breps, v0, f0, v1, f1
        out["runs"].append(run)
        print(json.dumps(run), file=sys.stderr, flush=True)
    out["gpu_after"] = _gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

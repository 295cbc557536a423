"""Threshold meshing timing on the C5 scene (the golden UDF network), as the runner's validate_mesh runs it: one JSON line.

    python tools/iso_mesh_bench.py [--sizes 256 512] [--thresholds 0.005 0.02] [--repeats 3] [--host-sizes 256]

Per lattice size (the +-1.01 box of validate_mesh without cameras): milliseconds of the lattice query
(udf_renderer_blending._grid_query_device, 64^3 blocks), and per threshold of each MC stage (active = nudf_iso_active +
nonzero, count = nudf_iso_count + cumsum, emit = nudf_iso_emit, weld = unique, vertices = nudf_iso_vertices) and of the
whole `extract_geometry` on the device path (lattice query, MC, host copy and the runner's vertex mapping); CUDA events or
a host clock after a synchronise, median of the repeats after one warm-up.  Also the GPU name and power limit, read in the
same process, and for --host-sizes the host time of the NumPy restatement (tests/proto/iso_mc.py, one run) -- labelled as
such: it is not PyMCubes, which is not installed and not measured.  Requires a CUDA device; writes nothing.
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
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _stages(df, N, level):
    """iso_marching_cubes_index's stages, each bracketed by CUDA events: (ms per stage, active cells, vertices, faces)"""
    import ctypes
    import torch
    from neuraludf_b200 import _lib
    from neuraludf_b200._lib import check, ptr
    L, st = _lib.lib(), _lib.stream_ptr()
    lat = ctypes.byref(_lib.Lattice(N, N, N, df.data_ptr(), None))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
    ev[0].record()
    flags = torch.empty(df.numel(), dtype=torch.uint8, device=df.device)
    check(L.nudf_iso_active(lat, level, ptr(flags), st), "nudf_iso_active")
    cells = torch.nonzero(flags).reshape(-1).contiguous()
    n = cells.numel()
    ev[1].record()
    counts = torch.empty(n, dtype=torch.int32, device=df.device)
    check(L.nudf_iso_count(lat, level, ptr(cells), n, ptr(counts), st), "nudf_iso_count")
    csum = torch.cumsum(counts, 0, dtype=torch.int64)
    n_faces = int(csum[-1]) if n else 0
    offsets = (csum - counts).contiguous()
    ev[2].record()
    keys = torch.empty(3 * n_faces, dtype=torch.int64, device=df.device)
    check(L.nudf_iso_emit(lat, level, ptr(cells), n, ptr(offsets), ptr(keys), st), "nudf_iso_emit")
    ev[3].record()
    ukeys, inv = torch.unique(keys, sorted=True, return_inverse=True)
    ukeys = ukeys.contiguous()
    ev[4].record()
    verts = torch.empty(ukeys.numel(), 3, dtype=torch.float64, device=df.device)
    check(L.nudf_iso_vertices(lat, level, ptr(cells), n, ptr(ukeys), ukeys.numel(), ptr(verts), st),
          "nudf_iso_vertices")
    ev[5].record()
    torch.cuda.synchronize()
    return [ev[i].elapsed_time(ev[i + 1]) for i in range(5)], n, int(ukeys.numel()), n_faces


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--thresholds", type=float, nargs="+", default=[0.005, 0.02])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--host-sizes", type=int, nargs="*", default=[256])
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("iso_mesh_bench needs a CUDA device")
    from neuraludf_b200.models import udf_renderer_blending as R
    from tests.golden_util import load_golden
    from tests.gpu_util import build_modules
    from tests.proto import iso_mc as P
    udf = build_modules(load_golden(), "cuda")[0]
    dev = torch.device("cuda", 0)
    query = lambda p: udf.udf_values(p)     # noqa: E731  (the renderer's extract_geometry query)
    bmin = torch.tensor([-1.01] * 3, dtype=torch.float32)
    bmax = torch.tensor([1.01] * 3, dtype=torch.float32)
    saved = sys.modules.get("mcubes", "absent")
    sys.modules["mcubes"] = None            # the device path of extract_geometry, even where PyMCubes is installed
    out = {"device": torch.cuda.get_device_name(0), "gpu": _gpu_info(), "scene": "C5 golden UDF network, box +-1.01",
           "sizes": {}}
    try:
        for N in args.sizes:
            rec = {"levels": {}}
            qms = []
            for rep in range(args.repeats + 1):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                with torch.no_grad():
                    df = R._grid_query_device(bmin, bmax, N, query, dev, 0)
                e1.record()
                torch.cuda.synchronize()
                if rep:
                    qms.append(e0.elapsed_time(e1))
            rec["query_ms"] = round(float(np.median(qms)), 3)
            flat = df.reshape(-1).contiguous()
            for level in args.thresholds:
                runs, whole = [], []
                for rep in range(args.repeats + 1):
                    ms, n, nv, nf = _stages(flat, N, float(np.float32(level)))
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    v, f = R.extract_geometry(bmin, bmax, N, level, query, dev)
                    wt = 1e3 * (time.perf_counter() - t)
                    if rep:
                        runs.append(ms)
                        whole.append(wt)
                med = np.median(np.array(runs), axis=0)
                lv = {"ms": dict(zip(["active", "count", "emit", "weld", "vertices"], [round(float(x), 3) for x in med])),
                      "mc_ms": round(float(med.sum()), 3), "extract_geometry_ms": round(float(np.median(whole)), 1),
                      "active_cells": n, "vertices": nv, "faces": nf}
                if N in args.host_sizes:
                    u = flat.cpu().numpy()
                    t = time.perf_counter()
                    _, pf, _ = P.marching_cubes(u, (N, N, N), level)
                    lv["restatement_host_ms"] = round(1e3 * (time.perf_counter() - t), 1)
                    lv["restatement_equal_faces"] = bool(np.array_equal(pf, f))
                rec["levels"][str(level)] = lv
            out["sizes"][str(N)] = rec
            del df, flat
            torch.cuda.empty_cache()
    finally:
        if saved == "absent":
            sys.modules.pop("mcubes", None)
        else:
            sys.modules["mcubes"] = saved
    print(json.dumps(out))


if __name__ == "__main__":
    main()

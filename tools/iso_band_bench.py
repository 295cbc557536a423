"""Narrow-band threshold meshing timing on the C5 scene (the golden UDF network), as the runner's validate_mesh runs it
with NUDF_BAND_MESH=1: one JSON line.

    python tools/iso_band_bench.py [--sizes 256 512 1024] [--dense-sizes 256 512] [--thresholds 0.005 0.02] [--repeats 3]

Per box (+-1.01, and the non-cubic [-1.01, -0.9, -1.01] .. [1.01, 1.01, 0.95]), lattice size and threshold: milliseconds of
each band level (grid.iso_band's level_ms: level 0 the coarse lattice, level k the block test, emission and evaluation of
stride k) and the fraction of the lattice evaluated; the MC of the band lattice (mesh.iso_marching_cubes_index, CUDA
events); the whole band `extract_geometry` (band lattice, MC, host copy and the runner's vertex mapping; host clock after a
synchronise) and, for --dense-sizes, the whole dense `extract_geometry` in the same run; peak max_memory_allocated of the
band path.  Median of the repeats after one warm-up.  Also the GPU name, power limit and SM clock, read in one nvidia-smi
call.  Requires a CUDA device; writes nothing.
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

BOXES = {"cube": ([-1.01] * 3, [1.01] * 3), "box": ([-1.01, -0.9, -1.01], [1.01, 1.01, 0.95])}


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def _timed(fn):
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, 1e3 * (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[256, 512, 1024])
    ap.add_argument("--dense-sizes", type=int, nargs="*", default=[256, 512])
    ap.add_argument("--thresholds", type=float, nargs="+", default=[0.005, 0.02])
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("iso_band_bench needs a CUDA device")
    from neuraludf_b200 import grid, mesh
    from neuraludf_b200.models import udf_renderer_blending as R
    from tests.golden_util import load_golden
    from tests.gpu_util import build_modules
    udf = build_modules(load_golden(), "cuda")[0]
    dev = torch.device("cuda", 0)
    query = lambda p: udf.udf_values(p)     # noqa: E731  (the renderer's extract_geometry query)
    saved_mc, saved_env = sys.modules.get("mcubes", "absent"), os.environ.get("NUDF_BAND_MESH")
    sys.modules["mcubes"] = None            # the device path of extract_geometry, even where PyMCubes is installed
    out = {"device": torch.cuda.get_device_name(0), "gpu": _gpu_info(), "scene": "C5 golden UDF network", "runs": []}

    def geometry(bmin, bmax, N, level, band):
        os.environ["NUDF_BAND_MESH"] = "1" if band else "0"
        return R.extract_geometry(bmin, bmax, N, level, query, dev)

    try:
        for box, (lo, hi) in BOXES.items():
            bmin, bmax = torch.tensor(lo, dtype=torch.float32), torch.tensor(hi, dtype=torch.float32)
            for N in args.sizes:
                dense_ms = None
                if N in args.dense_sizes:
                    ms = [_timed(lambda: geometry(bmin, bmax, N, args.thresholds[0], False))[1]
                          for _ in range(args.repeats + 1)][1:]
                    dense_ms = float(np.median(ms))
                for level in args.thresholds:
                    lv = float(np.float32(level))
                    torch.cuda.empty_cache()
                    torch.cuda.reset_peak_memory_stats()
                    levels, mc, whole, frac = [], [], [], None
                    for rep in range(args.repeats + 1):
                        df, info = grid.iso_band(query, bmin, bmax, N, lv, device=dev)
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        v, f, _ = mesh.iso_marching_cubes_index(df, (N, N, N), lv)
                        e1.record()
                        torch.cuda.synchronize()
                        n_faces = int(f.shape[0])
                        del df, v, f
                        (gv, gf), wt = _timed(lambda: geometry(bmin, bmax, N, level, True))
                        if rep:
                            levels.append(info["level_ms"] + [info["slope_ms"]])
                            mc.append(e0.elapsed_time(e1))
                            whole.append(wt)
                        frac = sum(info["points"]) / N ** 3
                    rec = {"box": box, "N": N, "level": level, "band_level_ms": [round(float(x), 2) for x in
                                                                                 np.median(np.array(levels), axis=0)],
                           "points": info["points"], "fraction_evaluated": round(frac, 5), "tau": info["tau"],
                           "mc_ms": round(float(np.median(mc)), 2), "band_extract_geometry_ms": round(float(np.median(whole)), 1),
                           "faces": n_faces, "peak_gb": round(torch.cuda.max_memory_allocated() / 1e9, 3)}
                    if dense_ms is not None:
                        rec["dense_extract_geometry_ms"] = round(dense_ms, 1)
                        rec["speedup"] = round(dense_ms / rec["band_extract_geometry_ms"], 2)
                    out["runs"].append(rec)
                    print(json.dumps(rec), file=sys.stderr, flush=True)
    finally:
        if saved_mc == "absent":
            sys.modules.pop("mcubes", None)
        else:
            sys.modules["mcubes"] = saved_mc
        if saved_env is None:
            os.environ.pop("NUDF_BAND_MESH", None)
        else:
            os.environ["NUDF_BAND_MESH"] = saved_env
    print(json.dumps(out))


if __name__ == "__main__":
    main()

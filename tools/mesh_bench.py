"""Mesh extraction timing on the C5 scene (the golden UDF network): one JSON line.

    python tools/mesh_bench.py [--sizes 256 512] [--repeats 3]

Per lattice size: milliseconds per stage (grid = grid.udf_grid, normals = grid.near_surface_cells, mc = the CUDA MeshUDF
marching cubes, filter = the vertex filter + compaction; CUDA events, median of the repeats after one warm-up), active
cells, vertices, faces, the polarity union-find's hooking rounds / pointer-jumping passes, and -- when the compiled reference MC is present (oracle/make_ref_mc.py) -- its CPU time on the
same inputs (dense normals, one run).  Requires a CUDA device; writes nothing.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("mesh_bench needs a CUDA device")
    from neuraludf_b200 import grid, mesh
    from oracle import make_ref_mc
    from tests.golden_util import load_golden
    from tests.gpu_util import build_modules
    udf = build_modules(load_golden(), "cuda")[0]
    out = {"device": torch.cuda.get_device_name(0), "scene": "C5 golden UDF network", "sizes": {}}
    for N in args.sizes:
        voxel = 2.0 / (N - 1)
        runs = []
        for rep in range(args.repeats + 1):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
            ev[0].record()
            df = grid.udf_grid(udf, N)
            ev[1].record()
            idx, nrm = grid.near_surface_cells(udf, N, df)
            ev[2].record()
            v, f, info = mesh.marching_cubes_index(df, (N, N, N), nrm, idx)
            v = v * voxel - 1.0
            ev[3].record()
            vd = udf.udf_values(v).reshape(-1)
            vf, ff = mesh._compact(v, f[vd[f].max(dim=1).values < voxel])
            ev[4].record()
            torch.cuda.synchronize()
            if rep:
                runs.append([ev[i].elapsed_time(ev[i + 1]) for i in range(4)])
        ms = np.median(np.array(runs), axis=0)
        rec = {"ms": dict(zip(["grid", "normals", "mc", "filter"], [round(float(x), 3) for x in ms])),
               "active_cells": int(info["active"].numel()), "vertices": int(vf.shape[0]), "faces": int(ff.shape[0]),
               "raw_faces": int(f.shape[0]), "polarity_rounds": info["polarity_rounds"],
               "polarity_jumps": info["polarity_jumps"]}
        if make_ref_mc.verify():
            ref = make_ref_mc.load()
            dense = torch.zeros(N ** 3, 3, device=df.device)
            dense[idx] = nrm
            vol, gr = df.reshape(N, N, N).cpu().numpy(), dense.reshape(N, N, N, 3).cpu().numpy()
            del dense
            t = time.perf_counter()
            rv, rf, _, _ = ref.udf_mc_lewiner(vol, gr, spacing=[voxel] * 3)
            rec["reference_mc_cpu_ms"] = round(1e3 * (time.perf_counter() - t), 1)
            rec["reference_raw_faces"] = int(len(rf))
        out["sizes"][str(N)] = rec
    print(json.dumps(out))


if __name__ == "__main__":
    main()

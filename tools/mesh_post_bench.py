"""Mesh post-processing timing on the C5 scene (the golden UDF network): one JSON line.

    python tools/mesh_post_bench.py [--sizes 512 1024] [--repeats 3]

Reported with the device name and power limit read in the same run.  Per lattice size, the band mesh after the vertex
filter at dist_threshold_ratio 5 (as Runner.extract_udf_mesh calls it) goes through mesh_post.postprocess; the tool
prints the CUDA-event milliseconds of each step (the first process pass: non-finite, merge, duplicate and degenerate faces;
hole filling; the fixed-point loop; border smoothing; the export merge), the whole postprocess, the whole udf_mesh_post,
and what each step changed.  Median of the repeats after one warm-up.  `restatement_host_ms` is the NumPy restatement
(tests/proto/mesh_post.py) on one host thread for the same input, checked to give the same bits: it is not trimesh's time,
which cannot be measured here.  Requires a CUDA device; writes nothing.
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
    ap.add_argument("--sizes", type=int, nargs="+", default=[512, 1024])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--ratio", type=float, default=5.0)
    args = ap.parse_args()
    import numpy as np
    import torch
    if not torch.cuda.is_available():
        sys.exit("mesh_post_bench needs a CUDA device")
    from neuraludf_b200 import grid, mesh, mesh_post
    from tests.golden_util import load_golden
    from tests.gpu_util import build_modules
    from tests.proto import mesh_post as P
    from tools.eval_bench import power_limit
    from tools.mesh_band_bench import timed
    udf = build_modules(load_golden(), "cuda")[0]
    out = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "scene": "C5 golden UDF network",
           "dist_threshold_ratio": args.ratio, "sizes": {}}
    r3 = lambda x: round(float(x), 3)
    for N in args.sizes:
        voxel = 2.0 / (N - 1)
        df, _ = grid.udf_band(udf, N)
        vi, faces = mesh._mc_lattice(udf, N, df, 0, 1 << 21)
        del df
        v64 = vi.double() * voxel - 1.0
        vd = udf.udf_values(v64.float()).reshape(-1)
        faces = faces[vd[faces].max(dim=1).values < voxel * args.ratio].contiguous()
        torch.cuda.empty_cache()
        runs = []
        for rep in range(args.repeats + 1):
            a, b, c = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            a.record()
            v, f, info = mesh_post.postprocess(v64, faces)
            b.record()
            ev, ef = mesh_post.export_merge(v, f)
            c.record()
            torch.cuda.synchronize()
            if rep:
                runs.append([info["ms"][k] for k in ("process", "holes", "loop", "smooth")]
                            + [b.elapsed_time(c), a.elapsed_time(b)])
        med = np.median(np.array(runs), axis=0)
        rec = {"mc_vertices": int(vi.shape[0]), "filtered_faces": int(faces.shape[0]),
               "ms": dict(zip(["process", "holes", "loop", "smooth", "export_merge", "postprocess"], [r3(x) for x in med])),
               "changed": {"process": info["process"], "hole_faces": info["hole_faces"], "loop": info["loop"],
                           "passes": info["passes"], "border_vertices": info["border_vertices"],
                           "export_merge_vertices": int(v.shape[0] - ev.shape[0])},
               "input": info["input"], "output": info["output"]}
        ms, _ = timed(lambda: mesh.udf_mesh_post(udf, N, dist_threshold_ratio=args.ratio), args.repeats)
        rec["udf_mesh_post_ms"] = r3(ms)
        hv, hf = v64.cpu().numpy(), faces.cpu().numpy()
        t = time.perf_counter()
        pv, pf, _ = P.postprocess(hv, hf)
        rec["restatement_host_ms"] = r3(1e3 * (time.perf_counter() - t))
        rec["restatement_same_bits"] = bool(np.array_equal(pf, f.cpu().numpy())
                                            and np.array_equal(pv.view(np.int64), v.cpu().numpy().view(np.int64)))
        del vi, faces, v64, vd, v, f, ev, ef
        torch.cuda.empty_cache()
        out["sizes"][str(N)] = rec
        print(json.dumps({str(N): rec}), file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()

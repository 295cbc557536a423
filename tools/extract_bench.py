"""Timing of the runner's extract_udf_mesh mesh path on the C5 scene (the golden UDF network): one JSON line.

    python tools/extract_bench.py [--sizes 256 512] [--no-reference]

Reported with the device name and power limit read in the same run.  Per lattice size, each measurement runs in its own
subprocess (so that the peak host RSS is per run), as Runner.extract_udf_mesh calls get_mesh_udf_fast: func = the network's
udf, func_grad its normalising closure, gradient=True, eps=0.005, dist_threshold_ratio 5, first with border gradients and
smoothing, again without them when that raises (the closed C5 surface always does).
  shadow      neuraludf_b200.extract_mesh after one warm-up call: the wall time of the two calls and, per call, the
              CUDA-event milliseconds of its stages (lattice, normals, mc, filter, post, gradient);
  reference   the unmodified get_mesh_udf_fast (extract_mesh.py:169-354) with the host lattice of
              get_udf_normals_grid_slow, the device MC drop-in (mesh.udf_mc_lewiner) and oracle/ref_post.py's trimesh
              stub: the wall time of the two calls, no warm-up.  The stub is not trimesh, so this is not trimesh's time.
Both run with the runner's default tensor type (torch.cuda.FloatTensor), so the reference's N^3 x 7 `samples` array is
allocated on the device, as under the runner.
Requires a CUDA device and, for the reference, the staged extract_mesh.py (oracle/make_ref.py); writes nothing.
"""
import argparse
import json
import os
import resource
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

EPS = 0.005
RATIO = 5.0


def _runner_calls(gmuf, func, func_grad, N, **kw):
    try:
        return [gmuf(func, func_grad, samples=None, indices=None, N_MC=N, gradient=True, eps=EPS, border_gradients=True,
                     smooth_borders=True, dist_threshold_ratio=RATIO, **kw)], True
    except Exception:
        return [gmuf(func, func_grad, samples=None, indices=None, N_MC=N, gradient=True, eps=EPS, border_gradients=False,
                     smooth_borders=False, dist_threshold_ratio=RATIO, **kw)], False


def _one(kind, N):
    import torch
    from tests.golden_util import load_golden
    from tests.gpu_util import build_modules
    udf = build_modules(load_golden(), "cuda")[0]

    def func_grad(xyz):                       # exp_runner_blending.py:767-771
        g = udf.gradient(xyz)
        return g / (torch.linalg.norm(g, ord=2, dim=-1, keepdim=True) + 1e-5)

    torch.set_default_tensor_type('torch.cuda.FloatTensor')     # as the runner runs (exp_runner_blending.py:872)
    res = {}
    if kind == "shadow":
        from neuraludf_b200 import extract_mesh as X
        infos = []

        def gmuf(*a, **k):
            infos.append({})
            return X.get_mesh_udf_fast(*a, info=infos[-1], **k)

        _runner_calls(gmuf, udf.udf, func_grad, N)
        torch.cuda.synchronize()
        infos.clear()
        t = time.perf_counter()
        (out,), smoothed = _runner_calls(gmuf, udf.udf, func_grad, N)
        torch.cuda.synchronize()
        res["wall_ms"] = (time.perf_counter() - t) * 1e3
        res["calls_stage_ms"] = [{k: round(v, 2) for k, v in i["stage_ms"].items()} for i in infos]
        res["mc"], res["filtered"], res["output"] = infos[-1]["mc"], infos[-1]["filtered"], infos[-1]["output"]
        res["device_peak_gb"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    else:
        from neuraludf_b200 import mesh
        from oracle import ref_post
        em = ref_post.load_extract_mesh()
        em.udf_mc_lewiner = mesh.udf_mc_lewiner
        t = time.perf_counter()
        (out,), smoothed = _runner_calls(em.get_mesh_udf_fast, udf.udf, func_grad, N)
        torch.cuda.synchronize()
        res["wall_ms"] = (time.perf_counter() - t) * 1e3
        res["output"] = (len(out[2].vertices), len(out[2].faces))
    res["smoothed"] = smoothed
    res["wall_ms"] = round(res["wall_ms"], 1)
    res["peak_host_rss_gb"] = round(resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20, 2)
    print("RESULT " + json.dumps(res))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--no-reference", action="store_true")
    ap.add_argument("--one", nargs=2, metavar=("KIND", "N"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("extract_bench needs a CUDA device")
    if args.one:
        return _one(args.one[0], int(args.one[1]))
    from tools.eval_bench import power_limit
    out = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(), "scene": "C5 golden UDF network",
           "dist_threshold_ratio": RATIO, "eps": EPS, "sizes": {}}
    for N in args.sizes:
        row = {}
        for kind in ["shadow"] + ([] if args.no_reference else ["reference"]):
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", kind, str(N)], cwd=ROOT,
                               capture_output=True, text=True)
            lines = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
            row[kind] = json.loads(lines[-1][7:]) if r.returncode == 0 and lines else {"error": r.stderr[-600:]}
        out["sizes"][str(N)] = row
    print(json.dumps(out))


if __name__ == "__main__":
    main()

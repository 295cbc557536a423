"""Run the UNMODIFIED reference evaluation scripts in-process -- test / baseline infrastructure only.

    python oracle/ref_eval.py          # <reference>/evaluation -> oracle/_ref/evaluation/  (dev container only)

`stage()` copies evaluation/eval_dtu_python.py and eval_deepfashion_python.py into the git-ignored `oracle/_ref/evaluation/`
with a sha256 manifest (as oracle/make_ref.py does for the render path), so that the GPU box, where the reference checkout
does not exist, can time the reference's `eval_cloud` (tools/eval_bench.py).

Both scripts import open3d, which is not installed.  `run_dtu` / `run_deepfashion` serve them an in-memory open3d stub
(meshes and clouds by path, vis clouds captured), replace the unseeded shuffle generator by a seeded one that records its
permutation, and wrap sklearn's NearestNeighbors to record what is fitted and queried.  DTU goes through `eval_cloud(args)`;
DeepFashion through its `__main__` block (runpy) with `glob.glob` answering for its hard-coded data directory, `os.makedirs`
ignoring that directory and the log redirected with `--log`.
"""
import contextlib
import glob as glob_mod
import hashlib
import importlib.util
import io
import json
import os
import runpy
import shutil
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(os.environ.get("NUDF_REFERENCE_ROOT", "/root/reference"), "evaluation")
DST = os.path.join(ROOT, "oracle", "_ref", "evaluation")
FILES = ["eval_dtu_python.py", "eval_deepfashion_python.py"]
DF_BASE = "/exp/udf/deepfashion3d/300/expname"          # eval_deepfashion_python.py's hard-coded data directory (:68)


def _sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def stage(verbose=True):
    """Copies the scripts; returns the manifest dict, or None when the reference checkout is absent."""
    if not all(os.path.isfile(os.path.join(SRC, f)) for f in FILES):
        return None
    os.makedirs(DST, exist_ok=True)
    for f in FILES:
        shutil.copyfile(os.path.join(SRC, f), os.path.join(DST, f))
    manifest = {f: _sha(os.path.join(DST, f)) for f in FILES}
    with open(os.path.join(DST, "MANIFEST.json"), "w") as fh:
        json.dump({"source": "xxlong0/NeuralUDF evaluation (unmodified copies)", "sha256": manifest}, fh, indent=1, sort_keys=True)
    if verbose:
        print("staged %d reference evaluation scripts under %s" % (len(manifest), DST))
    return manifest


def verify():
    """True when every staged script still has the recorded hash."""
    man_path = os.path.join(DST, "MANIFEST.json")
    if not os.path.isfile(man_path):
        return False
    man = json.load(open(man_path))["sha256"]
    return set(man) == set(FILES) and all(
        os.path.isfile(os.path.join(DST, f)) and _sha(os.path.join(DST, f)) == h for f, h in man.items())


# ---- the open3d stub -----------------------------------------------------------------------------------------------------
class _Mesh:
    def __init__(self, v, f):
        self.vertices, self.triangles = v, f


class _Cloud:
    def __init__(self, points=None):
        self.points = points
        self.colors = None


def open3d_stub(store, captured):
    """An `open3d` module serving store[path] = (vertices, faces or None) and capturing written clouds by file name."""
    o3d = types.ModuleType("open3d")
    o3d.geometry = types.SimpleNamespace(PointCloud=_Cloud)
    o3d.utility = types.SimpleNamespace(Vector3dVector=lambda a: np.asarray(a))
    o3d.io = types.SimpleNamespace(
        read_triangle_mesh=lambda p: _Mesh(np.array(store[p][0], np.float64), np.array(store[p][1], np.int32)),
        read_point_cloud=lambda p: _Cloud(np.array(store[p][0], np.float64)),
        write_point_cloud=lambda p, pc: captured.__setitem__(os.path.basename(p), (np.array(pc.points), np.array(pc.colors))))
    return o3d


@contextlib.contextmanager
def _recording(seed, rec):
    """seeded, recorded shuffle; recorded NearestNeighbors fits and queries"""
    import sklearn.neighbors as skln
    real_rng = np.random.default_rng
    NN = skln.NearestNeighbors
    saved = (NN.fit, NN.kneighbors, NN.radius_neighbors)

    class Shuffler:
        def shuffle(self, x, axis=0):
            assert axis == 0
            rec["data_pcd"] = np.array(x)
            perm = real_rng(seed).permutation(len(x))
            rec["perm"] = perm
            x[...] = x[perm]

    def fit(self, X, *a, **k):
        rec.setdefault("fits", []).append(np.array(X))
        return saved[0](self, X, *a, **k)

    def kneighbors(self, X=None, *a, **k):
        out = saved[1](self, X, *a, **k)
        rec.setdefault("kneighbors", []).append((np.array(X), np.array(out[0])))
        return out

    def radius_neighbors(self, X=None, *a, **k):
        out = saved[2](self, X, *a, **k)
        rec["radius_neighbors"] = out
        return out

    np.random.default_rng = lambda *a, **k: Shuffler()
    NN.fit, NN.kneighbors, NN.radius_neighbors = fit, kneighbors, radius_neighbors
    try:
        yield
    finally:
        np.random.default_rng = real_rng
        NN.fit, NN.kneighbors, NN.radius_neighbors = saved


def _load(name, stub):
    if not verify() and stage(verbose=False) is None:
        raise RuntimeError("reference evaluation scripts not staged (oracle/ref_eval.py)")
    sys.modules["open3d"] = stub
    spec = importlib.util.spec_from_file_location(name, os.path.join(DST, name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod                   # mp.Pool pickles sample_single_tri by module name
    spec.loader.exec_module(mod)
    return mod


def _kept(rec):
    """the scripts' loop (eval_dtu_python.py:93-97) over the recorded radius neighbourhoods -> kept positions"""
    idxs = rec["radius_neighbors"]
    mask = np.ones(len(idxs), dtype=np.bool_)
    for curr, ix in enumerate(idxs):
        if mask[curr]:
            mask[ix] = 0
            mask[curr] = 1
    return np.nonzero(mask)[0]


def run_dtu(data, faces, gt, obs_mask, bb, res, plane, seed, scan=1, density=0.2, patch=60.0, max_dist=20.0, vis=10.0):
    """eval_cloud of the unmodified script; returns the recorded stages and results (see module docstring)."""
    from scipy.io import savemat
    store, captured, rec = {}, {}, {}
    stub = open3d_stub(store, captured)
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "ObsMask"))
        savemat(os.path.join(tmp, "ObsMask", "ObsMask%d_10.mat" % scan), {"ObsMask": obs_mask, "BB": bb, "Res": res})
        savemat(os.path.join(tmp, "ObsMask", "Plane%d.mat" % scan), {"P": plane})
        store["data.ply"], store["gt.ply"] = (data, faces), (gt, None)
        args = types.SimpleNamespace(data="data.ply", gt="gt.ply", scan=scan, mode="mesh" if faces is not None else "pcd",
                                     dataset_dir=tmp, vis_out_dir=os.path.join(tmp, "vis"), downsample_density=density,
                                     patch_size=patch, max_dist=max_dist, visualize_threshold=vis,
                                     log=os.path.join(tmp, "log.txt"))
        mod = _load("eval_dtu_python", stub)
        with _recording(seed, rec), contextlib.redirect_stderr(io.StringIO()), contextlib.redirect_stdout(io.StringIO()):
            over_all, mean_d2s, mean_s2d = mod.eval_cloud(args)
    rec["kept_index"] = _kept(rec)
    rec.update(over_all=over_all, mean_d2s=mean_d2s, mean_s2d=mean_s2d, vis=captured)
    return rec


def run_deepfashion(data, faces, gt, seed, density=0.002, max_dist=0.1, vis=0.01):
    """the unmodified script's __main__ block for its scan 300 (runpy); returns the recorded stages, the printed results and
    the log text."""
    store, captured, rec = {}, {}, {}
    stub = open3d_stub(store, captured)
    with tempfile.TemporaryDirectory() as tmp:
        data_path = os.path.join(tmp, "mesh.ply")
        open(data_path, "w").close()             # the script checks that its data file exists; the stub serves its content
        store[data_path] = (data, faces)
        store["/dataset/deepfashion3d_point_cloud/300/300_pc_swap.ply"] = (gt, None)
        log = os.path.join(tmp, "log.txt")
        real_glob, real_makedirs = glob_mod.glob, os.makedirs
        glob_mod.glob = lambda p, *a, **k: [data_path] if p.startswith(DF_BASE) else real_glob(p, *a, **k)
        os.makedirs = lambda p, *a, **k: None if str(p).startswith("/exp/") else real_makedirs(p, *a, **k)
        argv = sys.argv
        sys.argv = ["eval_deepfashion_python.py", "--mode", "mesh" if faces is not None else "pcd", "--downsample_density",
                    repr(density), "--max_dist", repr(max_dist), "--visualize_threshold", repr(vis), "--log", log]
        out = io.StringIO()
        if not verify() and stage(verbose=False) is None:
            raise RuntimeError("reference evaluation scripts not staged (oracle/ref_eval.py)")
        sys.modules["open3d"] = stub
        try:
            with _recording(seed, rec), contextlib.redirect_stderr(io.StringIO()), contextlib.redirect_stdout(out):
                runpy.run_path(os.path.join(DST, "eval_deepfashion_python.py"), run_name="__main__")
        finally:
            glob_mod.glob, os.makedirs, sys.argv = real_glob, real_makedirs, argv
        with open(log) as f:
            rec["log"] = f.read()
    rec["stdout"] = out.getvalue()
    rec["kept_index"] = _kept(rec)
    rec["vis"] = captured
    vals = {}
    for line in out.getvalue().splitlines():          # "over_all: x; mean_d2gt: y; ..." -> {name: value}
        toks = line.replace(";", "").replace(":", "").rstrip(".").split()
        for k, v in zip(toks[::2], toks[1::2]):
            try:
                vals[k] = float(v.rstrip("."))
            except ValueError:
                pass
    rec["printed"] = vals
    return rec


if __name__ == "__main__":
    m = stage()
    if m is None:
        print("reference checkout not present at %s; nothing staged" % SRC)
        sys.exit(0 if verify() else 1)

"""Run the UNMODIFIED reference mesh-cleaning script in-process -- test / baseline infrastructure only.

    python oracle/ref_clean.py         # <reference>/evaluation/clean_dtu_mesh.py -> oracle/_ref/clean/  (dev container only)

`stage()` copies evaluation/clean_dtu_mesh.py into the git-ignored `oracle/_ref/clean/` with a sha256 manifest (as
oracle/ref_eval.py does for the evaluation scripts), so that the GPU box, where the reference checkout does not exist, can
time the reference's functions (tools/clean_bench.py).

The script imports trimesh, which is not installed, and reads its data from a `DTU_DIR` that only its main block sets.
`run_clean` serves it a trimesh stub (`load` returns arrays by path, `Trimesh(...).export(path)` captures the arrays under
that path, so the second stage loads exactly what the first exported), sets `DTU_DIR` on the module to a temporary tree of
scan<N>/cameras.npz and scan<N>/mask/%03d.png (cv2.imwrite), and runs clean_mesh_faces_by_mask then
clean_mesh_faces_by_visualhull as the main block chains them.  It records, per stage, the view counts (the accumulator the
script allocates with np.zeros), the thresholded dilated masks (cv2.dilate's outputs) and the exported arrays.
"""
import hashlib
import importlib.util
import json
import os
import shutil
import sys
import tempfile
import time
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(os.environ.get("NUDF_REFERENCE_ROOT", "/root/reference"), "evaluation")
DST = os.path.join(ROOT, "oracle", "_ref", "clean")
FILES = ["clean_dtu_mesh.py"]


def _sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def stage(verbose=True):
    """Copies the script; returns the manifest dict, or None when the reference checkout is absent."""
    if not all(os.path.isfile(os.path.join(SRC, f)) for f in FILES):
        return None
    os.makedirs(DST, exist_ok=True)
    for f in FILES:
        shutil.copyfile(os.path.join(SRC, f), os.path.join(DST, f))
    manifest = {f: _sha(os.path.join(DST, f)) for f in FILES}
    with open(os.path.join(DST, "MANIFEST.json"), "w") as fh:
        json.dump({"source": "xxlong0/NeuralUDF evaluation/clean_dtu_mesh.py (unmodified copy)", "sha256": manifest}, fh,
                  indent=1, sort_keys=True)
    if verbose:
        print("staged the reference mesh-cleaning script under %s" % DST)
    return manifest


def verify():
    """True when the staged script still has the recorded hash."""
    man_path = os.path.join(DST, "MANIFEST.json")
    if not os.path.isfile(man_path):
        return False
    man = json.load(open(man_path))["sha256"]
    return set(man) == set(FILES) and all(
        os.path.isfile(os.path.join(DST, f)) and _sha(os.path.join(DST, f)) == h for f, h in man.items())


class _Mesh:
    def __init__(self, vertices, faces, store=None):
        self.vertices, self.faces, self._store = np.asarray(vertices), np.asarray(faces), store

    def export(self, path):
        self._store[path] = (np.array(self.vertices), np.array(self.faces))


def trimesh_stub(store):
    """A `trimesh` module: load(path) serves store[path] = (vertices, faces); Trimesh(v, f).export(path) writes it back."""
    tm = types.ModuleType("trimesh")
    tm.load = lambda path, *a, **k: _Mesh(*store[path])
    tm.Trimesh = lambda vertices, faces, *a, **k: _Mesh(vertices, faces, store)
    return tm


class _Recorder:
    """Delegates to a module; records what np.zeros returns and what cv2.dilate returns."""

    def __init__(self, mod, name, sink):
        self._mod, self._name, self._sink = mod, name, sink

    def __getattr__(self, attr):
        fn = getattr(self._mod, attr)
        if attr != self._name:
            return fn

        def wrapped(*a, **k):
            out = fn(*a, **k)
            self._sink.append(out)
            return out
        return wrapped


def load_module(store):
    if not verify() and stage(verbose=False) is None:
        raise RuntimeError("reference mesh-cleaning script not staged (oracle/ref_clean.py)")
    sys.modules["trimesh"] = trimesh_stub(store)
    spec = importlib.util.spec_from_file_location("clean_dtu_mesh", os.path.join(DST, "clean_dtu_mesh.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def write_scan(root, scan, mats, masks):
    """<root>/scan<scan>/cameras.npz (world_mat_i) and mask/%03d.png"""
    import cv2
    d = os.path.join(root, "scan%d" % scan)
    os.makedirs(os.path.join(d, "mask"), exist_ok=True)
    np.savez(os.path.join(d, "cameras.npz"), **{"world_mat_%d" % i: np.asarray(m, np.float64) for i, m in enumerate(mats)})
    for i, m in enumerate(masks):
        assert cv2.imwrite(os.path.join(d, "mask", "%03d.png" % i), np.ascontiguousarray(m))
    return d


def run_clean(verts, faces, mats, masks, scan=24, imgs_idx=None, mask_kernel=11, minimal_vis=2):
    """The main block's two calls for one scan; returns [stage dict] * 2 with `verts`, `faces` (exported), `counts` (int64),
    `dilated` (channel 0 of every cv2.dilate output of the stage, [V, H, W] uint8) and `seconds` (the wall time of the call)."""
    store = {"mesh.ply": (np.asarray(verts, np.float64), np.asarray(faces, np.int64))}
    mod = load_module(store)
    zeros, dilated = [], []
    mod.np = _Recorder(np, "zeros", zeros)
    mod.cv = _Recorder(mod.cv, "dilate", dilated)
    out = []
    with tempfile.TemporaryDirectory() as tmp:
        write_scan(tmp, scan, mats, masks)
        mod.DTU_DIR = tmp
        calls = ((mod.clean_mesh_faces_by_mask, "mesh.ply", "clean_%03d.ply" % scan, mask_kernel),
                 (mod.clean_mesh_faces_by_visualhull, "clean_%03d.ply" % scan, "visualhull_%03d.ply" % scan, mask_kernel + 20))
        for fn, src, dst, kernel in calls:
            del zeros[:], dilated[:]
            t = time.perf_counter()
            fn(src, dst, scan, imgs_idx, minimal_vis=minimal_vis, mask_dilated_size=kernel)
            seconds = time.perf_counter() - t
            assert len(zeros) == 1
            counts = zeros[0]
            assert np.array_equal(counts, np.round(counts))
            v, f = store[dst]
            out.append(dict(verts=v, faces=f, counts=counts.astype(np.int64), seconds=seconds,
                            dilated=np.stack([d[:, :, 0] for d in dilated])))
    return out


if __name__ == "__main__":
    m = stage()
    if m is None:
        print("reference checkout not present at %s; nothing staged" % SRC)
        sys.exit(0 if verify() else 1)

"""Compile the reference's MeshUDF marching cubes (`custom_mc`, Cython) -- test / baseline infrastructure only.

    python oracle/make_ref_mc.py       # <reference>/custom_mc -> oracle/_ref/custom_mc/  (needs Cython)

The reference ships `_marching_cubes_lewiner_cy` prebuilt for CPython 3.6 only.  Its three sources are copied unmodified
into the git-ignored `oracle/_ref/custom_mc/`, a manifest with their sha256 is written beside them (as oracle/make_ref.py
does) and the extension is compiled there in C++ mode against numpy's headers -- the reference's own `setup.py` recipe.
The built module travels with the staged copy; `load()` imports it.  Consumers: the golden meshes
(oracle/make_golden_mesh.py), the GPU mesh tests (reference pipeline at N = 128) and tools/mesh_bench.py (CPU time of the
reference MC).  Without Cython or without the reference checkout nothing is built and a message says why.
"""
import glob
import hashlib
import importlib
import json
import os
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(os.environ.get("NUDF_REFERENCE_ROOT", "/root/reference"), "custom_mc")
DST = os.path.join(ROOT, "oracle", "_ref", "custom_mc")
FILES = ["_marching_cubes_lewiner_cy.pyx", "_marching_cubes_lewiner.py", "_marching_cubes_lewiner_luts.py"]

_SETUP = """
import numpy as np
from setuptools import setup, Extension
from Cython.Build import cythonize
ext = Extension("_marching_cubes_lewiner_cy", ["_marching_cubes_lewiner_cy.pyx"], include_dirs=[np.get_include()],
                language="c++")
setup(name="ref_custom_mc", ext_modules=cythonize([ext], include_path=[np.get_include()], quiet=True),
      script_args=["build_ext", "--inplace", "--build-temp", "_build"])
"""


def _sha(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def _built():
    return sorted(glob.glob(os.path.join(DST, "_marching_cubes_lewiner_cy*.so")))


def available():
    return bool(_built()) and os.path.isfile(os.path.join(DST, "MANIFEST.json"))


def verify():
    """True when every staged source still has the recorded hash and the compiled module is present."""
    if not available():
        return False
    man = json.load(open(os.path.join(DST, "MANIFEST.json")))["sha256"]
    return set(man) == set(FILES) and all(
        os.path.isfile(os.path.join(DST, f)) and _sha(os.path.join(DST, f)) == h for f, h in man.items())


def stage(verbose=True):
    """Copies and compiles; returns the manifest dict, or None when nothing could be built here."""
    if not all(os.path.isfile(os.path.join(SRC, f)) for f in FILES):
        if verbose and not available():
            print("make_ref_mc: no reference custom_mc at %s; reference MC not built" % SRC)
        return None
    try:
        import Cython  # noqa: F401
    except ImportError:
        if verbose:
            print("make_ref_mc: Cython is not installed; reference MC not built")
        return None
    os.makedirs(DST, exist_ok=True)
    manifest = {f: _sha(os.path.join(SRC, f)) for f in FILES}
    if verify() and json.load(open(os.path.join(DST, "MANIFEST.json")))["sha256"] == manifest:
        return manifest                                          # up to date
    for f in FILES:
        shutil.copyfile(os.path.join(SRC, f), os.path.join(DST, f))
    for so in _built():
        os.remove(so)
    r = subprocess.run([sys.executable, "-c", _SETUP], cwd=DST, capture_output=True, text=True)
    shutil.rmtree(os.path.join(DST, "_build"), ignore_errors=True)
    shutil.rmtree(os.path.join(DST, "build"), ignore_errors=True)
    if r.returncode != 0 or not _built():
        if verbose:
            print("make_ref_mc: compiling the reference MC failed; not built:\n" + r.stdout[-2000:] + r.stderr[-2000:])
        return None
    with open(os.path.join(DST, "MANIFEST.json"), "w") as f:
        json.dump({"source": "xxlong0/NeuralUDF custom_mc (unmodified copies, compiled with Cython in C++ mode)",
                   "sha256": {k: _sha(os.path.join(DST, k)) for k in FILES}}, f, indent=1, sort_keys=True)
    if verbose:
        print("make_ref_mc: built %s" % os.path.basename(_built()[0]))
    return manifest


def load():
    """The reference's `_marching_cubes_lewiner` module (its `udf_mc_lewiner`), imported from the staged build."""
    if not verify():
        raise RuntimeError("reference MC not built (oracle/make_ref_mc.py)")
    if DST not in sys.path:
        sys.path.insert(0, DST)
    mod = sys.modules.get("_marching_cubes_lewiner")
    if mod is not None and os.path.dirname(os.path.abspath(mod.__file__)) == DST:
        return mod
    sys.modules.pop("_marching_cubes_lewiner", None)
    return importlib.import_module("_marching_cubes_lewiner")


if __name__ == "__main__":
    m = stage()
    sys.exit(0 if (m is not None or available()) else 1)

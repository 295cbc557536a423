"""Run the reference's UNMODIFIED `exp_runner_blending.py` on top of the nudf modules.

    python -m neuraludf_b200.launch /path/to/NeuralUDF/exp_runner_blending.py [runner args ...]

`models.fields`, `models.embedder`, `models.udf_renderer_blending` and `models.patch_projector` are bound to the nudf
mirrors before the runner is executed from the reference root; everything else the runner imports (`dataset`, `loss`, ...)
still resolves from the reference checkout (its `models/` directory is a namespace package).  `custom_mc` (the Cython
MeshUDF marching cubes that extract_mesh.py imports) is bound to neuraludf_b200.mesh when the reference's own build cannot
be imported by the running interpreter.  With NUDF_DEVICE_LOSS=1 in the environment, `loss.loss` and `loss.patch_metric`
are bound to neuraludf_b200.loss (the colour loss on the device); without it the runner's own loss files run.  With
NUDF_BAND_MESH=1, `validate_mesh`'s `extract_geometry` (when PyMCubes cannot be imported) evaluates its lattice narrow-band
(grid.iso_band: the same mesh when the UDF is 2-Lipschitz and batch-invariant); without it the whole lattice is queried.
With NUDF_DEVICE_MESH=1, `extract_mesh` (the runner's get_mesh_udf_fast) is bound to neuraludf_b200.extract_mesh: the
lattice, MC, post-processing and gradient branch of extract_udf_mesh on the device, with no N^3 host array (NUDF_BAND_MESH=1
then evaluates its lattice narrow-band too); without it the runner's own extract_mesh.py runs.  NUDF_BAND_MESH=sparse
holds either band block-sparse (grid.iso_band_sparse / udf_band_sparse): the same meshes with no N^3 device array either,
for resolutions up to 2048.
"""
import importlib
import importlib.machinery
import os
import runpy
import sys
import types


def install_shadow_modules(reference_root=None):
    """Registers the mirrors under the names the reference imports. Returns the `models` namespace module."""
    from neuraludf_b200.models import embedder, fields, patch_projector, udf_renderer_blending
    pkg = sys.modules.get("models")
    if pkg is None:
        pkg = types.ModuleType("models")
        pkg.__path__ = []
        sys.modules["models"] = pkg
    if reference_root is not None:
        p = os.path.join(reference_root, "models")
        if os.path.isdir(p) and p not in list(pkg.__path__):
            pkg.__path__ = list(pkg.__path__) + [p]
    for name, mod in (("fields", fields), ("embedder", embedder), ("udf_renderer_blending", udf_renderer_blending),
                      ("patch_projector", patch_projector)):
        sys.modules["models." + name] = mod
        setattr(pkg, name, mod)
    _install_custom_mc(reference_root)
    if os.environ.get("NUDF_DEVICE_LOSS") == "1":
        _install_device_loss(reference_root)
    if os.environ.get("NUDF_DEVICE_MESH") == "1":
        from neuraludf_b200 import extract_mesh
        sys.modules["extract_mesh"] = extract_mesh
    return pkg


def _install_device_loss(reference_root):
    """Serves `loss.loss` (ColorLoss, ...) and `loss.patch_metric` (SSIM, NCC, ...) from neuraludf_b200.loss."""
    from neuraludf_b200 import loss
    pkg = sys.modules.get("loss")
    if pkg is None:
        pkg = types.ModuleType("loss")
        pkg.__path__ = []
        sys.modules["loss"] = pkg
    if reference_root is not None:
        p = os.path.join(reference_root, "loss")
        if os.path.isdir(p) and p not in list(pkg.__path__):
            pkg.__path__ = list(pkg.__path__) + [p]
    for name in ("loss", "patch_metric"):
        sys.modules["loss." + name] = loss
        setattr(pkg, name, loss)


def _native_custom_mc(reference_root):
    """True when `<root>/custom_mc` holds a `_marching_cubes_lewiner_cy` extension this interpreter can import (the
    reference ships one built for CPython 3.6 only)."""
    if reference_root is None:
        return False
    d = os.path.join(reference_root, "custom_mc")
    return any(os.path.isfile(os.path.join(d, "_marching_cubes_lewiner_cy" + s))
               for s in importlib.machinery.EXTENSION_SUFFIXES)


def _install_custom_mc(reference_root):
    """Serves `custom_mc._marching_cubes_lewiner.udf_mc_lewiner` (imported at module level by the runner's
    extract_mesh.py) from neuraludf_b200.mesh, unless the name is already bound or the reference's own Cython build can
    serve this interpreter."""
    if "custom_mc._marching_cubes_lewiner" in sys.modules or _native_custom_mc(reference_root):
        return
    from neuraludf_b200 import mesh
    pkg = sys.modules.get("custom_mc")
    if pkg is None:
        pkg = types.ModuleType("custom_mc")
        pkg.__path__ = []
        sys.modules["custom_mc"] = pkg
    mod = types.ModuleType("custom_mc._marching_cubes_lewiner")
    mod.__doc__ = "MeshUDF marching cubes on the nudf CUDA kernels (neuraludf_b200.mesh)"
    mod.udf_mc_lewiner = mesh.udf_mc_lewiner
    sys.modules["custom_mc._marching_cubes_lewiner"] = mod
    pkg._marching_cubes_lewiner = mod


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    if not argv:
        print(__doc__)
        return 2
    runner = os.path.abspath(argv[0])
    root = os.path.dirname(runner)
    install_shadow_modules(root)
    if root not in sys.path:
        sys.path.insert(1, root)
    os.chdir(root)
    sys.argv = [runner] + argv[1:]
    runpy.run_path(runner, run_name="__main__")
    return 0


if __name__ == "__main__":
    sys.exit(main())

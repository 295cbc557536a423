"""The NumPy restatement of get_mesh_udf_fast's gradient branch (tests/proto/mesh_grad.py) against the unmodified reference
run under the restated trimesh rules (tests/golden/grad_*.npz, oracle/make_golden_grad.py), and the NUDF_DEVICE_MESH switch
of launch.install_shadow_modules."""
import sys

import numpy as np
import pytest

from tests.golden_util import Fixtures
from tests.proto import mesh_grad as G

CASES = ["sheet", "closed", "empty", "lattice", "network"]


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference(name):
    fx = Fixtures("grad_" + name)
    v, f, eps, N = fx["mesh_verts"], fx["mesh_faces"], float(fx["eps"]), int(fx["N"])
    v32 = v.astype(np.float32)
    n = G.vertex_normals(v, f)
    p1, p2 = G.probes(v32, n, eps)
    assert np.array_equal(p1, fx["p1"]) and np.array_equal(p2, fx["p2"])
    nv = G.refine(v32, n, fx["s1"], fx["s2"], eps)
    assert nv.dtype == np.float32 and np.array_equal(nv.view(np.int32), fx["new_verts"].view(np.int32))
    ni = G.next_indices(nv, N)
    assert ni.dtype == np.int64 and np.array_equal(ni, fx["next_indices"])
    assert G.raises(f) == (not bool(fx["smoothed"]))
    print("%s: %d vertices, %d faces, smoothed %s, max |new - v| %.2e" % (name, len(v), len(f), bool(fx["smoothed"]),
                                                                        float(np.abs(nv - v32).max()) if len(v) else 0.0))


def test_raise_condition():
    closed = Fixtures("grad_closed")["mesh_faces"]
    sheet = Fixtures("grad_sheet")["mesh_faces"]
    empty = np.zeros((0, 3), np.int64)
    for f in (closed, empty):
        assert G.raises(f) and G.raises(f, border_gradients=False) and G.raises(f, gradient=False, border_gradients=True)
        assert not G.raises(f, border_gradients=False, smooth_borders=False)
        assert not G.raises(f, gradient=False, smooth_borders=False)
    assert not G.raises(sheet)


def test_next_indices_edge_values():
    """trunc toward zero, numpy's wrap-around for the clamped neighbours, INT64_MIN for NaN"""
    N = 5
    v = np.array([[-1.0, -1.0, 1.0], [-1.2, 0.0, 0.49], [np.nan, 0.0, 0.0]], np.float32)
    ni = G.next_indices(v, N).reshape(7, 3)
    assert ni[0, 0] == 0 * 25 + 0 * 5 + 4 and ni[3, 0] == 4 and ni[6, 0] == 3     # k at N - 1: +z clamps, -z steps
    assert ni[0, 1] == 0 * 25 + 2 * 5 + 2                                          # trunc(-0.2 / 0.5) = 0
    assert ni[0, 2] < -(1 << 62)


@pytest.mark.parametrize("flag", [None, "0", "1"])
def test_install_registers_extract_mesh_only_when_asked(monkeypatch, flag):
    from neuraludf_b200 import launch
    if flag is None:
        monkeypatch.delenv("NUDF_DEVICE_MESH", raising=False)
    else:
        monkeypatch.setenv("NUDF_DEVICE_MESH", flag)
    for k in ("extract_mesh", "models", "custom_mc", "custom_mc._marching_cubes_lewiner"):
        monkeypatch.delitem(sys.modules, k, raising=False)
    for k in [k for k in sys.modules if k.startswith("models.")]:
        monkeypatch.delitem(sys.modules, k)
    launch.install_shadow_modules(None)
    if flag == "1":
        from neuraludf_b200 import extract_mesh
        assert sys.modules["extract_mesh"] is extract_mesh
        assert sys.modules["extract_mesh"].get_mesh_udf_fast is extract_mesh.get_mesh_udf_fast
    else:
        assert "extract_mesh" not in sys.modules

"""The NumPy restatement of the threshold marching cubes (tests/proto/iso_mc.py) on analytic and seeded fields: topology,
vertex placement, orientation, the edge cases of the corner rule, and the CLI's argument rules."""
import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from tests.proto import iso_mc as P
from tests.proto import mesh_cases as C


def _edges(faces):
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    u, c = np.unique(np.sort(e, 1), axis=0, return_counts=True)
    return e, u, c


def _on_box(verts, dims):
    """[V, 6] bool: vertex on the box face (axis, low / high)"""
    hi = np.asarray(dims, np.float64) - 1
    return np.concatenate([verts == 0, verts == hi[None, :]], 1)


def _components(verts, faces):
    n = len(verts)
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]]])
    g = coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(n, n))
    _, lab = connected_components(g, directed=False)
    return [faces[lab[faces[:, 0]] == k] for k in np.unique(lab[faces[:, 0]])]


def _check_manifold(verts, faces, dims):
    """no edge in more than two faces; an edge in one face lies on a box face; no directed edge twice (consistent winding)"""
    e, u, c = _edges(faces)
    assert c.max() <= 2
    box = _on_box(verts, dims)
    b = u[c == 1]
    assert (box[b[:, 0]] & box[b[:, 1]]).any(1).all()
    _, cd = np.unique(e, axis=0, return_counts=True)
    assert cd.max() == 1


def test_shell_gives_two_closed_spheres():
    df, dims, level, _ = P.case("shell")
    v, f, _ = P.marching_cubes(df, dims, level)
    comps = _components(v, f)
    assert len(comps) == 2
    for cf in comps:
        s = C.mesh_stats(v, cf)
        assert s["boundary"] == 0 and s["nonmanifold"] == 0 and s["same_direction"] == 0
        assert s["euler"] == 2


def test_torus_has_euler_characteristic_zero():
    df, dims, level, _ = P.case("torus")
    v, f, _ = P.marching_cubes(df, dims, level)
    assert len(_components(v, f)) == 1
    s = C.mesh_stats(v, f)
    assert s["boundary"] == 0 and s["nonmanifold"] == 0 and s["euler"] == 0


def test_box_cut_has_boundary_only_on_the_box():
    df, dims, level, _ = P.case("cut")
    v, f, _ = P.marching_cubes(df, dims, level)
    s = C.mesh_stats(v, f)
    assert s["boundary"] > 0
    _check_manifold(v, f, dims)


@pytest.mark.parametrize("name", ["random0", "random1", "random2", "random3", "quantised", "ties"])
def test_random_fields_are_manifold(name):
    df, dims, level, _ = P.case(name)
    v, f, info = P.marching_cubes(df, dims, level)
    assert len(f) > 1000
    _check_manifold(v, f, dims)
    if name.startswith("random"):
        assert int((info["vertex_keys"] >= 3 * np.prod(dims)).sum()) > 0        # loop centres exercised


@pytest.mark.parametrize("name", P.CASES)
def test_vertices_interpolate_to_the_level(name):
    df, dims, level, _ = P.case(name)
    v, f, info = P.marching_cubes(df, dims, level)
    keys = info["vertex_keys"]
    ek = keys < 3 * int(np.prod(dims))
    g, ax = keys[ek] // 3, keys[ek] % 3
    strides = np.array([dims[1] * dims[2], dims[2], 1])
    vv = P.corner_values(df, level).astype(np.float64)
    va, vb = vv[g], vv[g + strides[ax]]
    assert ((va > 0) != (vb > 0)).all()                                        # every edge vertex is on a crossing edge
    rows = np.arange(len(g))
    lower = np.stack([g // strides[0], (g // strides[1]) % dims[1], g % dims[2]], 1).astype(np.float64)
    other = np.ones((len(g), 3), bool)
    other[rows, ax] = False
    assert (v[ek][other] == lower[other]).all()                                # the other coordinates are the edge's
    t = v[ek][rows, ax] - lower[rows, ax]
    assert (t >= 0).all() and (t <= 1).all()
    # the linear interpolation of v = f32(f - level) along the edge vanishes at the vertex: f interpolates to the level
    lin = va + t * (vb - va)
    assert (np.abs(lin) <= 1e-12 * np.maximum(np.abs(va), np.abs(vb))).all()
    assert np.isfinite(v).all()


@pytest.mark.parametrize("name", ["shell", "torus", "cut", "min"])
def test_faces_point_towards_decreasing_values(name):
    df, dims, level, grad = P.case(name)
    v, f, _ = P.marching_cubes(df, dims, level)
    h = [2.0 / (n - 1) for n in dims]
    w = -1.0 + v * np.asarray(h)[None, :]                                       # world coordinates
    n = np.cross(w[f[:, 1]] - w[f[:, 0]], w[f[:, 2]] - w[f[:, 0]])
    gr = grad(v[f].mean(1))
    assert ((n * gr).sum(1) < 0).all()


def test_minimum_lattice():
    df, dims, level, _ = P.case("min")
    v, f, info = P.marching_cubes(df, dims, level)
    assert info["active"].tolist() == [0] and len(f) == 1
    # v = -0.25 at corners 0..6 and 0.75 at corner 7: each crossing is a quarter of the way up from the lower corner
    assert sorted(map(tuple, v)) == [(0.25, 1.0, 1.0), (1.0, 0.25, 1.0), (1.0, 1.0, 0.25)]


def test_exact_zero_corners_sit_on_the_low_side():
    df = np.zeros(8, np.float32)
    df[0] = 1.0                            # corner 0 above the level 0, the rest exactly at it
    v, f, info = P.marching_cubes(df, (2, 2, 2), 0.0)
    assert len(f) == 1
    assert sorted(map(tuple, v)) == [(0.0, 0.0, 1.0), (0.0, 1.0, 0.0), (1.0, 0.0, 0.0)]
    v, f, _ = P.marching_cubes(df, (2, 2, 2), 1.0)                              # nothing above the level: no crossing
    assert v.shape == (0, 3) and f.shape == (0, 3)


def test_nan_cells_emit_nothing():
    df, dims, level, _ = P.case("shell")
    df = df.copy()
    df[len(df) // 2 + 7] = np.nan
    v, f, info = P.marching_cubes(df, dims, level)
    _, _, info0 = P.marching_cubes(P.case("shell")[0], dims, level)
    hit = set((len(df) // 2 + 7 - P.U.corner_offsets(dims)).tolist())
    assert not hit & set(info["active"].tolist())
    assert set(info["active"].tolist()) == set(info0["active"].tolist()) - hit


def test_level_is_rounded_to_fp32_once():
    df, dims, _, _ = P.case("random0")
    lv = 0.1 + 1e-12                                                             # the same fp32 as 0.1
    a, b = P.marching_cubes(df, dims, lv), P.marching_cubes(df, dims, np.float32(0.1))
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_cli_rejects_threshold_with_udf_options():
    from neuraludf_b200 import mesh
    for extra in (["--postprocess"], ["--dense"], ["--lipschitz", "2"], ["--dist_threshold_ratio", "1"]):
        with pytest.raises(SystemExit) as e:
            mesh.main(["--ckpt", "none.pth", "--out", "none.ply", "--threshold", "0.005"] + extra)
        assert e.value.code == 2


def test_threshold_box_matches_the_dataset():
    import os
    import tempfile
    from neuraludf_b200 import mesh
    lo, hi, sm = mesh.threshold_box(None)
    assert lo.tolist() == [np.float32(-1.01)] * 3 and hi.tolist() == [np.float32(1.01)] * 3 and sm is None
    s = np.eye(4)
    s[:3, :3] *= 1.7
    s[:3, 3] = [0.3, -0.2, 0.9]
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "cameras.npz")
        np.savez(p, scale_mat_0=s, world_mat_0=np.eye(4))
        lo, hi, sm = mesh.threshold_box(p)
    # dataset/dataset.py:112-123 with the same file for both camera roles: inv(fp32 scale) @ fp64 scale @ box
    want = np.linalg.inv(s.astype(np.float32)) @ s @ np.array([-1.01, -1.01, -1.01, 1.0])[:, None]
    assert np.array_equal(lo, want[:3, 0].astype(np.float32))
    assert sm.dtype == np.float32 and np.array_equal(sm, s.astype(np.float32))

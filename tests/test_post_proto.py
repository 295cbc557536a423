"""The NumPy restatement of the mesh post-processing (tests/proto/mesh_post.py) against the unmodified reference's
get_mesh_udf_fast run under the restated trimesh rules (tests/golden/post_*.npz, oracle/make_golden_post.py), and the
properties of its output."""
import numpy as np
import pytest

from tests.golden_util import Fixtures
from tests.proto import mesh_cases as C
from tests.proto import mesh_post as P

CASES = sorted(C.CASES) + ["network", "holes", "figure8", "duplicates", "slivers", "nan", "closed", "book"]


def _golden(name):
    fx = Fixtures("post_" + name)
    return fx


def _max_border_degree(faces, n_verts):
    if len(faces) == 0:
        return 0
    e, _ = P.boundary(faces, n_verts)
    return int(np.bincount(e.reshape(-1), minlength=n_verts).max()) if len(e) else 0


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference(name):
    fx = _golden(name)
    v, f, info = P.postprocess(fx["in_verts"], fx["in_faces"])
    v, f = P.export_merge(v, f)
    gv, gf = P.canonical(fx["out_verts"], fx["out_faces"])
    cv, cf = P.canonical(v, f)
    assert np.array_equal(cf, gf)
    assert cv.shape == gv.shape
    err = float(np.abs(cv - gv).max()) if len(cv) else 0.0
    assert err <= 1e-12
    if _max_border_degree(f, len(v)) <= 2:
        assert np.array_equal(cv, gv)                        # at most two border neighbours: the same sums, bit for bit
    # the reference smooths exactly when the mesh has border edges (else its smoothing raises and it falls back)
    assert bool(fx["smoothed"]) == (info["border_vertices"] > 0)
    print("%s: %s, passes %d, hole faces %d, border vertices %d, max |dv| %.1e"
          % (name, info["process"], info["passes"], info["hole_faces"], info["border_vertices"], err))


@pytest.mark.parametrize("name", CASES)
def test_networkx_disagreements(name):
    """trimesh's cycle_basis recipe against the hole rule, recounted on the mesh fill_holes sees"""
    from oracle import ref_post
    fx = _golden(name)
    _, _, info = P.postprocess(fx["in_verts"], fx["in_faces"])
    v, f = info["pre_fill"]
    ref_post.NX_DISAGREEMENTS[0] = 0
    m = ref_post.Trimesh(v, f, process=False)
    m.fill_holes()
    assert ref_post.NX_DISAGREEMENTS[0] == int(fx["nx_disagreements"])
    assert np.array_equal(np.sort(np.sort(m.faces[len(f):], 1), 0),
                          np.sort(np.sort(P.hole_faces(v, f), 1), 0))     # the stub adds the rule's faces
    if name == "figure8":
        assert int(fx["nx_disagreements"]) == 2                           # networkx fills both triangles, the rule neither


def _cycles_closed(v_pre, f_pre, new):
    """every added face (or pair) closes a 3- or 4-cycle of boundary edges of the mesh before filling"""
    e, _ = P.boundary(f_pre, len(v_pre))
    border = {tuple(x) for x in e.tolist()}
    edges_new = {}
    for t in new.tolist():
        for k in range(3):
            a, b = sorted((t[k], t[(k + 1) % 3]))
            edges_new[(a, b)] = edges_new.get((a, b), 0) + 1
    outer = {k for k, c in edges_new.items() if c == 1}
    return outer <= border


@pytest.mark.parametrize("name", CASES)
def test_output_properties(name):
    fx = _golden(name)
    v, f, info = P.postprocess(fx["in_verts"], fx["in_faces"])
    assert len(f) == 0 or (P.nondegenerate(v, f).all() and P.first_unique(f).all())
    assert np.array_equal(np.unique(f), np.arange(len(v)))                # no unreferenced vertices
    assert len(np.unique(P.merge_keys(v), axis=0)) == len(v)              # nothing left to merge
    assert np.isfinite(v).all()
    v0, f0 = info["pre_fill"]
    new = P.hole_faces(v0, f0)
    assert len(new) == info["hole_faces"]
    assert _cycles_closed(v0, f0, new)
    b_in = len(P.boundary(f0, len(v0))[0]) if len(f0) else 0
    b_out = len(P.boundary(f, len(v))[0]) if len(f) else 0
    assert b_out <= b_in                                                  # filling never adds border edges
    # the loop can only remove faces fill_holes added, whose vertices all belong to other faces: one pass
    assert info["passes"] == (1 if len(f) else 0)


def test_crafted_rules():
    fx = _golden("holes")
    v, f, info = P.postprocess(fx["in_verts"], fx["in_faces"], smooth_borders=False)
    assert info["hole_faces"] == 5                                        # triangle 1, quad 2, square 2; the 5-hole stays
    fx = _golden("slivers")
    _, _, info = P.postprocess(fx["in_verts"], fx["in_faces"])
    assert info["process"]["degenerate"] >= 4
    fx = _golden("duplicates")
    _, _, info = P.postprocess(fx["in_verts"], fx["in_faces"])
    assert info["process"]["duplicate"] == 4
    fx = _golden("nan")
    _, _, info = P.postprocess(fx["in_verts"], fx["in_faces"])
    assert info["process"]["nonfinite"] == 2
    fx = _golden("book")
    _, _, info = P.postprocess(fx["in_verts"], fx["in_faces"])
    assert info["hole_faces"] == 1 and info["loop"][0]["duplicate"] == 1   # the isolated triangle's reverse, removed
    fx = _golden("closed")
    v, f, info = P.postprocess(fx["in_verts"], fx["in_faces"])
    assert info["border_vertices"] == 0 and np.array_equal(v, fx["in_verts"])


def test_equal_diagonal_tie():
    """a square hole in a 4 x 4 grid: both diagonals equal, the split goes through the smallest vertex"""
    n = 4
    ij = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2)
    v = np.concatenate([ij.astype(float), np.zeros((n * n, 1))], 1)
    f = []
    for i in range(n - 1):
        for j in range(n - 1):
            if (i, j) != (1, 1):
                a, b, c, d = i * n + j, (i + 1) * n + j, (i + 1) * n + j + 1, i * n + j + 1
                f += [[a, c, b], [a, d, c]] if (i + j) % 2 else [[b, d, a], [b, c, d]]
    f = np.asarray(f)
    new = P.hole_faces(v, f)
    assert len(new) == 2 and all(5 in t and 10 in t for t in new.tolist())
    directed = {(g[j], g[(j + 1) % 3]) for g in f.tolist() for j in range(3)}
    for t in new.tolist():                                                # the fill runs against the existing faces
        assert not any((t[k], t[(k + 1) % 3]) in directed for k in range(3))

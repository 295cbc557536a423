"""The connected-component filters' NumPy restatement (tests/proto/mesh_cc.py) on the CPU: against a brute-force breadth-first
search over face adjacency on the crafted cases, and against the unmodified clean_outliers of the reference
(tests/golden/cc_*.npz, oracle/make_golden_cc.py)."""
from collections import deque

import numpy as np
import pytest

from tests.golden_util import Fixtures
from tests.proto import mesh_cc as C


def _bfs(faces):
    """(label, paired) by breadth-first search: faces are neighbours when an edge has exactly two slots, of different faces"""
    f = np.asarray(faces).reshape(-1, 3).tolist()
    slots = {}
    for i, t in enumerate(f):
        for k in range(3):
            a, b = t[k], t[(k + 1) % 3]
            slots.setdefault(frozenset((a, b)) if a != b else (a,), []).append(i)
    nb = [set() for _ in f]
    for s in slots.values():
        if len(s) == 2 and s[0] != s[1]:
            nb[s[0]].add(s[1])
            nb[s[1]].add(s[0])
    label = np.full(len(f), -1, np.int64)
    for s in range(len(f)):                     # ascending seeds: each component is labelled by its smallest face
        if label[s] >= 0:
            continue
        label[s] = s
        q = deque([s])
        while q:
            x = q.popleft()
            for y in nb[x]:
                if label[y] < 0:
                    label[y] = s
                    q.append(y)
    return label, np.array([len(n) > 0 for n in nb], np.uint8)


@pytest.mark.parametrize("name", C.CASES)
def test_labels_match_bfs(name):
    _, f = C.case(name)
    label, paired = C.face_components(f)
    bl, bp = _bfs(f)
    assert np.array_equal(label, bl) and np.array_equal(paired, bp)
    for shift in (1, 2):                        # the rule does not depend on where each face's vertex list starts
        g = np.roll(f, shift, axis=1)
        assert np.array_equal(C.face_components(g)[0], bl)


@pytest.mark.parametrize("name", C.CASES)
def test_filters_match_bfs(name):
    v, f = C.case(name)
    bl, bp = _bfs(f)
    sizes = {s: int((bl == s).sum()) for s in set(bl.tolist())}
    if len(f):
        best = min(sizes, key=lambda s: (-sizes[s], s))
        lv, lf = C.keep_largest(v, f)
        assert len(lf) == sizes[best]
        assert np.array_equal(lv[lf], v[f[bl == best]], equal_nan=True)
    for n in (1, 2, 3, 500):
        keep = np.array([bp[i] and int(bp[bl == bl[i]].sum()) >= n for i in range(len(f))], bool)
        sv, sf = C.remove_small_components(v, f, n)
        assert np.array_equal(sv[sf], v[f[keep]], equal_nan=True)
        assert np.array_equal(np.unique(f[keep]), np.nonzero(np.isin(np.arange(len(v)), f[keep]))[0])
        assert len(sv) == len(np.unique(f[keep]))


def test_crafted_rules():
    """the adjacency rules on the cases built for them"""
    lab = {n: C.face_components(C.case(n)[1]) for n in C.CASES}
    assert lab["fan3"][0].tolist() == [0, 0, 2, 2, 4, 4] and lab["fan4"][0].tolist() == [0, 0, 2, 2, 4, 4, 6, 6]
    assert lab["bowtie"][0].tolist() == [0, 1] and lab["bowtie"][1].tolist() == [0, 0]
    assert lab["duplicate_isolated"][0].tolist() == [0, 1, 2, 3, 3]    # a triangle thrice: each of its edges used 3 times
    l, p = lab["duplicate_embedded"]
    assert l[7] == 7 and l[18] == 18 and p[7] == 0 and p[18] == 0 and (np.delete(l, [7, 18]) == 0).all()
    l, p = lab["degenerate"]
    assert p[0] == 0 and p[1] == 0 and p[6] == 0 and l[6] == 6
    assert lab["isolated"][0].tolist() == [0, 1, 2, 3, 4] and not lab["isolated"][1].any()
    assert lab["empty"][0].shape == (0,) and lab["one_face"][0].tolist() == [0]
    l, _ = lab["tie"]
    assert l.tolist() == [0, 1, 2, 0, 1, 2]


@pytest.mark.parametrize("name", C.CASES)
def test_restatement_matches_reference(name):
    """clean_outliers(keep_largest=True) of the unmodified script under a trimesh stub; face order compared as a set (the
    reference's order inside a piece is not defined), vertices exactly"""
    fx = Fixtures("cc_" + name)
    v, f = C.case(name)
    assert np.array_equal(fx["in_faces"], f)
    assert np.array_equal(fx["in_verts"].view(np.int64), v.view(np.int64))
    pv, pf = C.clean_outliers(v, f, keep_largest=True)
    if "largest_error" in fx:
        assert str(fx["largest_error"]).startswith("ValueError") and len(pf) == 0 and len(f) == 0
        return
    gv, gf = fx["largest_verts"], fx["largest_faces"]
    assert np.array_equal(pv.view(np.int64), gv.view(np.int64))
    assert np.array_equal(np.sort(pf.view("i8,i8,i8").reshape(-1)), np.sort(gf.view("i8,i8,i8").reshape(-1)))


@pytest.mark.parametrize("name", C.CASES)
def test_reference_faces_num_cannot_run(name):
    """clean_mesh_by_faces_num raises wherever the port keeps a face: IndexError (its per-face mask is indexed with vertex
    ids), or ValueError when no component reaches faces_num (np.concatenate of nothing)"""
    fx = Fixtures("cc_" + name)
    v, f = C.case(name)
    for n in (500, 2):
        err = str(fx["faces_num_error_%d" % n])
        _, kept = C.clean_outliers(v, f, faces_num=n, keep_largest=False)
        assert err.startswith("IndexError" if len(kept) else "ValueError"), (n, err)

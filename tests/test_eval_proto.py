"""The NumPy restatement of the evaluation protocols (tests/proto/eval_pc.py) against the reference's golden evaluations, the
PLY reader / writer of neuraludf_b200/evaluate.py, and the properties of the greedy downsampling (CPU only)."""
import numpy as np
import pytest

from neuraludf_b200 import evaluate as E
from tests.golden_util import Fixtures
from tests.proto import eval_cases as C
from tests.proto import eval_pc as P


def _run_proto(fx, name):
    density, patch, max_dist, vis = (float(x) for x in fx["params"])
    faces = fx["faces"] if "faces" in fx else None
    if C.case(name)["protocol"] == "dtu":
        return P.eval_dtu(fx["data"], faces, fx["gt"], fx["obs_mask"], fx["bb"], fx["res"], fx["plane"], fx["perm"],
                          density=density, patch=patch, max_dist=max_dist, vis=vis)
    return P.eval_deepfashion(fx["data"], faces, fx["gt"], fx["perm"], density=density, max_dist=max_dist, vis=vis)


@pytest.mark.parametrize("name", C.CASES)
def test_proto_matches_reference(name):
    fx = Fixtures("eval_" + name)
    c = C.case(name)
    assert np.array_equal(fx["data"], c["data"]) and np.array_equal(fx["gt"], c["gt"])      # inputs regenerate
    assert np.array_equal(fx["perm"], P.seeded_permutation(len(fx["data_pcd"]), int(fx["seed"])))
    r = _run_proto(fx, name)
    assert np.array_equal(r["data_pcd"], fx["data_pcd"])                     # bit-identical samples, same order
    assert np.array_equal(r["kept_index"], fx["kept_index"])
    assert np.array_equal(r["dist_d2s"], fx["dist_d2s"]) and np.array_equal(r["dist_s2d"], fx["dist_s2d"])
    assert np.array_equal(r["data_color"], fx["data_color"]) and np.array_equal(r["gt_color"], fx["gt_color"])
    assert r["mean_d2gt"] == fx["mean_d2s"] and r["mean_gt2d"] == fx["mean_s2d"] and r["over_all"] == fx["over_all"]
    if "inbound" in fx:
        assert np.array_equal(r["inbound"], fx["inbound"])
        assert np.array_equal(np.where(r["inbound"])[0][r["grid_inbound"]][r["in_obs"]], fx["in_obs_index"])
        assert np.array_equal(r["above"], fx["above"])
        assert 0 < r["inbound"].sum() <= len(r["inbound"])
    else:
        printed = [r[k] for k in ("precision_1", "recall_1", "fscore_1", "precision_2", "recall_2", "fscore_2")]
        assert np.array_equal(printed, fx["printed"])
    if name == "dtu_sphere":        # the case exercises what it is meant to
        assert not r["inbound"].all() and not r["in_obs"].all() and not r["above"].all()
    if name == "dtu_patch":
        assert (r["dist_s2d"] >= 20.0).sum() > 1000


def test_deepfashion_log_format():
    fx = Fixtures("eval_deepfashion")
    r = _run_proto(fx, "deepfashion")
    assert E.format_log(r, "mesh", 6) == str(fx["log"])


def test_seeded_shuffle_is_the_scripts_shuffle():
    pts = np.random.default_rng(0).normal(size=(1000, 3))
    a = pts.copy()
    np.random.default_rng(42).shuffle(a, axis=0)
    assert np.array_equal(a, pts[E.seeded_permutation(1000, 42)])


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_greedy_set_properties(seed):
    rng = np.random.default_rng(seed)
    pts = rng.uniform(0, 10, size=(6000, 3))
    pts[:200] = pts[200:400]                                   # exact duplicates
    r = 0.4
    perm = rng.permutation(len(pts))
    kept_pts, kept = P.downsample(pts, r, perm)
    sp = pts[perm]
    from scipy.spatial import cKDTree
    t = cKDTree(kept_pts)
    pairs = t.query_pairs(r * (1 - 1e-9))
    assert not pairs                                           # no two kept points within r
    is_kept = np.zeros(len(sp), bool)
    is_kept[kept] = True
    nb = cKDTree(sp).query_ball_point(sp[~is_kept], r * (1 + 1e-9))
    dropped = np.nonzero(~is_kept)[0]
    for v, ns in zip(dropped, nb):                             # every dropped point has a lower-rank kept neighbour
        assert any(u < v and is_kept[u] for u in ns)


def _trimesh_style_binary(path, v, f):
    """a PLY as trimesh exports it: float vertices with extra properties, uchar-int face lists, a face colour"""
    head = ("ply\nformat binary_little_endian 1.0\ncomment https://github.com/mikedh/trimesh\nelement vertex %d\n"
            "property float x\nproperty float y\nproperty float z\nproperty float nx\nproperty uchar red\n"
            "element face %d\nproperty list uchar int vertex_indices\nproperty uchar alpha\nend_header\n" % (len(v), len(f)))
    vd = np.zeros(len(v), dtype=[("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("red", "u1")])
    vd["x"], vd["y"], vd["z"] = v[:, 0], v[:, 1], v[:, 2]
    fd = np.zeros(len(f), dtype=[("n", "u1"), ("i", "<i4", (3,)), ("alpha", "u1")])
    fd["n"], fd["i"] = 3, f
    with open(path, "wb") as fh:
        fh.write(head.encode())
        fh.write(vd.tobytes())
        fh.write(fd.tobytes())


def test_ply_trimesh_binary(tmp_path):
    v, f = C.uv_sphere(1.0, 6, 8)
    p = str(tmp_path / "m.ply")
    _trimesh_style_binary(p, v, f)
    rv, rf = E.read_ply(p)
    assert np.array_equal(rv, v.astype(np.float32).astype(np.float64)) and np.array_equal(rf, f)


def test_ply_ascii_mesh(tmp_path):
    v, f = C.grid_patch(3, 2.0)
    p = tmp_path / "a.ply"
    lines = ["ply", "format ascii 1.0", "element vertex %d" % len(v), "property double x", "property double y",
             "property double z", "property uchar green", "element face %d" % len(f), "property list uchar uint vertex_index",
             "end_header"] + ["%r %r %r 7" % tuple(float(c) for c in x) for x in v] + ["3 %d %d %d" % tuple(x) for x in f]
    p.write_text("\n".join(lines) + "\n")
    rv, rf = E.read_ply(str(p))
    assert np.array_equal(rv, v) and np.array_equal(rf, f)


@pytest.mark.parametrize("ascii", [False, True])
def test_ply_points_round_trip(tmp_path, ascii):
    rng = np.random.default_rng(3)
    pts, col = rng.normal(size=(500, 3)) * 100, rng.uniform(size=(500, 3))
    p = str(tmp_path / "c.ply")
    E.write_ply_points(p, pts, col, ascii=ascii)
    rv, rf = E.read_ply(p)
    assert rf is None and np.array_equal(rv, pts)
    assert np.array_equal(E.read_ply_colors(p), np.round(col * 255).astype(np.uint8))


def test_ply_rejects_other_formats(tmp_path):
    p = tmp_path / "b.ply"
    p.write_bytes(b"ply\nformat binary_big_endian 1.0\nelement vertex 0\nproperty float x\nend_header\n")
    with pytest.raises(ValueError):
        E.read_ply(str(p))

"""The NumPy restatement of the DTU mesh-cleaning protocol (tests/proto/mesh_clean.py) against the reference's golden
cleanings, the ellipse element and the dilation against OpenCV, and the mesh PLY writer (CPU only)."""
import numpy as np
import pytest

from neuraludf_b200 import clean as CL
from neuraludf_b200 import evaluate as E
from tests.golden_util import Fixtures
from tests.proto import clean_cases as C
from tests.proto import mesh_clean as M

cv2 = pytest.importorskip("cv2")


def run_case(name):
    """(case, fixtures, proto stages) with the views the case selects"""
    c = C.case(name)
    fx = Fixtures("clean_" + name)
    idx = c["imgs_idx"] if c["imgs_idx"] is not None else list(range(49))
    stages = M.clean_dtu_mesh(c["verts"], c["faces"], c["mats"][idx], c["masks"][idx], c["mask_kernel"], c["minimal_vis"])
    return c, fx, stages


@pytest.mark.parametrize("name", C.CASES)
def test_proto_matches_reference(name):
    c, fx, stages = run_case(name)
    assert str(fx["inputs_sha"]) == C.sha256(c["verts"], c["faces"], c["mats"], c["masks"])      # inputs regenerate
    for tag, (v, f, counts, keep, bits) in zip(("mask", "hull"), stages):
        assert np.array_equal(counts, fx["counts_" + tag])
        assert C.sha256(M.pack(bits)) == str(fx["packed_sha_" + tag])
        assert C.sha256(v.astype(np.float64), f.astype(np.int64)) == str(fx["out_sha_" + tag])
        assert [len(v), len(f)] == fx["out_size_" + tag].tolist()
    if name == "antialiased":           # the masks hold 127, 128 and 129 where vertices project
        assert {127, 128, 129} <= set(np.unique(c["masks"]).tolist())
    if name == "all_views":
        assert int(fx["params"][2]) == -1 and len(c["mats"]) == 49


def test_cases_exercise_the_corners():
    c = C.case("edges")
    mats = c["mats"]
    u, v = M.project(c["verts"], mats[0])
    for x in (-1, 0, C.W, C.W + 1):
        assert (u == x).any()
    for y in (-1, 0, C.H, C.H + 1):
        assert (v == y).any()
    assert (c["verts"][:, 2] < 0).any() and (np.abs(c["verts"]).sum(1) == 0).any()
    for name in ("sphere", "antialiased", "kernel31"):          # the screen holds: no projection near a half-integer
        c = C.case(name)
        idx = c["imgs_idx"]
        assert M.half_integer_distance(c["verts"], c["mats"][idx]).min() >= C.TIE_EPS


def test_ellipse_element_is_opencv():
    for k in range(1, 65):
        assert np.array_equal(CL.ellipse_element(k), cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (k, k))), k


@pytest.mark.parametrize("k", [1, 2, 3, 10, 11, 30, 31, 64, 101])
def test_dilation_is_opencv(k):
    rng = np.random.default_rng(k)
    img = rng.integers(0, 256, size=(157, 211), dtype=np.uint8)
    img[rng.uniform(size=img.shape) < 0.97] = 0
    img[0, 0], img[-1, -1], img[0, -1], img[-1, 0] = 255, 254, 253, 252            # maxima on the borders
    el = cv2.getStructuringElement(cv2.MORPH_ELLIPSE, (k, k))
    assert np.array_equal(M.dilate(img, k), cv2.dilate(img, el))
    assert np.array_equal(M.dilate(img[:, :, None].repeat(3, 2)[:, :, 0], k), cv2.dilate(img[:, :, None].repeat(3, 2), el)[:, :, 0])


def test_dilation_of_other_elements_is_opencv():
    rng = np.random.default_rng(0)
    img = (rng.uniform(size=(64, 80)) < 0.02).astype(np.uint8) * rng.integers(1, 256, size=(64, 80)).astype(np.uint8)
    for shape, size in ((cv2.MORPH_RECT, (7, 4)), (cv2.MORPH_CROSS, (5, 9)), (cv2.MORPH_RECT, (1, 6))):
        el = cv2.getStructuringElement(shape, size)
        assert np.array_equal(M.dilate(img, el), cv2.dilate(img, el))


def test_element_rows_rejects_split_rows():
    with pytest.raises(ValueError):
        CL.element_rows(np.array([[1, 0, 1]]))
    lo, hi = CL.element_rows(CL.ellipse_element(10))
    assert lo[0] == 5 and hi[0] == 6 and lo[5] == 0 and hi[5] == 10


def test_ply_mesh_round_trip(tmp_path):
    rng = np.random.default_rng(1)
    v = rng.normal(size=(300, 3)) * 100
    f = rng.integers(0, 300, size=(500, 3))
    p = str(tmp_path / "m.ply")
    E.write_ply_mesh(p, v, f)
    rv, rf = E.read_ply(p)
    assert np.array_equal(rv, v) and np.array_equal(rf, f)
    E.write_ply_mesh(p, v[:0], f[:0])
    rv, rf = E.read_ply(p)
    assert rv.shape == (0, 3) and rf.shape == (0, 3)

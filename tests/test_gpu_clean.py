"""CUDA mesh cleaning (neuraludf_b200/clean.py, csrc/mesh_clean.cu) against the reference's golden cleanings and the NumPy
restatement (tests/proto/mesh_clean.py): packed masks, view counts and compacted meshes exactly; the dilation at odd, even
and large kernels; exact half-integer ties; a full-size 49-view scan; determinism; udf_mesh -> clean -> eval_dtu; the CLI."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.golden_util import Fixtures
from tests.proto import clean_cases as C
from tests.proto import eval_pc as EP
from tests.proto import mesh_clean as M

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _views(c):
    idx = c["imgs_idx"] if c["imgs_idx"] is not None else list(range(49))
    return c["mats"][idx], c["masks"][idx]


def _packed_np(packed):
    return packed.cpu().numpy().view(np.uint32)


@pytest.mark.parametrize("name", C.CASES)
def test_fixture_matches(name):
    dev = _dev()
    from neuraludf_b200 import clean as CL
    c = C.case(name)
    fx = Fixtures("clean_" + name)
    mats, masks = _views(c)
    stages = CL.clean_dtu_mesh(torch.from_numpy(c["verts"]).to(dev), torch.from_numpy(c["faces"]).to(dev), mats,
                               torch.from_numpy(masks).to(dev), mask_kernel=c["mask_kernel"], minimal_vis=c["minimal_vis"])
    for tag, (v, f, info) in zip(("mask", "hull"), stages):
        assert C.sha256(_packed_np(info["packed"])) == str(fx["packed_sha_" + tag]), tag
        counts = info["counts"].cpu().numpy()
        assert np.array_equal(counts, fx["counts_" + tag]), tag
        assert np.array_equal(info["keep"].cpu().numpy(), counts < 5 if tag == "hull" else counts > c["minimal_vis"])
        assert [v.shape[0], f.shape[0]] == fx["out_size_" + tag].tolist()
        assert C.sha256(v.cpu().numpy().astype(np.float64), f.cpu().numpy().astype(np.int64)) == str(fx["out_sha_" + tag]), tag


@pytest.mark.parametrize("k", [1, 2, 10, 11, 30, 31, 101])
def test_dilation_bit_identical(k):
    dev = _dev()
    from neuraludf_b200 import clean as CL
    rng = np.random.default_rng(k)
    img = rng.integers(0, 256, size=(3, 203, 333), dtype=np.uint8)
    img[rng.uniform(size=img.shape) < 0.995] = 0
    img[:, 0, :] = rng.integers(0, 256, size=(3, 333))                  # values on every border
    img[:, :, -1] = rng.integers(0, 256, size=(3, 203))
    for t in (40, 128, 200):          # dilation commutes with the monotone shift: thresholds at 128 probe level t
        shifted = np.clip(img.astype(np.int32) + 128 - t, 0, 255).astype(np.uint8)
        for below in (False, True):
            got = CL.dilate_masks(torch.from_numpy(shifted).to(dev), k, below=below)
            want = np.stack([M.threshold(M.dilate(m, k), below) for m in shifted])
            assert np.array_equal(_packed_np(got), M.pack(want)), (t, below)
            assert np.array_equal(CL.unpack_masks(got, 333).cpu().numpy(), want)


def test_exact_half_integer_ties():
    dev = _dev()
    from neuraludf_b200 import clean as CL
    masks = np.zeros((1, 40, 64), np.uint8)
    masks[0, 5, 10] = masks[0, 5, 12] = masks[0, 6, 10] = 255
    # identity camera: q = (x / z, y / z); rint is half to even: 10.5 -> 10, 11.5 -> 12, 9.5 -> 10, 12.5 -> 12, 4.5 -> 4, 5.5 -> 6
    pts = np.array([[10.5, 5.0, 1.0], [11.5, 5.0, 1.0], [9.5, 5.0, 1.0], [12.5, 5.0, 1.0], [11.0, 5.0, 1.0], [13.5, 5.0, 1.0],
                    [10.0, 4.5, 1.0], [10.0, 5.5, 1.0], [21.0, 10.5, 2.0], [23.0, 10.0, 2.0]])
    mats = np.eye(4)[None]
    packed = CL.dilate_masks(torch.from_numpy(masks).to(dev), 1)
    got = CL.count_views(torch.from_numpy(pts).to(dev), mats, packed, 40, 64).cpu().numpy()
    want = M.count_views(pts, mats, masks > 128, 0)
    assert got.tolist() == want.tolist() == [1, 1, 1, 1, 0, 0, 0, 1, 1, 1]


def _compare_stages(stages, ref, verts, mats, what):
    """GPU stages against the restatement's: packed masks exactly; counts exactly except at vertices whose projection lies
    within 1e-6 px of a half-integer; the compacted meshes exactly when no count differs"""
    pts = verts
    for (gv, gf, info), (rv, rf, rcounts, rkeep, rbits) in zip(stages, ref):
        assert np.array_equal(_packed_np(info["packed"]), M.pack(rbits))
        counts = info["counts"].cpu().numpy()
        diff = np.nonzero(counts != rcounts)[0]
        print("%s: %d vertices, %d counts differ" % (what, len(pts), len(diff)))
        assert np.all(M.half_integer_distance(pts[diff], mats) < 1e-6)
        if len(diff):
            return False
        assert np.array_equal(gv.cpu().numpy(), rv) and np.array_equal(gf.cpu().numpy(), rf)
        pts = rv
    return True


def test_full_size_scan():
    """49 views at 1600 x 1200 and a ~400 k-vertex mesh: equal to the restatement except where a projection is within 1e-6
    px of a half-integer (the only place the summation order of the projection matters)"""
    dev = _dev()
    from neuraludf_b200 import clean as CL
    from tests.proto import eval_cases as EC
    rng = np.random.default_rng(77)
    mats = C.ring(49, seed=5)
    masks = np.stack([C.silhouette(P, (0., 0., 0.), 96.0) for P in mats])
    v, f = EC.uv_sphere(100.0, 450, 900)
    jv, jf = C.junk_sheets(rng)
    verts = np.concatenate([v, jv]) + rng.normal(scale=0.8, size=(len(v) + len(jv), 3))
    faces = np.concatenate([f, jf + len(v)])
    assert len(verts) > 400_000
    stages = CL.clean_dtu_mesh(torch.from_numpy(verts).to(dev), torch.from_numpy(faces).to(dev), mats,
                               torch.from_numpy(masks).to(dev))
    ref = M.clean_dtu_mesh(verts, faces, mats, masks)
    _compare_stages(stages, ref, verts, mats, "full-size scan")


def test_two_runs_bit_identical():
    dev = _dev()
    from neuraludf_b200 import clean as CL
    c = C.case("all_views")
    mats, masks = _views(c)
    args = (torch.from_numpy(c["verts"]).to(dev), torch.from_numpy(c["faces"]).to(dev), mats, torch.from_numpy(masks).to(dev))
    a, b = CL.clean_dtu_mesh(*args), CL.clean_dtu_mesh(*args)
    for (av, af, ai), (bv, bf, bi) in zip(a, b):
        assert torch.equal(av, bv) and torch.equal(af, bf)
        for k in ("counts", "keep", "packed"):
            assert torch.equal(ai[k], bi[k])


def test_udf_mesh_clean_eval_end_to_end():
    """udf_mesh of the golden network at N = 128, to world space (mm), cleaned under a ring of cameras, then eval_dtu; each
    step against its restatement"""
    dev = _dev()
    from neuraludf_b200 import clean as CL
    from neuraludf_b200 import evaluate as E
    from neuraludf_b200 import mesh
    from tests.golden_util import load_golden
    from tests.gpu_util import build_modules
    udf = build_modules(load_golden(), "cuda")[0]
    v, f = mesh.udf_mesh(udf, 128)
    assert f.shape[0] > 1000
    scale = torch.tensor(100.0, dtype=torch.float64, device=dev)              # scale_mat: diag(100) + translation
    vw = v.double() * scale + torch.tensor([3.0, -2.0, 1.0], dtype=torch.float64, device=dev)
    vn, fn = vw.cpu().numpy(), f.cpu().numpy()
    centre = vn.mean(0)
    mats = C.ring(12, dist=450.0, seed=9)
    masks = np.stack([C.silhouette(P, centre, np.percentile(np.linalg.norm(vn - centre, axis=1), 60)) for P in mats])
    stages = CL.clean_dtu_mesh(vw, f, mats, torch.from_numpy(masks).to(dev))
    _compare_stages(stages, M.clean_dtu_mesh(vn, fn, mats, masks), vn, mats, "udf_mesh N=128")
    (v1, f1, _), (v2, f2, _) = stages
    assert 0 < f2.shape[0] < f.shape[0]
    r2, rf2 = v2.cpu().numpy(), f2.cpu().numpy()
    rng = np.random.default_rng(4)
    gt = r2[rng.choice(len(r2), min(len(r2), 30000), replace=False)] + 0.3 * rng.normal(size=(min(len(r2), 30000), 3))
    bb = np.array([centre - 110.0, centre + 110.0])
    obs = np.ones((56, 56, 56), np.uint8)
    res, plane = np.array([[4.0]]), np.array([[0.0, 0.0, 1.0, 200.0]])
    r = E.eval_dtu(v2, f2, torch.from_numpy(gt).to(dev), obs, bb, res, plane, seed=3)
    p = EP.eval_dtu(r2, rf2, gt, obs, bb, res, plane, E.seeded_permutation(r["n_points"], 3))
    for k in ("mean_d2gt", "mean_gt2d", "over_all"):
        assert abs(r[k] - p[k]) <= 1e-12 * abs(p[k])
    print("udf_mesh N=128: %d -> %d -> %d faces, over_all %.4f mm" % (f.shape[0], f1.shape[0], f2.shape[0], r["over_all"]))


def test_cli(tmp_path):
    _dev()
    import cv2
    from neuraludf_b200 import evaluate as E
    c = C.case("sphere")
    fx = Fixtures("clean_sphere")
    scan_dir = tmp_path / "dtu" / ("scan%d" % C.SCAN)
    os.makedirs(scan_dir / "mask")
    np.savez(str(scan_dir / "cameras.npz"), **{"world_mat_%d" % i: m for i, m in enumerate(c["mats"])})
    for i, m in enumerate(c["masks"]):
        assert cv2.imwrite(str(scan_dir / "mask" / ("%03d.png" % i)), m)
    E.write_ply_mesh(str(tmp_path / "mesh.ply"), c["verts"], c["faces"])
    cmd = [sys.executable, "-m", "neuraludf_b200.clean", "--mesh", str(tmp_path / "mesh.ply"), "--dtu_dir",
           str(tmp_path / "dtu"), "--scan", str(C.SCAN), "--out_dir", str(tmp_path / "out"), "--mask_kernel",
           str(c["mask_kernel"]), "--minimal_vis", str(c["minimal_vis"]), "--imgs_idx"] + [str(i) for i in c["imgs_idx"]]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    for tag, stem in (("mask", "clean"), ("hull", "visualhull")):
        v, f = E.read_ply(str(tmp_path / "out" / ("%s_%03d.ply" % (stem, C.SCAN))))
        assert C.sha256(v, f.astype(np.int64)) == str(fx["out_sha_" + tag])

"""CUDA point-cloud evaluation (neuraludf_b200/evaluate.py, csrc/eval_pc.cu) against the reference's golden evaluations
stage by stage, against the NumPy / sklearn restatement (tests/proto/eval_pc.py) on ~1 M-point clouds and on a mesh of the
golden UDF network, the nearest-distance search against brute force, run-to-run determinism and the CLI."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.golden_util import Fixtures
from tests.proto import eval_cases as C
from tests.proto import eval_pc as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _ulp_equal(a, b, max_dist):
    """distances within 1 ulp where the reference's is below max_dist; both sides agree on which are >= max_dist"""
    a, b = np.asarray(a), np.asarray(b)
    far = b >= max_dist
    assert np.array_equal(a >= max_dist, far)
    assert np.all(np.isinf(a[far]))
    assert np.all(np.abs(a[~far] - b[~far]) <= np.spacing(b[~far]))


def _run(fx, name, dev, perm=None, colors=True):
    from neuraludf_b200 import evaluate as E
    density, patch, max_dist, vis = (float(x) for x in fx["params"])
    data = torch.from_numpy(fx["data"]).to(dev)
    faces = torch.from_numpy(fx["faces"]).to(dev) if "faces" in fx else None
    perm = fx["perm"] if perm is None else perm
    gt = torch.from_numpy(fx["gt"]).to(dev)
    if C.case(name)["protocol"] == "dtu":
        return E.eval_dtu(data, faces, gt, fx["obs_mask"], fx["bb"], fx["res"], fx["plane"], density=density, patch=patch,
                          max_dist=max_dist, visualize_threshold=vis, perm=perm, colors=colors)
    return E.eval_deepfashion(data, faces, gt, density=density, max_dist=max_dist, visualize_threshold=vis, perm=perm,
                              colors=colors)


@pytest.mark.parametrize("name", C.CASES)
def test_fixture_stages(name):
    dev = _dev()
    fx = Fixtures("eval_" + name)
    max_dist, thresholds = float(fx["params"][2]), ((1.0, 2.0) if name.startswith("dtu") else (0.001, 0.002))
    r = _run(fx, name, dev)
    s = r["stages"]
    assert np.array_equal(s["data_pcd"].cpu().numpy(), fx["data_pcd"])                 # bit-identical, same order
    assert np.array_equal(s["downsample"]["kept_index"].cpu().numpy(), fx["kept_index"])
    print("%s: %d points, %d kept, %d rounds" % (name, len(fx["data_pcd"]), len(fx["kept_index"]), s["downsample"]["rounds"]))
    if "inbound" in fx:
        inbound = s["inbound"].cpu().numpy()
        assert np.array_equal(inbound, fx["inbound"])
        idx = np.nonzero(inbound)[0][s["grid_inbound"].cpu().numpy()][s["in_obs"].cpu().numpy()]
        assert np.array_equal(idx, fx["in_obs_index"])
        assert np.array_equal(s["above"].cpu().numpy(), fx["above"])
    d2s, s2d = s["dist_d2s"].cpu().numpy(), s["dist_s2d"].cpu().numpy()
    _ulp_equal(d2s, fx["dist_d2s"], max_dist)
    _ulp_equal(s2d, fx["dist_s2d"], max_dist)
    for t in thresholds:                                                                 # threshold counts exact
        assert (d2s < t).sum() == (fx["dist_d2s"] < t).sum() and (s2d < t).sum() == (fx["dist_s2d"] < t).sum()
    for k, ref in (("mean_d2gt", fx["mean_d2s"]), ("mean_gt2d", fx["mean_s2d"]), ("over_all", fx["over_all"])):
        assert abs(r[k] - float(ref)) <= 1e-12 * abs(float(ref)), (k, r[k], float(ref))
    if "printed" in fx:
        got = [r[k] for k in ("precision_1", "recall_1", "fscore_1", "precision_2", "recall_2", "fscore_2")]
        assert np.array_equal(got, fx["printed"])
    np.testing.assert_allclose(r["data_color"].cpu().numpy(), fx["data_color"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(r["gt_color"].cpu().numpy(), fx["gt_color"], rtol=0, atol=1e-12)


def test_two_runs_bit_identical():
    dev = _dev()
    from neuraludf_b200 import evaluate as E
    fx = Fixtures("eval_dtu_sphere")
    a = _run(fx, "dtu_sphere", dev, perm=E.seeded_permutation(len(fx["data_pcd"]), 9))
    b = _run(fx, "dtu_sphere", dev, perm=E.seeded_permutation(len(fx["data_pcd"]), 9))
    for k in ("mean_d2gt", "mean_gt2d", "over_all", "precision_1", "recall_2", "n_down", "n_in_obs"):
        assert a[k] == b[k]
    for k in ("dist_d2s", "dist_s2d"):
        assert torch.equal(a["stages"][k], b["stages"][k])
    assert torch.equal(a["stages"]["downsample"]["kept_index"], b["stages"]["downsample"]["kept_index"])


def _check_downsample(pts, radius, seed, dev):
    from neuraludf_b200 import evaluate as E
    perm = E.seeded_permutation(len(pts), seed)
    kept_pts, info = E.downsample(torch.from_numpy(pts).to(dev), radius, perm=perm)
    ref_pts, ref_kept = P.downsample(pts, radius, perm)
    n = len(pts)
    print("downsample %d points r=%g: %d kept, %d edges, %d rounds" % (n, radius, len(ref_kept), info["edges"], info["rounds"]))
    assert np.array_equal(info["kept_index"].cpu().numpy(), ref_kept)
    assert np.array_equal(kept_pts.cpu().numpy(), ref_pts)
    assert 1 <= info["rounds"] <= 4 * int(np.log2(n)) ** 2


def test_downsample_1m_random_cloud():
    dev = _dev()
    rng = np.random.default_rng(5)
    pts = rng.uniform(0, 50, size=(1_000_000, 3))
    _check_downsample(pts, 0.6, 1, dev)


def test_sample_and_downsample_1m_mesh():
    dev = _dev()
    from neuraludf_b200 import evaluate as E
    v, f = C.uv_sphere(64.0, 120, 240, center=(3.0, -2.0, 10.0))
    pcd = E.sample_mesh(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev), 0.2).cpu().numpy()
    ref = P.sample_mesh(v, f, 0.2)
    assert len(ref) > 1_000_000
    assert np.array_equal(pcd, ref)
    _check_downsample(ref, 0.2, 2, dev)


def _brute(q, t):
    d2 = np.full(len(q), np.inf)
    for i in range(0, len(t), 512):
        tt = t[i:i + 512]
        dx, dy, dz = (q[:, None, k] - tt[None, :, k] for k in range(3))
        d2 = np.minimum(d2, ((dx * dx + dy * dy) + dz * dz).min(axis=1))
    return np.sqrt(d2)


@pytest.mark.parametrize("max_dist", [float("inf"), 0.5])
def test_nearest_brute_force(max_dist):
    dev = _dev()
    from neuraludf_b200 import evaluate as E
    rng = np.random.default_rng(8)
    t = np.concatenate([rng.normal(size=(5000, 3)), rng.uniform(-3, 3, size=(37, 3))])
    q = rng.uniform(-4, 4, size=(3000, 3))
    want = _brute(q, t)
    got = E.nearest_distance(torch.from_numpy(q).to(dev), torch.from_numpy(t).to(dev), max_dist).cpu().numpy()
    want = np.where(want < max_dist, want, np.inf)
    assert np.array_equal(got, want)
    assert np.array_equal(got, np.where(P.nearest(q, t) < max_dist, P.nearest(q, t), np.inf))


def test_nearest_all_beyond_max_dist():
    dev = _dev()
    from neuraludf_b200 import evaluate as E
    rng = np.random.default_rng(9)
    t = rng.normal(size=(4000, 3)) + 100.0
    q = rng.normal(size=(2000, 3))
    got = E.nearest_distance(torch.from_numpy(q).to(dev), torch.from_numpy(t).to(dev), 20.0)
    assert bool(torch.isinf(got).all())
    assert bool(torch.isinf(E.nearest_distance(torch.from_numpy(q).to(dev), torch.zeros(0, 3, device=dev))).all())


def test_udf_mesh_end_to_end():
    """udf_mesh of the golden network at N = 128, scaled to mm, through eval_dtu against the proto"""
    dev = _dev()
    from neuraludf_b200 import evaluate as E
    from neuraludf_b200 import mesh
    from tests.golden_util import load_golden
    from tests.gpu_util import build_modules
    udf = build_modules(load_golden(), "cuda")[0]
    v, f = mesh.udf_mesh(udf, 128)
    assert f.shape[0] > 1000
    vmm = v.double() * 100.0 + torch.tensor([0.0, 0.0, 50.0], dtype=torch.float64, device=dev)
    rng = np.random.default_rng(12)
    vn = vmm.cpu().numpy()
    gt = vn[rng.choice(len(vn), min(len(vn), 40000), replace=False)] + 0.3 * rng.normal(size=(min(len(vn), 40000), 3))
    bb = np.array([[-90.0, -90.0, -40.0], [90.0, 90.0, 140.0]])
    obs = (rng.uniform(size=(46, 46, 46)) > 0.05).astype(np.uint8)
    res, plane = np.array([[4.0]]), np.array([[0.0, 0.1, 1.0, -20.0]])
    r = E.eval_dtu(vmm, f, torch.from_numpy(gt).to(dev), obs, bb, res, plane, seed=3)
    pcd = r["stages"]["data_pcd"]
    fn = f.cpu().numpy()
    p = P.eval_dtu(vn, fn, gt, obs, bb, res, plane, E.seeded_permutation(pcd.shape[0], 3))
    assert np.array_equal(pcd.cpu().numpy(), p["data_pcd"])
    assert np.array_equal(r["stages"]["downsample"]["kept_index"].cpu().numpy(), p["kept_index"])
    _ulp_equal(r["stages"]["dist_d2s"].cpu().numpy(), p["dist_d2s"], 20.0)
    _ulp_equal(r["stages"]["dist_s2d"].cpu().numpy(), p["dist_s2d"], 20.0)
    for k in ("mean_d2gt", "mean_gt2d", "over_all"):
        assert abs(r[k] - p[k]) <= 1e-12 * abs(p[k])
    for k in ("precision_1", "recall_1", "fscore_1", "precision_2", "recall_2", "fscore_2"):
        assert r[k] == p[k]
    print("udf_mesh N=128: %d faces, %d points, %d kept, rounds %d, over_all %.6f mm" % (
        f.shape[0], pcd.shape[0], r["n_down"], r["downsample_rounds"], r["over_all"]))


def _write_mesh_ply(path, v, f):
    """binary PLY as trimesh exports it (float vertices, uchar-int face lists)"""
    head = ("ply\nformat binary_little_endian 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
            "element face %d\nproperty list uchar int vertex_indices\nend_header\n" % (len(v), len(f)))
    fd = np.zeros(len(f), dtype=[("n", "u1"), ("i", "<i4", (3,))])
    fd["n"], fd["i"] = 3, f
    with open(path, "wb") as fh:
        fh.write(head.encode())
        fh.write(np.ascontiguousarray(v, "<f4").tobytes())
        fh.write(fd.tobytes())


def test_cli_dtu(tmp_path):
    _dev()
    from scipy.io import savemat
    from neuraludf_b200 import evaluate as E
    fx = Fixtures("eval_dtu_sphere")
    v = fx["data"].astype(np.float32)
    _write_mesh_ply(str(tmp_path / "mesh.ply"), v, fx["faces"])
    E.write_ply_points(str(tmp_path / "stl.ply"), fx["gt"])
    os.makedirs(tmp_path / "ObsMask")
    savemat(str(tmp_path / "ObsMask" / "ObsMask5_10.mat"), {"ObsMask": fx["obs_mask"], "BB": fx["bb"], "Res": fx["res"]})
    savemat(str(tmp_path / "ObsMask" / "Plane5.mat"), {"P": fx["plane"]})
    cmd = [sys.executable, "-m", "neuraludf_b200.evaluate", "dtu", "--data", str(tmp_path / "mesh.ply"), "--gt",
           str(tmp_path / "stl.ply"), "--scan", "5", "--dataset_dir", str(tmp_path), "--patch_size", "1", "--seed", "4",
           "--vis_out_dir", str(tmp_path / "vis"), "--log", str(tmp_path / "log.txt")]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    # the proto on the same inputs: the float32 vertices of the file and the seed's permutation
    v64 = v.astype(np.float64)
    n = len(P.sample_mesh(v64, fx["faces"], 0.2))
    p = P.eval_dtu(v64, fx["faces"], fx["gt"], fx["obs_mask"], fx["bb"], fx["res"], fx["plane"], E.seeded_permutation(n, 4),
                   patch=1.0)
    lines = out.stdout.strip().splitlines()
    assert lines[-3].startswith("over_all: ") and lines[-2].startswith("precision_1mm: ")
    vals = dict(tok.split(": ") for tok in lines[-3].rstrip(".").split("; "))
    assert abs(float(vals["over_all"]) - p["over_all"]) <= 1e-12 * abs(p["over_all"])
    log = (tmp_path / "log.txt").read_text()
    assert log.endswith("[mesh] \n") and log.count("\n") == 4 and log.startswith("over_all ")
    got_pts, _ = E.read_ply(str(tmp_path / "vis" / "vis_005_d2gt.ply"))
    assert np.array_equal(got_pts, p["data_down"])
    assert np.array_equal(E.read_ply_colors(str(tmp_path / "vis" / "vis_005_gt2d.ply")),
                          np.round(p["gt_color"] * 255).astype(np.uint8))

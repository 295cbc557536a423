"""Mesh post-processing on the device (neuraludf_b200/mesh_post.py, csrc/mesh_post.cu): the kernels against their NumPy
restatement (tests/proto/mesh_post.py) bit for bit on every golden and crafted case, the device MC's coincident sheets and
the C5 network's band meshes at 256^3 and 512^3; determinism; `udf_mesh_post` against the unmodified get_mesh_udf_fast
under the restated trimesh rules; the CLI; and mesh -> postprocess -> clean_dtu_mesh -> eval_dtu on device tensors."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import make_ref, refshim
from tests.golden_util import Fixtures
from tests.proto import mesh_cases as C
from tests.proto import mesh_post as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_CASES = sorted(C.CASES) + ["network", "holes", "figure8", "duplicates", "slivers", "nan", "closed", "book"]


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def c5(golden):
    _dev()
    from tests.gpu_util import build_modules
    return build_modules(golden, "cuda")[0]


def _same(dv, df, dinfo, pv, pf, pinfo):
    """device result == restatement, bit for bit (same numbering, same order)"""
    assert np.array_equal(df.cpu().numpy(), pf)
    a = dv.cpu().numpy()
    assert a.shape == pv.shape and np.array_equal(a.view(np.int64), pv.view(np.int64))
    for k in ("process", "hole_faces", "loop", "passes", "border_vertices", "output"):
        assert dinfo[k] == pinfo[k], k


def _check(verts, faces, dev):
    pv, pf, pinfo = P.postprocess(verts, faces)
    from neuraludf_b200 import mesh_post
    dv, df, dinfo = mesh_post.postprocess(torch.from_numpy(np.asarray(verts, np.float64)).to(dev),
                                          torch.from_numpy(np.asarray(faces, np.int64)).to(dev))
    _same(dv, df, dinfo, pv, pf, pinfo)
    ev, ef = mesh_post.export_merge(dv, df)
    pev, pef = P.export_merge(pv, pf)
    assert np.array_equal(ef.cpu().numpy(), pef) and np.array_equal(ev.cpu().numpy(), pev)
    return dv, df, dinfo


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_kernels_match_restatement(name):
    dev = _dev()
    fx = Fixtures("post_" + name)
    _, _, info = _check(fx["in_verts"], fx["in_faces"], dev)
    print("%s: %s, hole faces %d, passes %d, border vertices %d" % (name, info["process"], info["hole_faces"], info["passes"],
                                                                    info["border_vertices"]))


def test_device_mc_coincident_sheets():
    """the device MC emits two coincident sheets where the surface passes through lattice points: they merge and the
    duplicates go"""
    dev = _dev()
    from neuraludf_b200 import mesh
    df, nrm, N = C.field("plane")
    idx = np.nonzero(df < 2 * (2.0 / (N - 1)))[0].astype(np.int64)
    v, f, _ = mesh.marching_cubes_index(torch.from_numpy(df).to(dev), (N, N, N), torch.from_numpy(nrm[idx]).to(dev),
                                        torch.from_numpy(idx).to(dev))
    vw = P.world64(v.cpu().numpy(), N)
    _, _, info = _check(vw, f.cpu().numpy(), dev)
    assert info["process"]["duplicate"] > 0
    print("plane, device MC: %s" % info["process"])


@pytest.mark.parametrize("N", [256, 512])
def test_band_meshes_match_restatement(c5, N):
    dev = _dev()
    from neuraludf_b200 import grid, mesh, mesh_post
    voxel = 2.0 / (N - 1)
    df, _ = grid.udf_band(c5, N)
    vi, faces = mesh._mc_lattice(c5, N, df, 0, 1 << 21)
    v64 = vi.double() * voxel - 1.0
    assert np.array_equal(v64.cpu().numpy(), P.world64(vi.cpu().numpy(), N))
    vd = c5.udf_values(v64.float()).reshape(-1)
    faces = faces[vd[faces].max(dim=1).values < voxel * 5.0]
    dv, dfc, info = _check(v64.cpu().numpy(), faces.cpu().numpy(), dev)
    v1, f1, _ = mesh.udf_mesh_post(c5, N)
    v2, f2, _ = mesh.udf_mesh_post(c5, N)
    assert torch.equal(v1, dv) and torch.equal(f1, dfc)
    assert torch.equal(v1, v2) and torch.equal(f1, f2)                      # bit-identical, run to run
    print("C5 band %d^3: %d faces -> %s, hole faces %d, border vertices %d, (V, F) %s"
          % (N, faces.shape[0], info["process"], info["hole_faces"], info["border_vertices"], info["output"]))


@pytest.mark.skipif(not os.path.isfile(os.path.join(refshim.REFERENCE_ROOT, "extract_mesh.py")) or not make_ref.available(),
                    reason="no staged reference copy")
def test_pipeline_matches_reference(c5):
    """udf_mesh_post at N = 128 against the unmodified get_mesh_udf_fast (trimesh stub) driven by the device drop-in MC on
    the same lattice and the same udf values"""
    dev = _dev()
    from neuraludf_b200 import grid, mesh, mesh_post
    from oracle import ref_post
    N = 128
    df = grid.udf_grid(c5, N)
    idx, nrm = grid.near_surface_cells(c5, N, df)
    dense = torch.zeros(N ** 3, 3, device=dev)
    dense[idx] = nrm
    r = ref_post.run_post(df.cpu().numpy(), dense.cpu().numpy(), N, mesh.udf_mc_lewiner,
                          lambda x: c5.udf_values(x).reshape(-1, 1), dist_threshold_ratio=5.0, device="cuda")
    v, f, info = mesh.udf_mesh_post(c5, N, dense=True)
    ev, ef = mesh_post.export_merge(v, f)
    gv, gf = P.canonical(r["verts"], r["faces"])
    cv, cf = P.canonical(ev.cpu().numpy(), ef.cpu().numpy())
    assert info["filtered"] == len(r["input"][1])
    assert np.array_equal(cf, gf)
    assert float(np.abs(cv - gv).max()) <= 1e-12
    assert r["smoothed"] == (info["border_vertices"] > 0)
    print("N=128: MC %s, filtered %d, %s, hole faces %d, border vertices %d, networkx disagreements %d, max |dv| %.1e"
          % (info["mc"], info["filtered"], info["process"], info["hole_faces"], info["border_vertices"],
             r["nx_disagreements"], float(np.abs(cv - gv).max())))


def test_cli_postprocess(c5, tmp_path):
    from neuraludf_b200 import mesh, mesh_post
    from neuraludf_b200.evaluate import read_ply
    ckpt, cams, out = (os.path.join(str(tmp_path), n) for n in ("ckpt_000100.pth", "cameras_sphere.npz", "mesh.ply"))
    torch.save({"udf_network_fine": c5.state_dict(), "iter_step": 100}, ckpt)
    sm = np.eye(4)
    sm[0, 0] = sm[1, 1] = sm[2, 2] = 212.5
    sm[:3, 3] = [-10.25, 3.5, 620.0]
    np.savez(cams, scale_mat_0=sm, world_mat_0=np.eye(4))
    r = subprocess.run([sys.executable, "-m", "neuraludf_b200.mesh", "--ckpt", ckpt, "--resolution", "128", "--cameras", cams,
                        "--dist_threshold_ratio", "5", "--postprocess", "--out", out], cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    v, f = read_ply(out)
    v1, f1, _ = mesh.udf_mesh_post(c5, 128)
    s32 = sm.astype(np.float32)
    w = torch.from_numpy(v1.cpu().numpy() * s32[0, 0] + s32[:3, 3][None]).cuda()
    ev, ef = mesh_post.export_merge(w, f1)
    assert f.shape[0] > 1000
    assert np.array_equal(v, ev.cpu().numpy()) and np.array_equal(f, ef.cpu().numpy())


def test_post_clean_eval_on_device(c5):
    """udf_mesh_post at N = 128, to world space (mm), clean_dtu_mesh under a ring of cameras, eval_dtu: device tensors
    throughout, each step against its restatement"""
    dev = _dev()
    from neuraludf_b200 import clean as CL
    from neuraludf_b200 import evaluate as E
    from neuraludf_b200 import mesh, mesh_post
    from tests.proto import clean_cases as CC
    from tests.proto import eval_pc as EP
    from tests.proto import mesh_clean as M
    v, f, _ = mesh.udf_mesh_post(c5, 128)
    assert v.is_cuda and f.is_cuda and f.shape[0] > 1000
    vw, fw = mesh_post.export_merge(v * 100.0 + torch.tensor([3.0, -2.0, 1.0], dtype=torch.float64, device=dev), f)
    vn, fn = vw.cpu().numpy(), fw.cpu().numpy()
    centre = vn.mean(0)
    mats = CC.ring(12, dist=450.0, seed=9)
    masks = np.stack([CC.silhouette(Pm, centre, np.percentile(np.linalg.norm(vn - centre, axis=1), 60)) for Pm in mats])
    (v1, f1, _), (v2, f2, _) = CL.clean_dtu_mesh(vw, fw, mats, torch.from_numpy(masks).to(dev))
    pst = M.clean_dtu_mesh(vn, fn, mats, masks)
    pf1, pf2 = pst[0][1], pst[1][1]
    assert np.array_equal(f1.cpu().numpy(), pf1) and np.array_equal(f2.cpu().numpy(), pf2)
    assert 0 < f2.shape[0] < fw.shape[0]
    r2, rf2 = v2.cpu().numpy(), f2.cpu().numpy()
    rng = np.random.default_rng(4)
    m = min(len(r2), 30000)
    gt = r2[rng.choice(len(r2), m, replace=False)] + 0.3 * rng.normal(size=(m, 3))
    bb = np.array([centre - 110.0, centre + 110.0])
    obs = np.ones((56, 56, 56), np.uint8)
    res, plane = np.array([[4.0]]), np.array([[0.0, 0.0, 1.0, 200.0]])
    r = E.eval_dtu(v2, f2, torch.from_numpy(gt).to(dev), obs, bb, res, plane, seed=3)
    p = EP.eval_dtu(r2, rf2, gt, obs, bb, res, plane, E.seeded_permutation(r["n_points"], 3))
    for k in ("mean_d2gt", "mean_gt2d", "over_all"):
        assert abs(r[k] - p[k]) <= 1e-12 * abs(p[k])
    print("udf_mesh_post N=128: %d -> %d -> %d faces, over_all %.4f mm" % (fw.shape[0], f1.shape[0], f2.shape[0], r["over_all"]))

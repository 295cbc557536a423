"""CUDA MeshUDF marching cubes (neuraludf_b200/mesh.py, csrc/mesh_udf.cu) against its NumPy restatement
(tests/proto/udf_mc.py) on every golden mesh, the `udf_mc_lewiner` drop-in against the reference's conventions, `udf_mesh`
against the reference pipeline, and the unmodified runner meshing through the new MC."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import make_ref_mc, refshim
from tests.golden_util import Fixtures
from tests.proto import mesh_cases as C
from tests.proto import udf_mc as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _inputs(name):
    if name == "random":         # random udf and normals: every cell active, many loops that need a centre vertex
        N = 24
        rng = np.random.default_rng(7)
        df = (rng.uniform(0.02, 1.0, N ** 3) * (2.0 / (N - 1))).astype(np.float32)
        g = rng.normal(size=(N ** 3, 3))
        return df, N, np.arange(N ** 3, dtype=np.int64), (g / np.linalg.norm(g, axis=1, keepdims=True)).astype(np.float32)
    if name == "network":
        fx = Fixtures("mesh_network")
        return fx["df"], 48, fx["idx"], fx["normals"]
    df, nrm, N = C.field(name)
    idx = np.nonzero(df < 2 * (2.0 / (N - 1)))[0].astype(np.int64)      # the sparse hand-off of grid.near_surface_cells
    return df, N, idx, nrm[idx]


@pytest.mark.parametrize("name", sorted(C.CASES) + ["network", "random"])
def test_cuda_matches_prototype(name):
    _need_gpu()
    from neuraludf_b200 import mesh
    df, N, idx, nrm = _inputs(name)
    pv, pf, pinfo = P.marching_cubes(df, (N, N, N), nrm, idx)
    dev = torch.device("cuda", 0)
    v, f, info = mesh.marching_cubes_index(torch.from_numpy(df).to(dev), (N, N, N), torch.from_numpy(nrm).to(dev),
                                           torch.from_numpy(idx).to(dev))
    assert np.array_equal(info["active"].cpu().numpy(), pinfo["active"])
    assert np.array_equal(info["mask"].cpu().numpy(), pinfo["mask"])
    assert np.array_equal(info["face_keys"].cpu().numpy(), pinfo["face_keys"])     # same faces, same order
    assert np.array_equal(f.cpu().numpy(), pf)
    if name == "random":
        assert int((info["vertex_keys"] >= 3 * N ** 3).sum()) > 50            # loop-centre vertices exercised
    # the polarity union-find: a handful of hooking rounds (cells are numbered by lattice index)
    print("%s: polarity rounds %d, pointer-jumping passes %d" % (name, info["polarity_rounds"], info["polarity_jumps"]))
    assert 1 <= info["polarity_rounds"] <= 16
    vw, _ = mesh.udf_marching_cubes(torch.from_numpy(df).to(dev), N, torch.from_numpy(idx).to(dev),
                                    torch.from_numpy(nrm).to(dev))
    assert float(np.abs(vw.cpu().numpy() - P.to_world(pv, N)).max()) <= 1e-6
    assert torch.isfinite(vw).all()


def test_drop_in_conventions():
    _need_gpu()
    from neuraludf_b200 import mesh
    fx = Fixtures("mesh_sphere")
    df, nrm, N = C.field("sphere")
    voxel = 2.0 / (N - 1)
    vol, gr = df.reshape(N, N, N), nrm.reshape(N, N, N, 3)
    v, f, n, val = mesh.udf_mc_lewiner(vol, gr, spacing=[voxel] * 3)
    assert v.shape[1] == 3 and f.shape[1] == 3 and n.shape == v.shape and val.shape == (len(v),)
    assert f.dtype == np.int32 and n.dtype == np.float32 and val.dtype == np.float32
    from scipy.spatial import cKDTree
    d, _ = cKDTree(v).query(fx["ref_verts"] + 1)                            # array-index order, scaled by spacing
    assert len(v) == len(fx["ref_verts"]) and d.max() < 1e-4 * voxel
    w = v - 1
    nf = np.cross(w[f[:, 1]] - w[f[:, 0]], w[f[:, 2]] - w[f[:, 0]])
    rv, rf = fx["ref_verts"], fx["ref_faces"]
    rn = np.cross(rv[rf[:, 1]] - rv[rf[:, 0]], rv[rf[:, 2]] - rv[rf[:, 0]])
    assert np.sign((nf * w[f].mean(1)).sum(1)).mean() == np.sign((rn * rv[rf].mean(1)).sum(1)).mean() == 1.0
    _, fa, _, _ = mesh.udf_mc_lewiner(vol, gr, gradient_direction="ascent")
    assert np.array_equal(fa, f[:, ::-1])
    with pytest.raises(ValueError):
        mesh.udf_mc_lewiner(vol[0], gr[0])
    with pytest.raises(ValueError):
        mesh.udf_mc_lewiner(vol[:1], gr[:1])
    with pytest.raises(ValueError):
        mesh.udf_mc_lewiner(vol, gr, gradient_direction="up")
    with pytest.raises(RuntimeError, match="No surface found at the given iso value."):
        mesh.udf_mc_lewiner(np.ones((8, 8, 8), np.float32), np.zeros((8, 8, 8, 3), np.float32))
    with pytest.raises(NotImplementedError):
        mesh.udf_mc_lewiner(vol, gr, step_size=2)
    with pytest.raises(NotImplementedError):
        mesh.udf_mc_lewiner(vol, gr, mask=np.ones(vol.shape, bool))


@pytest.mark.skipif(not os.path.isfile(os.path.join(refshim.REFERENCE_ROOT, "extract_mesh.py")) or not make_ref_mc.verify(),
                    reason="no staged reference copy / compiled reference MC")
def test_udf_mesh_against_reference_pipeline(golden):
    _need_gpu()
    from neuraludf_b200 import mesh
    from tests.gpu_util import build_modules
    from tests.test_gpu_grid import _ref_extract_mesh
    udf = build_modules(golden, "cuda")[0]
    N = 128
    voxel = 2.0 / (N - 1)
    v, f = mesh.udf_mesh(udf, N)
    assert f.shape[0] > 1000
    assert float(udf.udf_values(v).max()) < voxel                             # every kept vertex passes the filter

    def func_grad(xyz):                                                        # exp_runner_blending.py:767-771
        g = udf.gradient(xyz)
        return g / (torch.linalg.norm(g, ord=2, dim=-1, keepdim=True) + 1e-5)

    em = _ref_extract_mesh()
    torch.set_default_tensor_type("torch.cuda.FloatTensor")
    try:
        df, vecs, _ = em.get_udf_normals_grid_slow(udf.udf, func_grad, N=N, max_batch=1 << 18)
    finally:
        torch.set_default_tensor_type("torch.FloatTensor")
    ref = make_ref_mc.load()
    rv, rf, _, _ = ref.udf_mc_lewiner(df.cpu().numpy(), vecs.cpu().numpy(), spacing=[voxel] * 3)
    rv = rv - 1
    with torch.no_grad():
        rd = udf.udf(torch.from_numpy(rv).float().cuda()).cpu().numpy()
    rff = rf[np.max(rd[rf], axis=1)[:, 0] < voxel]
    vn, fn = v.cpu().numpy().astype(np.float64), f.cpu().numpy()
    # Chamfer between the vertex sets: at N = 128 a 20k-sample surface Chamfer sits at its own sampling floor
    # (~0.44 voxel for two identical face counts, measured), so the vertices are compared directly
    from scipy.spatial import cKDTree
    kept = np.unique(rff)
    cd = 0.5 * (cKDTree(rv[kept]).query(vn)[0].mean() + cKDTree(vn).query(rv[kept])[0].mean()) / voxel
    print("udf_mesh N=128: %d faces (reference %d), vertex chamfer %.2e voxel" % (len(fn), len(rff), cd))
    assert cd < 0.05
    a = C.mesh_stats(vn, fn)["area"] / C.mesh_stats(rv, rff)["area"]
    assert 0.98 < a < 1.02
    stats = C.mesh_stats(vn, fn)
    assert stats["nonmanifold"] == 0 and stats["same_direction"] == 0
    v1, f1 = mesh.udf_mesh(udf, 256)
    v2, f2 = mesh.udf_mesh(udf, 256)
    assert torch.equal(v1, v2) and torch.equal(f1, f2)                         # bit-identical, run to run


DRIVER = """
import sys
sys.path.insert(0, {root!r})
from tests import runner_env
runner_env.install_stubs()
for k in ("custom_mc", "custom_mc._marching_cubes_lewiner"):
    sys.modules.pop(k, None)                      # served by neuraludf_b200.mesh through the launcher
import torch
_load = torch.load
torch.load = lambda *a, **k: _load(*a, **dict(dict(weights_only=False), **k))
from neuraludf_b200 import launch, mesh
_mc = mesh.udf_mc_lewiner
def _recorded(volume, grads, **kw):
    out = _mc(volume, grads, **kw)
    print("MC_CALL shape=%s verts=%d faces=%d" % (volume.shape, len(out[0]), len(out[1])), flush=True)
    return out
mesh.udf_mc_lewiner = _recorded
try:
    rc = launch.main({argv!r})
except NotImplementedError as e:
    if "trimesh" not in str(e):
        raise
    print("REACHED_TRIMESH_STUB_AFTER_MC")
    rc = 0
sys.exit(rc)
"""


@pytest.mark.skipif(not refshim.available(), reason="no staged reference copy (oracle/make_ref.py)")
def test_unmodified_runner_meshes_through_cuda_mc(tmp_path):
    _need_gpu()
    from oracle import make_ref
    from tests import runner_env
    src = refshim.REFERENCE_ROOT
    ref = os.path.join(str(tmp_path), "ref")                  # the runner tree without any custom_mc build
    for rel in make_ref.PATH_FILES + make_ref.CALLER_FILES:
        if os.path.isfile(os.path.join(src, rel)):
            os.makedirs(os.path.dirname(os.path.join(ref, rel)), exist_ok=True)
            shutil.copyfile(os.path.join(src, rel), os.path.join(ref, rel))
    tmp = str(tmp_path)
    runner_env.write_synthetic_dtu(os.path.join(tmp, "data", "synth"), n_images=12, width=96, height=72)
    exp = os.path.join(tmp, "exp", "CASE_NAME") + "/"
    conf = runner_env.write_conf(ref, os.path.join(tmp, "synth.conf"), os.path.join(tmp, "data", "CASE_NAME") + "/", exp,
                                 end_iter=2, batch_size=256, save_freq=2, val_freq=100)
    drv = os.path.join(tmp, "drive.py")
    with open(drv, "w") as fh:
        fh.write(DRIVER.format(root=ROOT, argv=[os.path.join(ref, "exp_runner_blending.py"), "--mode", "train", "--conf",
                                                conf, "--case", "synth", "--gpu", "0"]))
    r = subprocess.run([sys.executable, drv], cwd=tmp, env=dict(os.environ, PYTHONUNBUFFERED="1"), capture_output=True,
                       text=True, timeout=1200)
    tail = r.stdout[-3000:] + "\n---- stderr ----\n" + r.stderr[-3000:]
    assert r.returncode == 0, tail
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("MC_CALL")]
    assert lines and "(512, 512, 512)" in lines[-1], tail
    assert int(lines[-1].split("faces=")[1]) > 0, tail
    assert "REACHED_TRIMESH_STUB_AFTER_MC" in r.stdout, tail

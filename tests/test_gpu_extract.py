"""get_mesh_udf_fast on the device (neuraludf_b200/extract_mesh.py, csrc/mesh_grad.cu): the gradient-branch kernels
against their NumPy restatement (tests/proto/mesh_grad.py) on the golden cases and the C5 network's band meshes; the shadow
against the unmodified get_mesh_udf_fast (trimesh stub, device MC drop-in) through the runner's try/except; its raise,
band, gradient=False and samples behaviour; and the unmodified runner with NUDF_DEVICE_MESH=1."""
import glob
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import make_ref, refshim
from tests.golden_util import Fixtures
from tests.proto import mesh_grad as G
from tests.proto import mesh_post as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_CASES = ["sheet", "closed", "empty", "lattice", "network"]
EPS = 0.005
has_ref = pytest.mark.skipif(not os.path.isfile(os.path.join(refshim.REFERENCE_ROOT, "extract_mesh.py"))
                             or not make_ref.available(), reason="no staged reference copy")


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def c5(golden):
    _dev()
    from tests.gpu_util import build_modules
    return build_modules(golden, "cuda")[0]


def _runner_func_grad(net):
    def func_grad(xyz):                       # exp_runner_blending.py:767-771
        gradients = net.gradient(xyz)
        gradients_mag = torch.linalg.norm(gradients, ord=2, dim=-1, keepdim=True)
        return gradients / (gradients_mag + 1e-5)
    return func_grad


def _ulps(a, b):
    """fp32 ulp distance per element (same-sign values; zeros of either sign equal)"""
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, np.int64(-(1 << 31)) - ia, ia)
    ib = np.where(ib < 0, np.int64(-(1 << 31)) - ib, ib)
    return np.abs(ia - ib)


def _kernels_vs_restatement(v64, faces, func, eps, N, what):
    """vertex_normals / probes / refine on the device against the restatement; s1, s2 = func at the device probes fed to
    both.  Returns (normal components off by one ulp, vertices whose normals differ)."""
    from neuraludf_b200 import extract_mesh as X
    dev = _dev()
    vt = torch.from_numpy(np.asarray(v64, np.float64)).to(dev)
    ft = torch.from_numpy(np.asarray(faces, np.int64)).to(dev)
    nd = X.vertex_normals(vt, ft).cpu().numpy()
    assert np.array_equal(X.vertex_normals(vt, ft).cpu().numpy().view(np.int32), nd.view(np.int32))   # run to run
    npr = G.vertex_normals(v64, faces)
    u = _ulps(nd, npr)
    assert int(u.max(initial=0)) <= 1, what
    same = (u == 0).all(1)
    nv, ni = X.refine(func, vt, ft, eps, N)
    nv2, ni2 = X.refine(func, vt, ft, eps, N)
    assert torch.equal(nv, nv2) and np.array_equal(ni, ni2)                                                # run to run
    v32 = np.asarray(v64, np.float64).astype(np.float32)
    p1, p2 = G.probes(v32, nd, eps)                    # the device normals: the probe values then match the device's
    s1 = func(torch.from_numpy(p1).to(dev)).reshape(-1).cpu().numpy()
    s2 = func(torch.from_numpy(p2).to(dev)).reshape(-1).cpu().numpy()
    pnv = G.refine(v32, nd, s1, s2, eps)
    assert np.array_equal(nv.cpu().numpy(), pnv)                                       # by value: +-0 equal
    assert np.array_equal(ni, G.next_indices(pnv, N))
    # with the restatement's own normals: equal wherever the normals are
    qnv = G.refine(v32, npr, s1, s2, eps)
    assert np.array_equal(nv.cpu().numpy()[same], qnv[same])
    print("%s: %d vertices, %d normal components 1 ulp off (%d vertices)" % (what, len(v32), int((u == 1).sum()),
                                                                            int((~same).sum())))


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_kernels_match_restatement(name):
    dev = _dev()
    from neuraludf_b200 import extract_mesh as X
    fx = Fixtures("grad_" + name)
    v, f, eps, N = fx["mesh_verts"], fx["mesh_faces"], float(fx["eps"]), int(fx["N"])
    s1, s2 = fx["s1"], fx["s2"]
    calls = iter([torch.from_numpy(s1).to(dev), torch.from_numpy(s2).to(dev)] * 2)
    vt, ft = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
    nd = X.vertex_normals(vt, ft).cpu().numpy()
    same = (_ulps(nd, G.vertex_normals(v, f)) == 0).all(1)
    assert int(_ulps(nd, G.vertex_normals(v, f)).max(initial=0)) <= 1
    nv, ni = X.refine(lambda x: next(calls), vt, ft, eps, N)
    nv = nv.cpu().numpy()
    assert np.array_equal(nv[same], fx["new_verts"][same])
    if same.all():
        assert np.array_equal(ni, fx["next_indices"])
    print("%s: %d vertices, %d with a normal 1 ulp off" % (name, len(v), int((~same).sum())))


@pytest.mark.parametrize("N", [256, 512])
def test_band_meshes_match_restatement(c5, N):
    from neuraludf_b200 import mesh
    v, f, _ = mesh.udf_mesh_post(c5, N)
    _kernels_vs_restatement(v.cpu().numpy(), f.cpu().numpy(), lambda x: c5.udf_values(x), EPS, N, "C5 band %d^3" % N)


def _lattice(func, func_grad, N):
    """the dense lattice get_udf_normals_grid_fast would return for func / func_grad: (df [N^3], normals [N^3,3]) NumPy"""
    from neuraludf_b200 import extract_mesh as X
    from neuraludf_b200 import grid
    field = X.CallerField(func, func_grad)
    with torch.no_grad():
        df = grid.udf_grid(field, N, max_batch=X.LATTICE_BATCH)
        idx, nrm = grid.near_surface_cells(field, N, df, max_batch=X.LATTICE_BATCH // 2)
    dense = torch.zeros(N ** 3, 3, device=df.device)
    dense[idx] = nrm
    return df.cpu().numpy(), dense.cpu().numpy()


def _runner_call(gmuf, func, func_grad, N, ratio=5.0):
    """Runner.extract_udf_mesh's two calls (exp_runner_blending.py:777-790): (output tuple, first call raised)"""
    try:
        return gmuf(func, func_grad, samples=None, indices=None, N_MC=N, gradient=True, eps=EPS, border_gradients=True,
                    smooth_borders=True, dist_threshold_ratio=ratio), False
    except Exception:
        return gmuf(func, func_grad, samples=None, indices=None, N_MC=N, gradient=True, eps=EPS, border_gradients=False,
                    smooth_borders=False, dist_threshold_ratio=ratio), True


def _same_as_reference(out, fell_back, r):
    """the shadow's runner call against ref_grad.run_grad's: exported mesh, fallback, new_verts and next_indices"""
    from neuraludf_b200 import mesh_post
    from neuraludf_b200.extract_mesh import vertex_normals
    ev, ef = mesh_post.export_merge(torch.from_numpy(out[2].vertices).cuda(), torch.from_numpy(out[2].faces).cuda())
    gv, gf = P.canonical(r["verts"], r["faces"])
    cv, cf = P.canonical(ev.cpu().numpy(), ef.cpu().numpy())
    assert np.array_equal(cf, gf)
    assert cv.shape == gv.shape and (len(cv) == 0 or float(np.abs(cv - gv).max()) <= 1e-12)
    assert fell_back == (not r["smoothed"])
    assert out[3] is None and out[4].dtype == np.int64 and out[0].dtype == torch.float32
    rv, rf = r["mesh"]
    if rf.shape == out[2].faces.shape and np.array_equal(rf, out[2].faces) and np.array_equal(rv, out[2].vertices):
        # the same mesh into the branch: new_verts / next_indices equal wherever the normals are
        n_dev = vertex_normals(torch.from_numpy(rv).cuda(), torch.from_numpy(rf).cuda()).cpu().numpy()
        same = (_ulps(n_dev, G.vertex_normals(rv, rf)) == 0).all(1)
        assert np.array_equal(out[0].cpu().numpy()[same], r["new_verts"][same])
        ni, rni = out[4].reshape(7, -1), r["next_indices"].reshape(7, -1)
        assert np.array_equal(ni[:, same], rni[:, same])
        return int((~same).sum()), True
    return -1, False


@has_ref
def test_shadow_matches_reference(c5):
    """N = 128 on C5 with the runner's func / func_grad: the shadow against the unmodified get_mesh_udf_fast"""
    from neuraludf_b200 import extract_mesh as X
    from neuraludf_b200 import mesh
    from oracle import ref_grad
    N = 128
    func, func_grad = c5.udf, _runner_func_grad(c5)
    df, dense = _lattice(func, func_grad, N)
    r = ref_grad.run_grad(df, dense, N, mesh.udf_mc_lewiner, func, func_grad, dist_threshold_ratio=5.0, device="cuda")
    info = {}
    out, fell_back = _runner_call(lambda *a, **k: X.get_mesh_udf_fast(*a, info=info, **k), func, func_grad, N)
    off, same_mesh = _same_as_reference(out, fell_back, r)
    assert same_mesh                                   # the reference's mesh and the shadow's, vertex for vertex
    print("C5 N=128: fallback %s, MC %s, filtered %d, output %s, normals 1 ulp off at %d vertices, stage ms %s"
          % (fell_back, info["mc"], info["filtered"], info["output"], off,
             {k: round(v, 2) for k, v in info["stage_ms"].items()}))


def _sphere_fields(dev, r=0.5):
    def func(x):
        return (torch.linalg.norm(x, dim=1, keepdim=True) - r).abs()

    def func_grad(x):
        n = torch.linalg.norm(x, dim=1, keepdim=True)
        return (x / n * torch.sign(n - r)).unsqueeze(1)
    return func, func_grad


@has_ref
def test_closed_surface_falls_back():
    dev = _dev()
    from neuraludf_b200 import extract_mesh as X
    from neuraludf_b200 import mesh
    from oracle import ref_grad
    N = 64
    func, func_grad = _sphere_fields(dev)
    with pytest.raises(IndexError):
        X.get_mesh_udf_fast(func, func_grad, N_MC=N, gradient=True, eps=EPS, border_gradients=True, smooth_borders=True,
                            dist_threshold_ratio=5.0)
    with pytest.raises(IndexError):                    # no smoothing, but border gradients
        X.get_mesh_udf_fast(func, func_grad, N_MC=N, gradient=True, eps=EPS, border_gradients=True, smooth_borders=False,
                            dist_threshold_ratio=5.0)
    out, fell_back = _runner_call(X.get_mesh_udf_fast, func, func_grad, N)
    assert fell_back and out[2].faces.shape[0] > 1000
    df, dense = _lattice(func, func_grad, N)
    r = ref_grad.run_grad(df, dense, N, mesh.udf_mc_lewiner, func, func_grad, dist_threshold_ratio=5.0, device="cuda")
    off, same_mesh = _same_as_reference(out, fell_back, r)
    assert same_mesh
    print("sphere N=64: %d faces, normals 1 ulp off at %d vertices" % (out[2].faces.shape[0], off))


def test_band_equals_dense(c5, monkeypatch):
    from neuraludf_b200 import extract_mesh as X
    func, func_grad = c5.udf, _runner_func_grad(c5)
    outs = []
    for flag in ("0", "1"):
        monkeypatch.setenv("NUDF_BAND_MESH", flag)
        outs.append(_runner_call(X.get_mesh_udf_fast, func, func_grad, 128))
    (a, fa), (b, fb) = outs
    assert fa == fb
    assert np.array_equal(a[2].vertices, b[2].vertices) and np.array_equal(a[2].faces, b[2].faces)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and np.array_equal(a[4], b[4])


def test_gradient_false_and_samples(c5):
    from neuraludf_b200 import extract_mesh as X
    func, func_grad = c5.udf, _runner_func_grad(c5)
    kw = dict(N_MC=96, eps=EPS, border_gradients=False, smooth_borders=False, dist_threshold_ratio=5.0)
    out = X.get_mesh_udf_fast(func, func_grad, gradient=False, **kw)
    assert len(out) == 3
    v, f, m = out
    assert v.dtype == torch.float32 and v.is_cuda and f.dtype == torch.int64 and f.is_cuda
    assert m.vertices.dtype == np.float64 and m.faces.dtype == np.int64
    assert np.array_equal(v.cpu().numpy(), m.vertices.astype(np.float32)) and np.array_equal(f.cpu().numpy(), m.faces)
    g = X.get_mesh_udf_fast(func, func_grad, gradient=True, **kw)
    assert len(g) == 5 and np.array_equal(g[2].vertices, m.vertices) and g[4].shape == (7 * len(m.vertices),)
    with pytest.raises(NotImplementedError):
        X.get_mesh_udf_fast(func, func_grad, samples=torch.zeros(96 ** 3, 7), indices=g[4], gradient=True, **kw)


DRIVER = """
import sys
sys.path.insert(0, {root!r})
from tests import runner_env
runner_env.install_stubs()
import types
import torch
from oracle import ref_post
from neuraludf_b200.evaluate import write_ply_mesh


class Trimesh(ref_post.Trimesh):
    def export(self, path, *a, **k):
        write_ply_mesh(path, self.vertices, self.faces)


tm = ref_post.trimesh_stub()
tm.Trimesh = Trimesh
tm.smoothing = types.ModuleType("trimesh.smoothing")
sys.modules["trimesh"] = tm
_load = torch.load
torch.load = lambda *a, **k: _load(*a, **dict(dict(weights_only=False), **k))
from neuraludf_b200 import launch
sys.exit(launch.main({argv!r}))
"""


def _run(tmp, argv, timeout=1200):
    drv = os.path.join(tmp, "drive_mesh.py")
    with open(drv, "w") as f:
        f.write(DRIVER.format(root=ROOT, argv=argv))
    env = dict(os.environ, PYTHONUNBUFFERED="1", NUDF_DEVICE_MESH="1")
    env.pop("NUDF_BAND_MESH", None)
    return subprocess.run([sys.executable, drv], cwd=tmp, env=env, capture_output=True, text=True, timeout=timeout)


@pytest.mark.skipif(not refshim.available(), reason="no staged reference copy (oracle/make_ref.py)")
def test_unmodified_runner_meshes_on_device(tmp_path):
    """--mode train finishes with its 512^3 mesh; --mode extract_udf_mesh --is_continue writes the shadow's mesh"""
    _dev()
    from neuraludf_b200 import extract_mesh as X
    from neuraludf_b200 import mesh, mesh_post
    from neuraludf_b200.evaluate import read_ply
    from tests import runner_env
    ref = refshim.REFERENCE_ROOT
    runner = os.path.join(ref, "exp_runner_blending.py")
    tmp = str(tmp_path)
    runner_env.write_synthetic_dtu(os.path.join(tmp, "data", "synth"), n_images=12, width=96, height=72)
    exp = os.path.join(tmp, "exp", "CASE_NAME") + "/"
    conf = runner_env.write_conf(ref, os.path.join(tmp, "synth.conf"), os.path.join(tmp, "data", "CASE_NAME") + "/", exp,
                                 end_iter=2, batch_size=256, save_freq=2, val_freq=100)
    r = _run(tmp, [runner, "--mode", "train", "--conf", conf, "--case", "synth", "--gpu", "0"])
    tail = r.stdout[-3000:] + "\n---- stderr ----\n" + r.stderr[-3000:]
    assert r.returncode == 0, tail
    exp_dir = os.path.join(tmp, "exp", "synth", "udf_dtu")
    assert os.path.isfile(os.path.join(exp_dir, "udf_meshes", "udf_res512_step2.ply")), tail
    r = _run(tmp, [runner, "--mode", "extract_udf_mesh", "--conf", conf, "--case", "synth", "--gpu", "0", "--is_continue",
                   "--resolution", "128"])
    tail = r.stdout[-3000:] + "\n---- stderr ----\n" + r.stderr[-3000:]
    assert r.returncode == 0, tail
    v, f = read_ply(os.path.join(exp_dir, "udf_meshes", "udf_res128_step2.ply"))
    ck = torch.load(sorted(glob.glob(os.path.join(exp_dir, "checkpoints", "ckpt_*.pth")))[-1], map_location="cpu",
                    weights_only=False)
    net = mesh.udf_network_from_state(ck["udf_network_fine"]).cuda()
    out, fell_back = _runner_call(X.get_mesh_udf_fast, net.udf, _runner_func_grad(net), 128)
    # world transform with the synthetic dataset's identity scale_mat (exp_runner_blending.py:793-794), the final Trimesh
    ev, ef = mesh_post.export_merge(torch.from_numpy(out[2].vertices * 1.0 + 0.0).cuda(), torch.from_numpy(out[2].faces).cuda())
    assert f.shape[0] > 100
    assert np.array_equal(f, ef.cpu().numpy()) and np.array_equal(v, ev.cpu().numpy())
    pv, pf, _ = mesh.udf_mesh_post(net, 128, dense=True)                    # the network's own meshing path
    pv, pf = mesh_post.export_merge(pv * 1.0 + 0.0, pf)
    assert torch.equal(pf, ef) and torch.equal(pv, ev)
    print("runner extract_udf_mesh 128^3: %d vertices, %d faces, fallback %s" % (v.shape[0], f.shape[0], fell_back))

"""Surface point clouds on the device (cloud.udf_point_cloud, csrc/udf_cloud.cu, UDFNetwork.value_gradient): the step,
filter and resample kernels bit for bit against their NumPy restatement (tests/proto/udf_cloud.py); the seeds against the
restatement's on the analytic fields' lattices; the pipeline on the analytic fields (on the surface, coverage, count,
determinism, batch invariance); the C5 network against the fp64 oracle; the checkpoint-to-PLY CLI and its scoring."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.gpu_util import parity, report
from tests.proto import udf_cloud as U

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SURFACE_TOL = 1e-6          # tests/test_cloud_proto.py's bound: fp32 rounding of the coordinates, with slack


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _bits(t):
    return t.detach().contiguous().cpu().numpy().view(np.int32)


def _same_bits(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


class _Field:
    """an analytic field on the device: tests/proto/udf_cloud.udf_grad in fp64 with torch, rounded to fp32 once (the same bits
    as the restatement's NumPy field)"""

    def __init__(self, name):
        self.name = name

    def value_gradient(self, x):
        u, g = U.udf_grad(self.name, x.reshape(-1, 3).double(), torch)
        return u.float(), g.float()

    def udf_values(self, x):
        return self.value_gradient(x)[0]


def _crafted(n, seed=0):
    """(p, u, g) fp32: random rows and every kind the step drops or keeps specially, scattered"""
    rng = np.random.default_rng(seed)
    p = rng.uniform(-1, 1, (n, 3)).astype(np.float32)
    u = rng.uniform(0, 0.1, n).astype(np.float32)
    g = rng.normal(size=(n, 3)).astype(np.float32)
    k = rng.integers(0, 10, n)
    u[k == 0] = np.nan
    u[k == 1] = np.inf
    g[k == 2, rng.integers(0, 3)] = np.nan
    g[k == 3] = 0.0
    g[k == 4] = np.float32(1e-30)                                   # |g| underflows to 0
    u[k == 5] = 0.0
    g[k == 6] = np.float32(1e30)                                    # |g| overflows: the step is 0
    p[k == 7] = np.float32(0.999)                                   # many of these leave the box
    g[k == 8, 0] = -np.inf
    return p, u, g


def test_step_kernel_matches_restatement():
    dev = _dev()
    from neuraludf_b200 import cloud
    for n in (1, 255, 257, 100_003):
        p, u, g = _crafted(n, n)
        q, keep = U.step(p, u, g)
        out = cloud.project_step(*(torch.from_numpy(a).to(dev) for a in (p, u, g)))
        assert _same_bits(out.cpu().numpy(), q), n
        report("cloud_step_kernel", n=n, kept=int(keep.sum()))
    empty = torch.empty(0, 3, device=dev)
    assert cloud.project_step(empty, torch.empty(0, device=dev), empty).shape == (0, 3)


def test_filter_kernel_matches_restatement():
    dev = _dev()
    from neuraludf_b200 import cloud
    p, u, _ = _crafted(70_001, 5)
    for thr in (0.0, 0.03, 2.0 / 255):
        out = cloud.filter_points(torch.from_numpy(p).to(dev), torch.from_numpy(u).to(dev), thr)
        assert _same_bits(out.cpu().numpy(), U.filter_points(p, u, np.float32(thr)))


@pytest.mark.parametrize("seed", [0, 1, 12345, 2 ** 32 + 7, -3])
def test_resample_kernel_matches_restatement(seed):
    dev = _dev()
    from neuraludf_b200 import cloud
    pool = np.random.default_rng(1).uniform(-0.6, 0.6, (1237, 3)).astype(np.float32)
    pd = torch.from_numpy(pool).to(dev)
    for r in range(4):
        for m, N in ((1, 64), (300_001, 1024)):
            out = cloud.resample(pd, m, seed, r, 2.0 / (N - 1))
            assert _same_bits(out.cpu().numpy(), U.resample(pool, m, seed, r, 2.0 / (N - 1))), (r, m)
    assert cloud.resample(pd, 0, seed, 0, 0.1).shape == (0, 3)


class _NormalsField(_Field):
    """near_surface_cells_sparse's normals come from surface_normals when a field has one"""

    def surface_normals(self, pts):
        return -self.value_gradient(pts)[1]


@pytest.mark.parametrize("name", sorted(U.CASES))
def test_seeds_match_restatement(name):
    _dev()
    from neuraludf_b200 import grid
    N = U.CASES[name]
    field = _Field(name)
    band, _ = grid.udf_band_sparse(field, N)
    idx = grid.near_surface_indices_sparse(band)
    ref, pts = U.seeds(U.Analytic(name).values, N)
    assert np.array_equal(idx.cpu().numpy(), ref)
    assert _same_bits(grid._index_points(idx, N).cpu().numpy(), pts)
    i2, nrm = grid.near_surface_cells_sparse(_NormalsField(name), band)
    assert torch.equal(i2, idx) and nrm.shape == (idx.numel(), 3)


@pytest.mark.parametrize("name", sorted(U.CASES))
def test_pipeline_on_analytic_fields(name):
    _dev()
    from scipy.spatial import cKDTree
    from neuraludf_b200 import cloud
    N = U.CASES[name]
    h = 2.0 / (N - 1)
    field = _Field(name)
    info = {}
    a = cloud.udf_point_cloud(field, N, 30000, info=info)
    b = cloud.udf_point_cloud(field, N, 30000)
    assert a.shape == (30000, 3) and torch.equal(a.view(torch.int32), b.view(torch.int32))
    pts = a.double().cpu().numpy()
    dist = U.udf_grad(name, pts)[0]
    assert float(dist.max()) < SURFACE_TOL
    d, _ = cKDTree(pts).query(U.surface_samples(name, 20000))
    assert float(d.max()) < h
    with pytest.warns(RuntimeWarning, match="lattice order"):
        assert cloud.udf_point_cloud(field, N, 1000).shape == (1000, 3)
    ref, rinfo = U.point_cloud(U.Analytic(name), N, 30000)
    same = _same_bits(a.cpu().numpy(), ref)
    assert same and {k: info[k] for k in rinfo} == rinfo
    report("cloud_analytic", case=name, N=N, seeds=info["seeds"], filtered=info["filtered"], rounds=info["rounds_used"],
           max_surface_dist=float(dist.max()), max_cover_dist_voxels=float(d.max()) / h, equals_restatement=same)


def test_batch_invariance():
    """seeds and cloud at max_batch 2^16 and 2^20 on a lattice whose seeds span several 2^16 batches"""
    _dev()
    from neuraludf_b200 import cloud
    field = _Field("sphere")
    i16, i20 = {}, {}
    a = cloud.udf_point_cloud(field, 256, 1 << 19, max_batch=1 << 16, info=i16)
    b = cloud.udf_point_cloud(field, 256, 1 << 19, max_batch=1 << 20, info=i20)
    assert i16["seeds"] > 3 * (1 << 16) and i16["seeds"] == i20["seeds"] and i16["steps"] == i20["steps"]
    assert torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.fixture(scope="module")
def c5():
    _dev()
    from neuraludf_b200 import synthetic as S
    from neuraludf_b200.models.fields import UDFNetwork
    net = UDFNetwork(d_in=3, d_out=257, d_hidden=256, n_layers=8, skip_in=(4,), multires=6, bias=0.5, scale=1.0,
                     geometric_init=True, weight_norm=True, udf_type="abs")
    net.load_state_dict(S.make_udf_params(S.udf_cfg(), 0))
    return net.cuda()


def test_value_gradient_matches_value_and_gradient(c5):
    from neuraludf_b200 import grid
    g = torch.Generator(device="cpu").manual_seed(0)
    for pts in ((torch.rand(100_003, 3, generator=g) * 2 - 1).cuda(), grid.lattice_points(0, 64 ** 3, 64, "cuda")):
        u, gr = c5.value_gradient(pts)
        out, gr2 = c5.value_and_gradient(pts)
        assert u.shape == (pts.shape[0],) and gr.shape == (pts.shape[0], 3) and not u.requires_grad
        assert np.array_equal(_bits(u), _bits(out[:, 0])) and np.array_equal(_bits(gr), _bits(gr2))
    u, gr = c5.value_gradient(torch.empty(0, 3, device="cuda"))
    assert u.shape == (0,) and gr.shape == (0, 3)


def test_network_step_against_fp64_oracle(c5):
    """one projection step from the N = 128 seeds (every 16th): the kernel's step from the chain's (u, g) against the
    step from the fp64 oracle's, within 2x the fp32 oracle's own noise (gpu_util.parity)"""
    from neuraludf_b200 import cloud, grid
    from neuraludf_b200 import synthetic as S
    from oracle import oracle_torch as O
    band, _ = grid.udf_band_sparse(c5, 128)
    seeds = grid._index_points(grid.near_surface_indices_sparse(band), 128)[::16].contiguous()
    u, g = c5.value_gradient(seeds)
    new = cloud.project_step(seeds, u, g)
    assert new.shape == seeds.shape and seeds.shape[0] > 500

    def step(dtype):
        cfg = S.udf_cfg()
        out, gr = O.udf_value_and_gradient_analytic(O.to_dtype(S.make_udf_params(cfg, 0), dtype), cfg, seeds.cpu().to(dtype))
        return seeds.cpu().to(dtype) - (out[:, :1] / gr.norm(dim=1, keepdim=True)) * gr

    parity("cloud_step_c5", new.cpu(), step(torch.float64), step(torch.float32))


def test_network_cloud(c5):
    from neuraludf_b200 import cloud
    N, n = 256, 1 << 19
    h = 2.0 / (N - 1)
    i16, i20 = {}, {}
    a = cloud.udf_point_cloud(c5, N, n, max_batch=1 << 16, info=i16)
    b = cloud.udf_point_cloud(c5, N, n, max_batch=1 << 20, info=i20)
    assert a.shape == (n, 3) and i16["seeds"] == i20["seeds"] > 100_000
    u = c5.udf_values(a)
    assert bool((u < np.float32(h)).all())
    invariant = bool(torch.equal(a.view(torch.int32), b.view(torch.int32)))
    report("cloud_c5", N=N, seeds=i16["seeds"], steps=i16["steps"], filtered=i16["filtered"], rounds=i16["rounds"],
           batch_invariant=invariant, max_udf_voxels=float(u.max()) / h, ms=i20["ms"])
    print("C5 N=%d: %d seeds, steps %s, %d kept, rounds %s, batch-invariant %s" % (
        N, i16["seeds"], i16["steps"], i16["filtered"], i16["rounds"], invariant))


def test_cli_round_trip(c5, tmp_path):
    from neuraludf_b200 import cloud
    from neuraludf_b200.evaluate import eval_deepfashion, read_ply, write_ply_points
    ckpt = os.path.join(str(tmp_path), "ckpt_000100.pth")
    torch.save({"udf_network_fine": c5.state_dict(), "iter_step": 100}, ckpt)
    cams = os.path.join(str(tmp_path), "cameras_sphere.npz")
    sm = np.eye(4)
    sm[:3, :3] *= 1.7
    sm[:3, 3] = [0.25, -0.5, 3.0]
    np.savez(cams, scale_mat_0=sm, world_mat_0=np.eye(4))
    N, n = 256, 1 << 19                     # more than the 340 k points that survive the filter: densified, not cut
    pts = cloud.udf_point_cloud(c5, N, n, seed=5).double().cpu().numpy()
    sm32 = sm.astype(np.float32)
    env = dict(os.environ, PYTHONPATH=ROOT)
    for extra, want in (([], pts), (["--cameras", cams], pts * sm32[0, 0] + sm32[:3, 3][None])):
        out = os.path.join(str(tmp_path), "cloud%d.ply" % len(extra))
        r = subprocess.run([sys.executable, "-m", "neuraludf_b200.cloud", "--ckpt", ckpt, "--resolution", str(N), "--points",
                            str(n), "--seed", "5", "--out", out] + extra, cwd=ROOT, env=env, capture_output=True, text=True,
                           timeout=1800)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        v, f = read_ply(out)
        assert f is None and np.array_equal(v, want)
    # the C5 surface is a perturbed sphere: along 1000 rays the fp64 oracle's udf is smallest at mean |r - 0.5| = 0.074
    # (0.091 weighted by area), so the mean of the two Chamfer directions to the radius-0.5 sphere is about 0.083
    rng = np.random.default_rng(0)
    gt = rng.normal(size=(200_000, 3))
    gt = 0.5 * gt / np.linalg.norm(gt, axis=1, keepdims=True)
    res = eval_deepfashion(torch.from_numpy(pts).cuda(), None, gt, max_dist=1.0)
    assert float(res["over_all"]) < 0.11
    gt_ply = os.path.join(str(tmp_path), "gt.ply")
    write_ply_points(gt_ply, gt)
    r = subprocess.run([sys.executable, "-m", "neuraludf_b200.evaluate", "deepfashion", "--data",
                        os.path.join(str(tmp_path), "cloud0.ply"), "--gt", gt_ply, "--mode", "pcd", "--log",
                        os.path.join(str(tmp_path), "eval.txt")], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    lines = r.stdout.strip().splitlines()
    assert len(lines) == 3 and lines[0].startswith("over_all:") and lines[2].startswith("precision_2mm:")
    report("cloud_cli", over_all=float(res["over_all"]), mean_d2gt=float(res["mean_d2gt"]),
           mean_gt2d=float(res["mean_gt2d"]), eval=lines)

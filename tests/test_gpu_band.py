"""Narrow-band meshing (grid.udf_band, mesh.udf_mesh_band, csrc/mesh_band.cu): the kernels against their NumPy restatement
(tests/proto/udf_band.py) exactly; the batch invariance of udf_values / gradient that exactness rests on; the band against
the dense sweep and the band mesh against udf_mesh bit for bit on the C5 network and the analytic fields; the Lipschitz
warning; a closed 1024^3 raw mesh; determinism; the checkpoint-to-PLY CLI."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.gpu_util import report
from tests.proto import mesh_cases as C
from tests.proto import udf_band as B

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


class _Analytic(torch.nn.Module):
    """an analytic field behind the udf_values / gradient interface (fp64 on the device, rounded to fp32)"""

    def __init__(self, name, dev, gain=1.0):
        super().__init__()
        self.name, self.gain = name, gain
        self.anchor = torch.nn.Parameter(torch.zeros(1, device=dev))      # the device, for udf_mesh / near_surface_cells

    def udf_values(self, x):
        return (self.gain * B.exact_udf(self.name, x.reshape(-1, 3).double(), torch)).float()

    def gradient(self, x):
        with torch.enable_grad():
            p = x.detach().reshape(-1, 3).double().requires_grad_(True)
            g, = torch.autograd.grad((self.gain * B.exact_udf(self.name, p, torch)).sum(), p)
        return g.float().unsqueeze(1)


class _Lookup:
    """a field given by its lattice values: udf_values reads them back at the lattice points"""

    def __init__(self, u, N, dev):
        self.u, self.N = torch.from_numpy(u).to(dev), N
        self.voxel = 2.0 / (N - 1)

    def udf_values(self, x):
        i = torch.round((x.double() + 1.0) / self.voxel).to(torch.int64)
        return self.u[(i[:, 0] * self.N + i[:, 1]) * self.N + i[:, 2]]


@pytest.fixture(scope="module")
def c5(golden):
    _dev()
    from tests.gpu_util import build_modules
    return build_modules(golden, "cuda")[0]


@pytest.mark.parametrize("N,strides,name", [(50, [6, 3, 1], "cylinder"), (65, [8, 4, 2, 1], "sphere"),
                                            (33, [16, 4, 1], "patch"), (129, [8, 2, 1], "plane")])
def test_kernels_match_restatement(N, strides, name):
    dev = _dev()
    from neuraludf_b200 import grid
    u = B.exact_udf(name, C.lattice(N)).astype(np.float32)
    u[0] = np.nan                                               # a NaN corner keeps its block
    df_np, levels, flags_np = B.band(lambda i: u[i], N, strides)
    lattice = grid.lattice_points(0, N ** 3, N, dev)
    ud = torch.from_numpy(u).to(dev)
    df = torch.full((N ** 3,), float("inf"), device=dev)
    idx, pts = grid.band_sublattice(N, strides[0], dev)
    assert np.array_equal(idx.cpu().numpy(), levels[0])
    assert torch.equal(pts, lattice[idx])                       # bit for bit
    df[idx] = ud[idx]
    parent = None
    for k, s in enumerate(strides[:-1]):
        flags, slope = grid.band_block_test(df, N, s, parent, strides[k - 1] if k else 0)
        assert np.array_equal(flags.cpu().numpy(), flags_np[k])
        _, slope_np = B.block_test(df.cpu().numpy(), N, s, None if parent is None else parent.cpu().numpy(),
                                   strides[k - 1] if k else 0)
        assert slope == slope_np
        idx, pts, n_kept = grid.band_points(flags, N, s, strides[k + 1])
        assert n_kept == int(flags_np[k].sum())
        assert np.array_equal(idx.cpu().numpy(), levels[k + 1])
        assert torch.equal(pts, lattice[idx])
        df[idx] = ud[idx]
        parent = flags
    assert np.array_equal(df.cpu().numpy(), df_np, equal_nan=True)
    band, info = grid.udf_band(_Lookup(u, N, dev), N, strides=strides)
    assert np.array_equal(band.cpu().numpy(), df_np, equal_nan=True)
    assert info["points"] == [len(x) for x in levels]


def test_batch_invariance(c5):
    dev = _dev()
    g = torch.Generator(device="cpu").manual_seed(5)
    P = 1 << 21
    pts = (torch.rand(P, 3, generator=g) * 2.0 - 1.0).to(dev)
    perm = torch.randperm(P, generator=g).to(dev)
    with torch.no_grad():
        for name, fn in (("udf_values", lambda x: c5.udf_values(x).reshape(-1)),
                         ("gradient", lambda x: c5.gradient(x.clone()).reshape(-1, 3))):   # gradient() flags its input
            full = fn(pts)
            assert torch.equal(fn(pts[perm]), full[perm]), name
            single = torch.randint(0, P, (64,), generator=g).tolist()
            for j in single:
                assert torch.equal(fn(pts[j:j + 1]), full[j:j + 1]), (name, j)
            for b in (127, 4096):
                for head in list(range(0, 16 * b, b)) + [P - b - 5, P // 2 + 3]:
                    assert torch.equal(fn(pts[head:head + b]), full[head:head + b]), (name, b, head)
            del full
            torch.cuda.empty_cache()


@pytest.mark.parametrize("N", [256, 512])
def test_band_equals_dense_grid(c5, N):
    from neuraludf_b200 import grid
    dense = grid.udf_grid(c5, N)
    band, info = grid.udf_band(c5, N)
    tau = 2.0 * (2.0 / (N - 1))
    near = dense < tau                                          # near_surface_cells' comparison
    assert torch.equal(band[near], dense[near])
    ev = torch.isfinite(band)
    assert torch.equal(band[ev], dense[ev])                     # every evaluated point has the dense bits
    assert bool((dense[~ev] >= tau).all())
    report("band_vs_dense", N=N, evaluated=int(ev.sum()), fraction=float(ev.float().mean()),
           max_edge_slope=info["max_edge_slope"], points=info["points"], kept_blocks=info["kept_blocks"])
    print("N=%d: %s, evaluated %.4f of N^3" % (N, info, float(ev.float().mean())))


@pytest.mark.parametrize("N", [128, 256, 512])
def test_mesh_band_equals_dense_mesh(c5, N):
    from neuraludf_b200 import mesh
    v0, f0 = mesh.udf_mesh(c5, N)
    v1, f1 = mesh.udf_mesh_band(c5, N)
    assert f0.shape[0] > 1000
    assert torch.equal(v0, v1) and torch.equal(f0, f1)


@pytest.mark.parametrize("strides", [None, [6, 3, 1]], ids=["default", "6-3-1"])
@pytest.mark.parametrize("name", sorted(C.CASES))
def test_mesh_band_equals_dense_mesh_on_fields(name, strides):
    dev = _dev()
    from neuraludf_b200 import mesh
    field = _Analytic(name, dev)
    for N in (64, 65):
        v0, f0 = mesh.udf_mesh(field, N)
        v1, f1 = mesh.udf_mesh_band(field, N, strides=strides)
        assert f0.shape[0] > 100
        assert torch.equal(v0, v1) and torch.equal(f0, f1), (name, N)


def test_steep_field_warns():
    dev = _dev()
    from neuraludf_b200 import grid
    with pytest.warns(RuntimeWarning, match="lipschitz"):
        _, info = grid.udf_band(_Analytic("plane", dev, gain=3.0), 33, lipschitz=2.0)
    assert 2.9 < info["max_edge_slope"] <= 3.0 + 1e-5


def test_1024_raw_mesh_is_an_oriented_two_manifold(c5):
    """The raw MC output at 1024^3: no edge in more than two triangles, none used twice in the same direction.  It is not
    closed: C5's surface has one open patch near (0.21, -0.30, 0.23), far from the lattice's border, whose boundary the
    dense udf_mesh shows as well at 128 ... 512 (24, 87, 333 boundary edges); 1024 has 1359."""
    from neuraludf_b200 import grid, mesh
    N = 1024
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    df, info = grid.udf_band(c5, N)
    idx, nrm = grid.near_surface_cells(c5, N, df)
    v, f, _ = mesh.marching_cubes_index(df, (N, N, N), nrm, idx)
    peak = torch.cuda.max_memory_allocated()
    assert f.shape[0] > 1_000_000
    V = v.shape[0]
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    key = e[:, 0] * V + e[:, 1]
    ks, _ = torch.sort(key)
    assert bool((ks[1:] != ks[:-1]).all()), "a directed edge is used twice"
    _, uses = torch.unique(torch.minimum(e[:, 0], e[:, 1]) * V + torch.maximum(e[:, 0], e[:, 1]), return_counts=True)
    assert int(uses.max()) == 2, "an edge is in more than two triangles"
    boundary = torch.nonzero(~torch.isin(e[:, 1] * V + e[:, 0], ks)).reshape(-1)
    w = v[e[boundary].reshape(-1)] * (2.0 / (N - 1)) - 1.0
    centre = torch.tensor([0.21, -0.30, 0.23], device=w.device)
    assert boundary.numel() < 1e-3 * e.shape[0]
    assert float((w - centre).norm(dim=1).max()) < 0.15, "a boundary edge outside the known open patch"
    report("band_1024", faces=int(f.shape[0]), vertices=V, boundary_edges=int(boundary.numel()), peak_gb=peak / 1e9,
           points=info["points"], max_edge_slope=info["max_edge_slope"])
    print("N=1024: %d faces, %d vertices, %d boundary edges, peak max_memory_allocated %.2f GB, points %s" % (
        f.shape[0], V, boundary.numel(), peak / 1e9, info["points"]))


def test_deterministic(c5):
    from neuraludf_b200 import grid, mesh
    a, _ = grid.udf_band(c5, 256)
    b, _ = grid.udf_band(c5, 256)
    assert torch.equal(a, b)
    v0, f0 = mesh.udf_mesh_band(c5, 256)
    v1, f1 = mesh.udf_mesh_band(c5, 256)
    assert torch.equal(v0, v1) and torch.equal(f0, f1)


def test_cli_meshes_a_runner_checkpoint(c5, tmp_path):
    from neuraludf_b200 import mesh
    from neuraludf_b200.evaluate import read_ply
    ckpt, cams, out = (os.path.join(str(tmp_path), n) for n in ("ckpt_000100.pth", "cameras_sphere.npz", "mesh.ply"))
    torch.save({"udf_network_fine": c5.state_dict(), "iter_step": 100}, ckpt)      # exp_runner_blending.py:484-494's keys
    sm = np.eye(4)
    sm[0, 0] = sm[1, 1] = sm[2, 2] = 212.5
    sm[:3, 3] = [-10.25, 3.5, 620.0]
    np.savez(cams, scale_mat_0=sm, world_mat_0=np.eye(4))
    r = subprocess.run([sys.executable, "-m", "neuraludf_b200.mesh", "--ckpt", ckpt, "--resolution", "128", "--cameras", cams,
                        "--out", out], cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    v, f = read_ply(out)
    v1, f1 = mesh.udf_mesh_band(c5, 128)
    s32 = sm.astype(np.float32)
    ref = v1.double().cpu().numpy() * s32[0, 0] + s32[:3, 3][None]
    assert f.shape[0] > 1000
    assert np.array_equal(v, ref) and np.array_equal(f, f1.cpu().numpy())
    net = mesh.udf_network_from_state(c5.state_dict())
    assert (net.num_layers, net.skip_in, net.multires, net.d_out) == (c5.num_layers, c5.skip_in, c5.multires, c5.d_out)

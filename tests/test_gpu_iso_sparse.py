"""Block-sparse narrow-band threshold meshing (grid.iso_band_sparse, mesh.iso_marching_cubes_sparse / iso_mesh_sparse,
the BrickDf instantiations of the table block test and of the threshold MC, and the active-cell enumeration
nudf_iso_lat_cells_*): the store against iso_band's df bit for bit, the mesh against iso_mesh_band bit for bit on the C5
network on three boxes, on a steep field and with a small batch; the enumeration on dense lattices against
nudf_iso_active; the runner's NUDF_BAND_MESH=sparse switch; the 1024^3 memory bound; the 2048^3 CLI."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.gpu_util import report
from tests.test_gpu_extract import _runner_call, _runner_func_grad
from tests.test_gpu_iso_band import BOX, _box
from tests.test_gpu_sparse import _peak, _workspace

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LEVELS = (0.005, 0.02)


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def c5(golden):
    _dev()
    from tests.gpu_util import build_modules
    return build_modules(golden, "cuda")[0]


@pytest.fixture(scope="module")
def boxes(tmp_path_factory):
    from neuraludf_b200 import mesh
    s = np.eye(4)
    s[:3, :3] *= 1.3
    s[:3, 3] = [0.2, -0.1, 0.4]
    cams = str(tmp_path_factory.mktemp("cams") / "cameras.npz")
    np.savez(cams, scale_mat_0=s, world_mat_0=np.eye(4))
    lo, hi, _ = mesh.threshold_box(cams)
    return {"cube": _box([-1.01] * 3, [1.01] * 3), "box": _box(*BOX), "cameras": (torch.from_numpy(lo), torch.from_numpy(hi))}


def _bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.contiguous().view(torch.uint8),
                                                                      b.contiguous().view(torch.uint8))


def _same_mesh(a, b):
    (v0, f0, i0), (v1, f1, i1) = a, b
    for k in ("active", "face_keys", "vertex_keys"):
        assert torch.equal(i0[k], i1[k]), k
    assert torch.equal(f0, f1) and _bits(v0, v1)


@pytest.mark.parametrize("N", [64, 97, 256])
@pytest.mark.parametrize("box", ["cube", "box", "cameras"])
def test_store_reads_iso_band(c5, boxes, box, N):
    from neuraludf_b200 import grid
    query = lambda p: c5.udf_values(p)                          # noqa: E731
    for level in LEVELS:
        df, info = grid.iso_band(query, *boxes[box], N, level)
        band, sinfo = grid.iso_band_sparse(query, *boxes[box], N, level)
        for k in ("points", "kept_blocks", "edge_slope", "tau", "pad", "spacing"):
            assert sinfo[k] == info[k], k
        assert _bits(band.values(torch.arange(N ** 3, device=df.device)), df)
        report("iso_sparse_store", box=box, N=N, level=level, bricks=sinfo["bricks"], bytes=sinfo["bytes"])


@pytest.mark.parametrize("N", [128, 256, 512])
@pytest.mark.parametrize("box", ["cube", "box", "cameras"])
def test_sparse_mesh_equals_band_mesh(c5, boxes, box, N):
    from neuraludf_b200 import mesh
    query = lambda p: c5.udf_values(p)                          # noqa: E731
    for level in LEVELS:
        a = mesh.iso_mesh_band(query, *boxes[box], N, level)
        b = mesh.iso_mesh_sparse(query, *boxes[box], N, level)
        _same_mesh(a, b)
        assert b[2]["band"]["points"] == a[2]["band"]["points"]
        if level == 0.02 and box == "cube":
            assert a[1].shape[0] > 1000


def test_steep_field_and_small_batch(c5, boxes):
    """exact with no Lipschitz precondition (a 40-Lipschitz field the band under-samples) and with batches of 4099"""
    from neuraludf_b200 import mesh
    steep = lambda p: 40.0 * (p[:, 2] - 0.13).abs() + 0.3 * torch.sin(7 * p[:, 0])     # noqa: E731
    for N in (65, 130):
        for level in (0.4, 1.5):
            with pytest.warns(RuntimeWarning, match="lipschitz"):
                a = mesh.iso_mesh_band(steep, *boxes["box"], N, level)
            with pytest.warns(RuntimeWarning, match="lipschitz"):
                b = mesh.iso_mesh_sparse(steep, *boxes["box"], N, level)
            _same_mesh(a, b)
    query = lambda p: c5.udf_values(p)                          # noqa: E731
    for level in LEVELS:
        _same_mesh(mesh.iso_mesh_band(query, *boxes["cube"], 128, level),
                   mesh.iso_mesh_sparse(query, *boxes["cube"], 128, level, max_batch=4099))


def test_enumeration_on_dense_lattices(c5, boxes):
    from neuraludf_b200 import mesh
    from neuraludf_b200.models import udf_renderer_blending as R
    dev = _dev()
    g = torch.Generator(device="cpu").manual_seed(3)
    for dims in ((2, 2, 2), (3, 5, 2), (17, 30, 9), (64, 64, 64)):
        n = dims[0] * dims[1] * dims[2]
        df = (torch.rand(n, generator=g) * 0.6 - 0.05).to(dev)
        df[torch.randint(0, n, (max(n // 50, 1),), generator=g).to(dev)] = float("nan")
        df[torch.randint(0, n, (max(n // 30, 1),), generator=g).to(dev)] = float(np.float32(0.02))
        df[torch.randint(0, n, (max(n // 40, 1),), generator=g).to(dev)] = float("inf")
        for level in (0.02, 0.3, -1.0, 5.0):
            want = mesh.iso_marching_cubes_index(df, dims, level)[2]["active"]
            assert torch.equal(mesh.iso_active_cells(df, level, dims), want), (dims, level)
    with torch.no_grad():
        dense = R._grid_query_device(*boxes["box"], 256, lambda p: c5.udf_values(p), dev, 0).reshape(-1)
    for level in LEVELS:
        want = mesh.iso_marching_cubes_index(dense, (256, 256, 256), level)[2]["active"]
        assert want.numel() > 1000
        assert torch.equal(mesh.iso_active_cells(dense, level, (256, 256, 256)), want)


@pytest.mark.parametrize("N", [64, 97])
def test_extract_geometry_sparse_env(c5, boxes, monkeypatch, N):
    from neuraludf_b200.models import udf_renderer_blending as R
    monkeypatch.setitem(sys.modules, "mcubes", None)
    query = lambda p: c5.udf_values(p)                          # noqa: E731
    for box in ("cube", "box", "cameras"):
        for level in LEVELS:
            out = []
            for flag in ("1", "sparse"):
                monkeypatch.setenv("NUDF_BAND_MESH", flag)
                out.append(R.extract_geometry(*boxes[box], N, level, query, torch.device("cuda")))
            (v0, f0), (v1, f1) = out
            assert v1.dtype == np.float64 and f1.dtype == np.int64
            assert np.array_equal(v0, v1) and np.array_equal(f0, f1)


def test_get_mesh_udf_fast_sparse_env(c5, monkeypatch):
    """NUDF_BAND_MESH=sparse serves get_mesh_udf_fast the band mesh, also for a func with negative values (clamped to 0
    on the store as on the band lattice)"""
    from neuraludf_b200 import extract_mesh as X
    func_grad = _runner_func_grad(c5)
    for func in (c5.udf, lambda p: c5.udf(p) - 0.004):
        outs = []
        for flag in ("1", "sparse"):
            monkeypatch.setenv("NUDF_BAND_MESH", flag)
            outs.append(_runner_call(X.get_mesh_udf_fast, func, func_grad, 128))
        (a, fa), (b, fb) = outs
        assert fa == fb
        assert np.array_equal(a[2].vertices, b[2].vertices) and np.array_equal(a[2].faces, b[2].faces)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and np.array_equal(a[4], b[4])
        assert len(a[2].faces) > 1000


def test_1024_memory_bound(c5, boxes):
    """the sparse threshold mesh at 1024^3 needs less than R^3 bytes beside the value chain's batch workspace"""
    from neuraludf_b200 import mesh
    N = 1024
    ws = _workspace(c5, 1 << 21)
    (v, f, info), peak = _peak(lambda: mesh.iso_mesh_sparse(lambda p: c5.udf_values(p), *boxes["cube"], N, 0.005))
    b = info["band"]
    report("iso_sparse_memory", N=N, peak_gb=peak / 1e9, workspace_gb=ws / 1e9, rest_gb=(peak - ws) / 1e9,
           bound_gb=N ** 3 / 1e9, faces=int(f.shape[0]), bricks=b["bricks"], bytes=b["bytes"], points=b["points"])
    print("N=%d: peak %.3f GB, workspace %.3f GB, rest %.3f GB (bound %.3f), %d faces, %s" % (
        N, peak / 1e9, ws / 1e9, (peak - ws) / 1e9, N ** 3 / 1e9, f.shape[0], b["bytes"]))
    assert f.shape[0] > 1_000_000
    assert peak - ws < N ** 3


def test_cli_2048(c5, tmp_path):
    from neuraludf_b200.evaluate import read_ply
    ckpt, out = str(tmp_path / "ckpt.pth"), str(tmp_path / "iso.ply")
    torch.save({"udf_network_fine": {k: v.cpu() for k, v in c5.state_dict().items()}}, ckpt)
    from tests.golden_util import load_golden
    scale = float(load_golden().udf_c["scale"])
    code = ("import sys, torch\nfrom neuraludf_b200 import mesh\nmesh.main(sys.argv[1:])\n"
            "print('PEAK_BYTES', torch.cuda.max_memory_allocated())\n")
    r = subprocess.run([sys.executable, "-c", code, "--ckpt", ckpt, "--resolution", "2048", "--threshold", "0.005",
                        "--band", "--sparse", "--scale", repr(scale), "--out", out], cwd=ROOT,
                       env=dict(os.environ, PYTHONPATH=ROOT), capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    v, f = read_ply(out)
    assert len(f) > 1_000_000 and np.isfinite(v).all()
    peak = int(r.stdout.split("PEAK_BYTES")[-1].split()[0])
    report("iso_sparse_cli_2048", faces=len(f), peak_gb=peak / 1e9)
    print("2048^3 --threshold 0.005 --band --sparse: %d faces, peak %.3f GB" % (len(f), peak / 1e9))

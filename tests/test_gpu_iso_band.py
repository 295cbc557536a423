"""Narrow-band threshold meshing (grid.iso_band, mesh.iso_mesh_band, csrc/mesh_band.cu's table form): the box kernels
against their NumPy restatement (tests/proto/iso_band.py) exactly; the band against the dense lattice and the band mesh
against extract_geometry's dense device path bit for bit on the C5 network, on three boxes; the device linspace tables; a
1024^3 band mesh; the Lipschitz warning; determinism; the --threshold --band CLI; and the unmodified runner's
--mode validate_mesh under NUDF_BAND_MESH=1."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import refshim
from tests.proto import iso_band as I
from tests.proto import mesh_cases as C
from tests.proto import udf_band as B
from tests.test_gpu_iso import DRIVER

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# test_gpu_iso.py's runner driver, seeded: the runner does not seed its generators, so without this the two runs compared
# below would build differently initialised networks (geometric init draws random weights) and mesh different fields
_SEED = "import numpy as np\nimport torch\ntorch.manual_seed(0)\nnp.random.seed(0)\n"
assert DRIVER.count("import numpy as np\n") == 1
SEEDED_DRIVER = DRIVER.replace("import numpy as np\n", _SEED)
BOX = ([-1.01, -0.9, -1.01], [1.01, 1.01, 0.95])          # test_gpu_iso.py's non-cubic box


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _box(lo, hi):
    return torch.tensor(lo, dtype=torch.float32), torch.tensor(hi, dtype=torch.float32)


@pytest.fixture(scope="module")
def c5(golden):
    _dev()
    from tests.gpu_util import build_modules
    return build_modules(golden, "cuda")[0]


@pytest.fixture(scope="module")
def boxes(tmp_path_factory):
    """+-1.01, the non-cubic box, and threshold_box of a cameras file (the dataset's object box)"""
    from neuraludf_b200 import mesh
    s = np.eye(4)
    s[:3, :3] *= 1.3
    s[:3, 3] = [0.2, -0.1, 0.4]
    cams = str(tmp_path_factory.mktemp("cams") / "cameras.npz")
    np.savez(cams, scale_mat_0=s, world_mat_0=np.eye(4))
    lo, hi, _ = mesh.threshold_box(cams)
    return {"cube": _box([-1.01] * 3, [1.01] * 3), "box": _box(*BOX), "cameras": (torch.from_numpy(lo), torch.from_numpy(hi))}


@pytest.mark.parametrize("N,strides,name", [(50, [6, 3, 1], "cylinder"), (65, [8, 4, 2, 1], "sphere"),
                                            (33, [16, 4, 1], "patch"), (97, [8, 2, 1], "plane")])
def test_box_kernels_match_restatement(N, strides, name):
    dev = _dev()
    from neuraludf_b200 import grid
    axes = grid.axis_tables(*_box(*BOX), N, dev)
    ax = [x.cpu().numpy() for x in axes]
    u = B.exact_udf(name, I.lattice(ax).astype(np.float64)).astype(np.float32)
    u[0] = np.nan                                               # a NaN corner keeps its block
    u[N ** 3 // 2 + 3] = np.nan
    level = float(np.float32(0.02))
    df_np, levels, flags_np, tau_np = I.band(lambda i: u[i], ax, strides, level)
    h, e = grid.table_spacing(axes)
    assert (h, e) == I.table_spacing(ax)
    tau, pad = grid.iso_cull(level, 2.0, h, e)
    assert tau == tau_np
    ud = torch.from_numpy(u).to(dev)
    df = torch.full((N ** 3,), float("inf"), device=dev)
    idx, pts = grid.band_sublattice_box(axes, strides[0])
    assert np.array_equal(idx.cpu().numpy(), levels[0])
    assert np.array_equal(pts.cpu().numpy(), I.points(ax, levels[0]))      # bit for bit
    df[idx] = ud[idx]
    parent = None
    for k, s in enumerate(strides[:-1]):
        ps = strides[k - 1] if k else 0
        flags, slope = grid.band_block_test_box(df, axes, s, parent, ps, h, pad, 2.0, tau)
        assert np.array_equal(flags.cpu().numpy(), flags_np[k])
        _, slope_np = I.block_test(df.cpu().numpy(), ax, s, None if parent is None else parent.cpu().numpy(), ps, h, pad,
                                   2.0, tau)
        assert slope == slope_np
        idx, pts, n_kept = grid.band_points(flags, N, s, strides[k + 1], axes)
        assert n_kept == int(flags_np[k].sum())
        assert np.array_equal(idx.cpu().numpy(), levels[k + 1])
        assert np.array_equal(pts.cpu().numpy(), I.points(ax, levels[k + 1]))
        df[idx] = ud[idx]
        parent = flags
    assert np.array_equal(df.cpu().numpy(), df_np, equal_nan=True)
    band, info = grid.iso_band(lambda p: ud[_lookup(p, axes)], *_box(*BOX), N, level, strides=strides)
    assert np.array_equal(band.cpu().numpy(), df_np, equal_nan=True)
    assert info["points"] == [len(x) for x in levels] and info["tau"] == tau and info["pad"] == 0.0


def _lookup(p, axes):
    """flat lattice indices of points that lie exactly on the table coordinates"""
    N = axes[0].numel()
    i = [torch.searchsorted(axes[a], p[:, a].contiguous()) for a in range(3)]
    return (i[0] * N + i[1]) * N + i[2]


def test_device_tables_are_monotone():
    dev = _dev()
    from neuraludf_b200 import grid, mesh
    lo, hi, _ = mesh.threshold_box(None)
    for box in (_box(lo, hi), _box(*BOX), _box([-3.5, 0.25, -0.01], [2.0, 7.5, 0.02])):
        for N in (2, 64, 96, 97, 128, 256, 512, 1024, 2048):
            axes = grid.axis_tables(*box, N, dev)
            assert all(bool((x[1:] > x[:-1]).all()) for x in axes)
            h, e = grid.table_spacing(axes)
            assert e == [0.0, 0.0, 0.0]
            assert all(x[0].item() == float(box[0][a]) and x[-1].item() == float(box[1][a]) for a, x in enumerate(axes))


@pytest.mark.parametrize("N", [64, 96, 97, 128, 256, 512])
@pytest.mark.parametrize("box", ["cube", "box", "cameras"])
def test_band_equals_dense_and_meshes_the_same(c5, boxes, box, N):
    from neuraludf_b200 import grid, mesh
    from neuraludf_b200.models import udf_renderer_blending as R
    dev = torch.device("cuda", 0)
    bmin, bmax = boxes[box]
    query = lambda p: c5.udf_values(p)                          # noqa: E731
    with torch.no_grad():
        dense = R._grid_query_device(bmin, bmax, N, query, dev, 0).reshape(-1)
    q5 = float(torch.kthvalue(dense, max(1, int(0.05 * dense.numel()))).values)
    for level in (0.005, 0.02, q5):
        lv = float(np.float32(level))
        band, info = grid.iso_band(query, bmin, bmax, N, level, device=dev)
        near = dense < info["tau"]
        assert torch.equal(band[near], dense[near])
        ev = torch.isfinite(band)
        assert torch.equal(band[ev], dense[ev])                 # every evaluated point has the dense bits
        assert bool((dense[~ev] >= info["tau"]).all())
        assert info["pad"] == 0.0
        v0, f0, i0 = mesh.iso_marching_cubes_index(dense, (N, N, N), lv)
        v1, f1, i1 = mesh.iso_mesh_band(query, bmin, bmax, N, level, device=dev)
        for k in ("active", "face_keys", "vertex_keys"):
            assert torch.equal(i0[k], i1[k]), k
        assert torch.equal(f0, f1) and torch.equal(v0, v1)
        if level == q5:
            assert f0.shape[0] > 100
        print("%s N=%d level=%.5f: evaluated %.4f, tau %.5f, %d faces" % (box, N, lv, float(ev.float().mean()), info["tau"],
                                                                           f0.shape[0]))


@pytest.mark.parametrize("N", [64, 97])
def test_extract_geometry_band_env(c5, boxes, monkeypatch, N):
    from neuraludf_b200.models import udf_renderer_blending as R
    monkeypatch.setitem(sys.modules, "mcubes", None)
    query = lambda p: c5.udf_values(p)                          # noqa: E731
    for box in ("cube", "box", "cameras"):
        bmin, bmax = boxes[box]
        for level in (0.005, 0.02):
            monkeypatch.delenv("NUDF_BAND_MESH", raising=False)
            v0, f0 = R.extract_geometry(bmin, bmax, N, level, query, torch.device("cuda"))
            monkeypatch.setenv("NUDF_BAND_MESH", "1")
            v1, f1 = R.extract_geometry(bmin, bmax, N, level, query, torch.device("cuda"))
            assert v1.dtype == np.float64 and f1.dtype == np.int64
            assert np.array_equal(v0, v1) and np.array_equal(f0, f1)
            if box == "cube" and level == 0.02:
                assert len(f0) > 100


def test_1024_band_mesh_is_edge_manifold(c5):
    from neuraludf_b200 import mesh
    N = 1024
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    v, f, info = mesh.iso_mesh_band(lambda p: c5.udf_values(p), *_box([-1.01] * 3, [1.01] * 3), N, 0.005)
    peak = torch.cuda.max_memory_allocated()
    assert f.shape[0] > 1_000_000
    s = C.mesh_stats(v.cpu().numpy(), f.cpu().numpy())
    assert s["nonmanifold"] == 0 and s["same_direction"] == 0
    print("N=1024: %d faces, %s, evaluated %.4f, peak %.2f GB" % (f.shape[0], s, sum(info["band"]["points"]) / N ** 3,
                                                                   peak / 1e9))


def test_steep_field_warns():
    dev = _dev()
    from neuraludf_b200 import grid
    with pytest.warns(RuntimeWarning, match="lipschitz"):
        _, info = grid.iso_band(lambda p: 3.0 * p[:, 2].abs(), *_box(*BOX), 33, 0.1, lipschitz=2.0, device=dev)
    assert 2.9 < info["max_edge_slope"] <= 3.0 + 1e-5


def test_deterministic(c5, boxes):
    from neuraludf_b200 import grid, mesh
    bmin, bmax = boxes["box"]
    query = lambda p: c5.udf_values(p)                          # noqa: E731
    a, _ = grid.iso_band(query, bmin, bmax, 256, 0.005)
    b, _ = grid.iso_band(query, bmin, bmax, 256, 0.005)
    assert torch.equal(a, b)
    v0, f0, _ = mesh.iso_mesh_band(query, bmin, bmax, 256, 0.005)
    v1, f1, _ = mesh.iso_mesh_band(query, bmin, bmax, 256, 0.005)
    assert torch.equal(v0, v1) and torch.equal(f0, f1)


def test_threshold_band_cli(c5, golden, tmp_path, monkeypatch):
    from neuraludf_b200 import mesh
    from neuraludf_b200.evaluate import read_ply
    monkeypatch.setitem(sys.modules, "mcubes", None)
    ck = str(tmp_path / "ckpt.pth")
    torch.save({"udf_network_fine": {k: v.cpu() for k, v in c5.state_dict().items()}}, ck)
    s = np.eye(4)
    s[:3, :3] *= 1.3
    s[:3, 3] = [0.2, -0.1, 0.4]
    cams = str(tmp_path / "cameras.npz")
    np.savez(cams, scale_mat_0=s, world_mat_0=np.eye(4))
    scale = float(golden.udf_c["scale"])
    for extra in ([], ["--cameras", cams]):
        base = ["--ckpt", ck, "--threshold", "0.02", "--resolution", "96", "--scale", repr(scale)] + extra
        a, b = str(tmp_path / "dense.ply"), str(tmp_path / "band.ply")
        mesh.main(base + ["--out", a])
        mesh.main(base + ["--band", "--lipschitz", "2", "--out", b])
        with open(a, "rb") as fa, open(b, "rb") as fb:
            assert fa.read() == fb.read()
        v, f = read_ply(b)
        assert len(f) > 500


@pytest.mark.skipif(not refshim.available(), reason="no staged reference copy (oracle/make_ref.py)")
def test_unmodified_runner_validate_mesh_band(tmp_path):
    _dev()
    from tests import runner_env
    ref = refshim.REFERENCE_ROOT
    tmp = str(tmp_path)
    runner_env.write_synthetic_dtu(os.path.join(tmp, "data", "synth"), n_images=12, width=96, height=72)
    exp = os.path.join(tmp, "exp", "CASE_NAME") + "/"
    conf = runner_env.write_conf(ref, os.path.join(tmp, "synth.conf"), os.path.join(tmp, "data", "CASE_NAME") + "/", exp,
                                 end_iter=2)
    argv = [os.path.join(ref, "exp_runner_blending.py"), "--mode", "validate_mesh", "--conf", conf, "--case", "synth",
            "--gpu", "0", "--threshold", "0.05", "--resolution", "64"]
    meshes = []
    for band in (False, True):
        out = os.path.join(tmp, "validate_mesh_%d.npz" % band)
        drv = os.path.join(tmp, "drive_%d.py" % band)
        with open(drv, "w") as fh:
            fh.write(SEEDED_DRIVER.format(root=ROOT, argv=argv, out=out))
        env = dict(os.environ, PYTHONUNBUFFERED="1")
        env.pop("NUDF_BAND_MESH", None)
        if band:
            env["NUDF_BAND_MESH"] = "1"
        r = subprocess.run([sys.executable, drv], cwd=tmp, env=env, capture_output=True, text=True, timeout=900)
        tail = r.stdout[-3000:] + "\n---- stderr ----\n" + r.stderr[-3000:]
        assert r.returncode == 0, tail
        assert "EXPORT 00000000_thresh0.0500_res64.ply" in r.stdout, tail
        m = np.load(out)
        meshes.append((m["vertices"], m["faces"]))
    (v0, f0), (v1, f1) = meshes
    assert len(f0) > 100
    assert np.array_equal(v0, v1) and np.array_equal(f0, f1)

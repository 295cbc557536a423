"""CUDA threshold marching cubes (nudf_iso_*, neuraludf_b200/mesh.py's iso_marching_cubes_index) against its NumPy
restatement (tests/proto/iso_mc.py) bit for bit; the runner's extract_geometry with and without PyMCubes; the --threshold
CLI; and the unmodified runner's --mode validate_mesh meshing on the device."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

from oracle import refshim
from tests.proto import iso_mc as P
from tests.proto import mesh_cases as C

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _compare(df, dims, level):
    from neuraludf_b200 import mesh
    pv, pf, pinfo = P.marching_cubes(df, dims, level)
    v, f, info = mesh.iso_marching_cubes_index(torch.from_numpy(np.ascontiguousarray(df, np.float32)).cuda(), dims, level)
    assert v.dtype == torch.float64 and f.dtype == torch.int64
    assert np.array_equal(info["active"].cpu().numpy(), pinfo["active"])
    assert np.array_equal(info["face_keys"].cpu().numpy(), pinfo["face_keys"])
    assert np.array_equal(info["vertex_keys"].cpu().numpy(), pinfo["vertex_keys"])
    assert np.array_equal(f.cpu().numpy(), pf)
    assert np.array_equal(v.cpu().numpy(), pv)                                 # fp64 bits
    return pv, pf, pinfo


@pytest.mark.parametrize("name", P.CASES)
def test_cuda_matches_restatement(name):
    _need_gpu()
    df, dims, level, _ = P.case(name)
    _compare(df, dims, level)


def test_cuda_matches_restatement_on_the_network_lattice(golden):
    _need_gpu()
    from neuraludf_b200 import grid
    from tests.gpu_util import build_modules
    udf = build_modules(golden, "cuda")[0]
    N = 128
    df = grid.udf_grid(udf, N).cpu().numpy()
    level = float(np.quantile(df, 0.05))
    _, pf, pinfo = _compare(df, (N, N, N), level)
    assert len(pf) > 10000
    print("network 128^3 at %.5f: %d active cells, %d faces" % (level, len(pinfo["active"]), len(pf)))


def test_nan_cells_and_empty_output():
    _need_gpu()
    from neuraludf_b200 import mesh
    df, dims, level, _ = P.case("shell")
    df = df.copy()
    rng = np.random.default_rng(3)
    df[rng.choice(df.size, 200, replace=False)] = np.nan
    _compare(df, dims, level)
    for lv in (10.0, -10.0):                                                     # nothing crosses
        v, f, info = mesh.iso_marching_cubes_index(torch.from_numpy(df).cuda(), dims, lv)
        assert v.shape == (0, 3) and f.shape == (0, 3) and info["active"].numel() == 0
        v, f = mesh.iso_marching_cubes(df.reshape(dims), lv)
        assert v.shape == (0, 3) and f.shape == (0, 3) and v.dtype == np.float64 and f.dtype == np.int64
    v, f = mesh.iso_marching_cubes(np.full((4, 4, 4), np.nan, np.float32), 0.0)
    assert v.shape == (0, 3) and f.shape == (0, 3)


def test_numpy_interface_and_argument_errors():
    _need_gpu()
    from neuraludf_b200 import mesh
    df, dims, level, _ = P.case("torus")
    pv, pf, _ = P.marching_cubes(df, dims, level)
    v, f = mesh.iso_marching_cubes(df.reshape(dims).astype(np.float64), level)   # fp64 input is meshed as fp32
    assert v.dtype == np.float64 and f.dtype == np.int64
    assert np.array_equal(v, pv) and np.array_equal(f, pf)
    vol = df.reshape(dims)
    for bad in (vol[0], vol[None], vol[:1], vol[:, :1]):
        with pytest.raises(ValueError):
            mesh.iso_marching_cubes(bad, level)
    for lv in (np.nan, np.inf, -np.inf, 1e39):
        with pytest.raises(ValueError):
            mesh.iso_marching_cubes(vol, lv)
    t = torch.from_numpy(df).cuda()
    with pytest.raises(ValueError):
        mesh.iso_marching_cubes_index(t.cpu(), dims, level)
    with pytest.raises(ValueError):
        mesh.iso_marching_cubes_index(t.double(), dims, level)
    with pytest.raises(ValueError):
        mesh.iso_marching_cubes_index(t, (dims[0] + 1, dims[1], dims[2]), level)


def _golden_udf(golden):
    from tests.gpu_util import build_modules
    return build_modules(golden, "cuda")[0]


def test_extract_geometry_device_path(golden, monkeypatch):
    _need_gpu()
    from neuraludf_b200.models import udf_renderer_blending as R
    udf = _golden_udf(golden)
    monkeypatch.setitem(sys.modules, "mcubes", None)                            # `import mcubes` raises ImportError
    bmin = torch.tensor([-1.01, -0.9, -1.01], dtype=torch.float32)
    bmax = torch.tensor([1.01, 1.01, 0.95], dtype=torch.float32)
    res, thr = 96, 0.02
    v, f = R.extract_geometry(bmin, bmax, res, thr, lambda p: udf.udf_values(p), torch.device("cuda"))
    assert isinstance(v, np.ndarray) and isinstance(f, np.ndarray) and v.dtype == np.float64 and f.dtype == np.int64
    u = R.extract_fields(bmin, bmax, res, lambda p: udf.udf_values(p), torch.device("cuda"))
    pv, pf, _ = P.marching_cubes(u, u.shape, thr)
    assert len(pf) > 1000
    assert np.array_equal(f, pf)
    assert np.array_equal(v, P.reference_mapping(pv, res, bmin.numpy(), bmax.numpy()))


def test_extract_geometry_calls_pymcubes_when_importable(golden, monkeypatch):
    _need_gpu()
    from neuraludf_b200.models import udf_renderer_blending as R
    udf = _golden_udf(golden)
    calls = []

    def marching_cubes(u, threshold):
        calls.append((u, threshold))
        return np.array([[0.0, 1.0, 2.0], [3.0, 4.0, 5.0], [6.0, 7.0, 8.0]]), np.array([[0, 1, 2]])
    monkeypatch.setitem(sys.modules, "mcubes", types.SimpleNamespace(marching_cubes=marching_cubes))
    bmin = torch.tensor([-1.01] * 3, dtype=torch.float32)
    bmax = torch.tensor([1.01] * 3, dtype=torch.float32)
    v, f = R.extract_geometry(bmin, bmax, 32, 0.005, lambda p: udf.udf_values(p), torch.device("cuda"))
    assert len(calls) == 1 and calls[0][1] == 0.005
    u = calls[0][0]
    assert isinstance(u, np.ndarray) and u.shape == (32, 32, 32) and u.dtype == np.float32
    assert np.array_equal(u, R.extract_fields(bmin, bmax, 32, lambda p: udf.udf_values(p), torch.device("cuda")))
    assert f.tolist() == [[0, 1, 2]]
    assert np.array_equal(v, P.reference_mapping(np.arange(9.0).reshape(3, 3), 32, bmin.numpy(), bmax.numpy()))


def test_threshold_cli(golden, tmp_path, monkeypatch):
    _need_gpu()
    from neuraludf_b200 import mesh
    from neuraludf_b200.evaluate import read_ply
    from neuraludf_b200.models import udf_renderer_blending as R
    monkeypatch.setitem(sys.modules, "mcubes", None)
    udf = _golden_udf(golden)
    ck = str(tmp_path / "ckpt.pth")
    torch.save({"udf_network_fine": {k: v.cpu() for k, v in udf.state_dict().items()}}, ck)
    s = np.eye(4)
    s[:3, :3] *= 1.3
    s[:3, 3] = [0.2, -0.1, 0.4]
    cams = str(tmp_path / "cameras.npz")
    np.savez(cams, scale_mat_0=s, world_mat_0=np.eye(4))
    out = str(tmp_path / "m.ply")
    scale = float(golden.udf_c["scale"])
    v, f = mesh.main(["--ckpt", ck, "--threshold", "0.02", "--resolution", "64", "--cameras", cams, "--out", out,
                      "--scale", repr(scale)])
    rv, rf = read_ply(out)
    assert np.array_equal(rv, v) and np.array_equal(rf, f) and len(f) > 500
    # validate_mesh(world_space=True): the dataset's box, extract_geometry, then scale_mat_0's transform
    lo, hi, sm = mesh.threshold_box(cams)
    ev, ef = R.extract_geometry(torch.from_numpy(lo), torch.from_numpy(hi), 64, 0.02, lambda p: udf.udf_values(p),
                                torch.device("cuda"))
    assert np.array_equal(f, ef)
    assert np.array_equal(v, ev * sm[0, 0] + sm[:3, 3][None])
    v0, f0 = mesh.main(["--ckpt", ck, "--threshold", "0.02", "--resolution", "64", "--out", out, "--scale", repr(scale)])
    assert (np.abs(v0) <= np.float32(1.01)).all()                                # +-1.01 without cameras


DRIVER = """
import sys
sys.path.insert(0, {root!r})
from tests import runner_env
runner_env.install_stubs()
sys.modules.pop("mcubes", None)                   # no PyMCubes: extract_geometry meshes on the device
import numpy as np
import trimesh


class _Recorder:
    def __init__(self, vertices, faces, *a, **k):
        np.savez({out!r}, vertices=np.asarray(vertices), faces=np.asarray(faces))

    def export(self, path, *a, **k):
        print("EXPORT " + path.rsplit("/", 1)[-1], flush=True)


trimesh.Trimesh = _Recorder
from neuraludf_b200 import launch
sys.exit(launch.main({argv!r}))
"""


@pytest.mark.skipif(not refshim.available(), reason="no staged reference copy (oracle/make_ref.py)")
def test_unmodified_runner_validate_mesh(tmp_path):
    _need_gpu()
    from tests import runner_env
    ref = refshim.REFERENCE_ROOT
    tmp = str(tmp_path)
    runner_env.write_synthetic_dtu(os.path.join(tmp, "data", "synth"), n_images=12, width=96, height=72)
    exp = os.path.join(tmp, "exp", "CASE_NAME") + "/"
    conf = runner_env.write_conf(ref, os.path.join(tmp, "synth.conf"), os.path.join(tmp, "data", "CASE_NAME") + "/", exp,
                                 end_iter=2)
    argv = [os.path.join(ref, "exp_runner_blending.py"), "--mode", "validate_mesh", "--conf", conf, "--case", "synth",
            "--gpu", "0", "--threshold", "0.05", "--resolution", "64"]
    drv = os.path.join(tmp, "drive.py")
    with open(drv, "w") as fh:
        fh.write(DRIVER.format(root=ROOT, argv=argv, out=os.path.join(tmp, "validate_mesh.npz")))
    r = subprocess.run([sys.executable, drv], cwd=tmp, env=dict(os.environ, PYTHONUNBUFFERED="1"), capture_output=True,
                       text=True, timeout=900)
    tail = r.stdout[-3000:] + "\n---- stderr ----\n" + r.stderr[-3000:]
    assert r.returncode == 0, tail
    assert "EXPORT 00000000_thresh0.0500_res64.ply" in r.stdout, tail
    m = np.load(os.path.join(tmp, "validate_mesh.npz"))
    v, f = m["vertices"], m["faces"]
    assert len(f) > 100, tail
    s = C.mesh_stats(v, f)
    assert s["boundary"] == 0 and s["nonmanifold"] == 0 and s["same_direction"] == 0
    assert (np.abs(v) <= 1.01 + 1e-6).all()                                      # world_space=False: the object box

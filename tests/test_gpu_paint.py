"""Camera visibility, orientation and colour on the device (paint.py, csrc/udf_paint.cu): every kernel bit for bit against
its NumPy restatement (tests/proto/udf_paint.py), the whole visibility pipeline on the analytic fields bit for bit and at
two batch sizes, the edge cases and input checks, the colour network's colours on the C5 networks against the module and
the fp64 oracle, mesh painting, and the cloud and mesh CLIs' PLY output on a synthetic scan."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.gpu_util import parity, report
from tests.proto import udf_paint as P

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
H, W = 64, 80
N = 256
VOXEL = 2.0 / (N - 1)


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.int32), b.view(np.int32))


def _d(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


class _Field:
    """an analytic field on the device: P.udf_grad in fp64 with torch, rounded to fp32 once"""

    def __init__(self, name):
        self.name = name

    def value_gradient(self, x):
        u, g = P.udf_grad(self.name, x.reshape(-1, 3).double(), torch)
        return u.float(), g.float()

    def udf_values(self, x):
        return self.value_gradient(x)[0]

    def surface_normals(self, x):
        return -torch.nn.functional.normalize(self.value_gradient(x)[1], dim=1)


def _cams(centres):
    intr, poses = P.cameras(np.asarray(centres, np.float64), H, W)
    mats, c = P.camera_matrices(intr, poses)
    return intr, poses, mats, c


def test_camera_matrices_match_restatement():
    _dev()
    from neuraludf_b200 import paint
    intr, poses, mats, c = _cams(P.cap_centres(49))
    m2, c2 = paint.camera_matrices(_d(intr), _d(poses))
    assert _same_bits(m2.cpu().numpy(), mats) and _same_bits(c2.cpu().numpy(), c)


def test_kernels_match_restatement():
    _dev()
    from neuraludf_b200 import paint
    rng = np.random.default_rng(0)
    g = rng.normal(size=(5003, 3)).astype(np.float32)
    g[::7] = 0
    g[1::11, 1] = np.nan
    g[2::13, 2] = np.inf
    g[3::17] = 1e-30
    assert _same_bits(paint.unit_normals(_d(g)).cpu().numpy(), P.normals(g)[0])
    _, _, mats, c = _cams(P.cap_centres(49, seed=3))
    p, _ = P.surface_samples("sphere", 20011, seed=1)
    n = P.normals(rng.normal(size=p.shape).astype(np.float32) * 0.3 + p)[0]
    md, cd = _d(mats), _d(c)
    for K, cos_min in ((4, 0.2), (8, 0.0), (1, 0.5)):
        cand = paint.rank_candidates(_d(p), _d(n), md, cd, H, W, cos_min, K).cpu().numpy()
        assert np.array_equal(cand, P.rank(p, n, mats, c, H, W, cos_min, K)), (K, cos_min)
    cand = P.rank(p, n, mats, c, H, W, 0.2, 4)
    view = np.where(rng.uniform(size=len(p)) < 0.3, cand[:, 1], -1).astype(np.int32)
    t_start, hit = np.float32(2 * VOXEL), np.float32(VOXEL)
    for r in range(4):
        ref = P.start(p, n, cand, r, view, c, t_start)
        got = paint.start_pairs(_d(p), _d(n), _d(cand), r, _d(view), cd, float(t_start))
        assert all(_same_bits(a.cpu().numpy(), b) for a, b in zip(got, ref)), r
    pairs = P.start(p, n, cand, 0, view, c, t_start)
    v_ref, v_dev = view.copy(), _d(view)
    ref, got = pairs, tuple(_d(a) for a in pairs)
    for step in range(64):                          # the sphere's udf, the first step's perturbed
        if not len(ref[0]):
            break
        u = P.Analytic("sphere").values(ref[3])
        if step == 0:
            u[::5] = rng.uniform(0, 3 * VOXEL, len(u[::5]))
            u[::97] = np.nan
        ref = P.trace_step(p, c, *ref[:3], u, hit, v_ref)
        got = paint.trace_step(_d(p), cd, got, _d(u), float(hit), v_dev)
        assert all(_same_bits(a.cpu().numpy(), b) for a, b in zip(got, ref)), step
        assert np.array_equal(v_dev.cpu().numpy(), v_ref), step
    assert (v_ref != view).sum() > 1000 and step > 2
    assert _same_bits(paint.orient_normals(_d(p), _d(n), v_dev, cd).cpu().numpy(), P.orient(p, n, v_ref, c))
    images = rng.uniform(size=(49, H, W, 3)).astype(np.float32)
    assert _same_bits(paint.gather_colors(_d(p), v_dev, md, _d(images)).cpu().numpy(), P.gather(p, v_ref, mats, images, H, W))
    report("paint_kernels", points=len(p), pairs=len(pairs[0]), active=len(ref[0]), resolved=int((v_ref != view).sum()))


CASES = {"sphere": (lambda: P.cap_centres(16), 6000), "nested": (lambda: P.cap_centres(16), 6000),
         "disc": (lambda: [(1.5, 0.0, 2.0), (-1.5, 0.0, -2.0)], 4000), "occluded": (lambda: [(0.0, 0.0, 2.5)], 6000)}


@pytest.mark.parametrize("name", sorted(CASES))
def test_pipeline_on_analytic_fields(name):
    _dev()
    from neuraludf_b200 import paint
    centres, M = CASES[name]
    _, _, mats, c = _cams(centres())
    p, n0 = P.surface_samples(name, M, seed=2)
    field = _Field(name)
    # the normal lines from the field where it gives one (off the exact surface), the exact ones elsewhere
    n = paint.point_normals(field, _d(p)).cpu().numpy()
    zero = (n == 0).all(1)
    n[zero] = n0[zero]
    ref_view, ref_n, ref_info = P.surface_views(P.Analytic(name).values, p, n, mats, c, H, W, VOXEL)
    outs = []
    for mb in (1 << 20, 1000):
        info = {}
        view, out = paint.surface_views(field, _d(p), _d(n), _d(mats), _d(c), H, W, VOXEL, max_batch=mb, info=info)
        outs.append((view.cpu().numpy(), out.cpu().numpy()))
        assert np.array_equal(outs[-1][0], ref_view) and _same_bits(outs[-1][1], ref_n), mb
        assert {k: info[k] for k in ref_info} == ref_info
    report("paint_analytic", case=name, points=M, seen=int((ref_view >= 0).sum()), rounds=ref_info["rounds"],
           evaluations=ref_info["evaluations"], undecided=ref_info["undecided"], ms=info["ms"])


def test_edge_cases_and_input_checks():
    dev = _dev()
    from neuraludf_b200 import paint
    _, _, mats, c = _cams(P.cap_centres(4))
    md, cd = _d(mats), _d(c)
    f = _Field("sphere")
    e = torch.empty(0, 3, device=dev)
    view, out = paint.surface_views(f, e, e, md, cd, H, W, VOXEL)
    assert view.shape == (0,) and out.shape == (0, 3)
    p, n = P.surface_samples("sphere", 100)
    pd, nd = _d(p), _d(n)
    info = {}
    view, out = paint.surface_views(f, pd, nd, torch.empty(0, 12, device=dev), torch.empty(0, 3, device=dev), H, W, VOXEL,
                                    info=info)
    assert (view == -1).all() and torch.equal(out, nd) and info["no_candidate"] == 100 and info["evaluations"] == 0
    assert paint.gather_colors(pd, view, torch.empty(0, 12, device=dev), torch.empty(0, H, W, 3, device=dev)).abs().sum() == 0
    many = md.repeat(17, 1)[:65].contiguous(), cd.repeat(17, 1)[:65].contiguous()
    bad = [((pd.cpu(), nd, md, cd), {}), ((pd.double(), nd, md, cd), {}), ((pd[:, :2].contiguous(), nd, md, cd), {}),
           ((pd, nd[:50], md, cd), {}), ((pd, nd, md[:3], cd), {}), ((pd, nd) + many, {}), ((pd, nd, md, cd), {"candidates": 9}),
           ((pd, nd, md, cd), {"max_steps": 0})]
    for args, kw in bad:
        with pytest.raises(ValueError):
            paint.surface_views(f, args[0], args[1], args[2], args[3], H, W, VOXEL, **kw)
    with pytest.raises(ValueError):
        paint.point_colors(pd, view, nd, "texture")
    with pytest.raises(ValueError):
        paint.gather_colors(pd, view.long(), md, torch.zeros(4, H, W, 3, device=dev))


@pytest.fixture(scope="module")
def c5():
    _dev()
    from neuraludf_b200 import synthetic as S
    from neuraludf_b200.models import fields as F
    udf = F.UDFNetwork(d_in=3, d_out=257, d_hidden=256, n_layers=8, skip_in=(4,), multires=6, bias=0.5, scale=1.0,
                       geometric_init=True, weight_norm=True, udf_type="abs")
    udf.load_state_dict(S.make_udf_params(S.udf_cfg(), 0))
    col = F.ResidualRenderingNetwork(d_feature=256, mode="no_normal", d_in=6, d_out=3, d_hidden=128, n_layers=4,
                                     weight_norm=True, multires_view=4, squeeze_out=True, blending_cand_views=10)
    col.load_state_dict(S.make_color_params(S.color_cfg(), 1))
    return udf.cuda(), col.cuda()


def _c5_cloud(udf, n_points=100_000):
    from neuraludf_b200 import cloud
    return cloud.udf_point_cloud(udf, 128, n_points)


def test_network_colors(c5):
    from neuraludf_b200 import paint
    from neuraludf_b200 import synthetic as S
    from oracle import oracle_torch as O
    udf, col = c5
    pts = _c5_cloud(udf)
    _, _, mats, c = _cams(P.cap_centres(49, seed=5))
    md, cd = _d(mats), _d(c)
    info = {}
    n = paint.point_normals(udf, pts, info=info)
    view, n = paint.surface_views(udf, pts, n, md, cd, H, W, 2.0 / 127)
    assert int((view >= 0).sum()) > 1000 and int((view < 0).sum()) > 1000
    rgb = paint.point_colors(pts, view, n, "network", centres=cd, udf_network=udf, color_network=col)
    dirs = paint.view_directions(pts, view, n, cd)
    _, feat, _ = udf.value_feature_gradient(pts)
    want = col(pts, None, dirs, feat)[1]
    assert torch.equal(rgb, want.flip(1))
    cc = S.color_cfg()
    params = S.make_color_params(cc, 1)
    sel = torch.arange(0, pts.shape[0], 37, device=pts.device)

    def oracle(dt):
        with torch.no_grad():
            return O.color_mlp(O.to_dtype(params, dt), cc, pts[sel].cpu().to(dt), dirs[sel].cpu().to(dt),
                               feat[sel].cpu().to(dt))[1]

    parity("paint_network_color_c5", rgb[sel].flip(1).cpu(), oracle(torch.float64), oracle(torch.float32))
    d = cd[view.clamp(min=0).long()] - pts
    seen = view >= 0
    assert bool(((n * d).sum(1)[seen] > 0).all())
    report("paint_c5", points=int(pts.shape[0]), seen=int(seen.sum()), zero_normals=info["zero"])


def test_paint_mesh_sphere():
    _dev()
    from neuraludf_b200 import mesh, paint
    field = _Field("sphere")
    verts, faces, _ = mesh._mesh_post(field, 64, "dense", 5.0, True)
    centres = P.cap_centres(16, seed=7)
    _, _, mats, c = _cams(centres)
    key = np.stack([(np.arange(16) + 1) / 32.0, np.full(16, 0.5), np.full(16, 0.25)], 1).astype(np.float32)
    images = np.ascontiguousarray(np.broadcast_to(key[:, None, None, :], (16, H, W, 3)))
    info = {}
    rgb, view = paint.paint_mesh(verts, faces, field, _d(mats), _d(c), H, W, 2.0 / 63, "image", images=_d(images), info=info)
    assert rgb.shape == (verts.shape[0], 3) and view.shape == (verts.shape[0],)
    rgb, view, v = rgb.cpu().numpy(), view.cpu().numpy(), verts.cpu().numpy()
    seen = view >= 0
    assert seen.sum() > 100 and (~seen).sum() > 100 and (rgb[~seen] == 0).all()
    named = np.rint(rgb[seen, 2] * 32).astype(np.int64) - 1             # blue: the BGR image's first channel
    assert np.array_equal(named, view[seen])
    assert (((c[named] - v[seen]) * v[seen]).sum(1) > 0).all()


def _synthetic_scan(root, centres):
    import cv2
    intr, poses = P.cameras(np.asarray(centres, np.float64), H, W)
    os.makedirs(os.path.join(root, "image"))
    cams = {}
    for i in range(len(poses)):
        img = np.zeros((H, W, 3), np.uint8)
        img[:, :, 0] = 40 + 10 * i
        img[:, :, 1] = np.arange(W)[None, :] * 3
        img[:, :, 2] = np.arange(H)[:, None] * 3
        cv2.imwrite(os.path.join(root, "image", "%03d.png" % i), img)
        cams["world_mat_%d" % i] = (intr[i].astype(np.float64) @ np.linalg.inv(poses[i].astype(np.float64)))
        cams["scale_mat_%d" % i] = np.eye(4)
    np.savez(os.path.join(root, "cameras.npz"), **cams)


def _header(path):
    with open(path, "rb") as f:
        lines = []
        while True:
            lines.append(f.readline().decode("ascii").strip())
            if lines[-1] == "end_header":
                return lines, f.read()


def test_cli_round_trips(c5, tmp_path):
    from neuraludf_b200.evaluate import read_ply, read_ply_colors
    udf, col = c5
    tmp = str(tmp_path)
    ckpt = os.path.join(tmp, "ckpt.pth")
    torch.save({"udf_network_fine": udf.state_dict(), "color_network_fine": col.state_dict()}, ckpt)
    scan = os.path.join(tmp, "scan")
    _synthetic_scan(scan, P.cap_centres(12, seed=9))
    env = dict(os.environ, PYTHONPATH=ROOT)

    def run(module, out, extra):
        r = subprocess.run([sys.executable, "-m", module, "--ckpt", ckpt, "--resolution", "128", "--out", out] + extra,
                           cwd=ROOT, env=env, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        return r.stdout

    plain = os.path.join(tmp, "plain.ply")
    run("neuraludf_b200.cloud", plain, ["--points", "50000"])
    head, _ = _header(plain)
    assert head == ["ply", "format binary_little_endian 1.0", head[2], "property double x", "property double y",
                    "property double z", "end_header"]
    for mode in ("image", "network"):
        out = os.path.join(tmp, "cloud_%s.ply" % mode)
        printed = run("neuraludf_b200.cloud", out, ["--points", "50000", "--scan_dir", scan, "--normals", "--colors", mode])
        assert "unseen" in printed
        head, body = _header(out)
        assert head[3:-1] == ["property double x", "property double y", "property double z", "property float nx",
                              "property float ny", "property float nz", "property uchar red", "property uchar green",
                              "property uchar blue"]
        v, f = read_ply(out)
        assert f is None and np.array_equal(v, read_ply(plain)[0])
        rgb = read_ply_colors(out)
        rec = np.frombuffer(body, dtype=[("x", "<f8", (3,)), ("n", "<f4", (3,)), ("c", "u1", (3,))])
        norms = np.linalg.norm(rec["n"].astype(np.float64), axis=1)
        assert rgb.shape == v.shape and np.array_equal(rec["c"], rgb)
        assert ((np.abs(norms - 1) < 1e-5) | (norms == 0)).all()
        assert (rgb.astype(np.int64).sum(1) > 0).sum() > 1000
    mplain = os.path.join(tmp, "mesh_plain.ply")
    run("neuraludf_b200.mesh", mplain, [])
    head, _ = _header(mplain)
    assert head[3:6] == ["property double x", "property double y", "property double z"]
    assert head[6].startswith("element face") and len(head) == 9
    mcol = os.path.join(tmp, "mesh_col.ply")
    run("neuraludf_b200.mesh", mcol, ["--scan_dir", scan, "--colors", "network"])
    head, _ = _header(mcol)
    assert head[6:9] == ["property uchar red", "property uchar green", "property uchar blue"]
    v0, f0 = read_ply(mplain)
    v1, f1 = read_ply(mcol)
    assert np.array_equal(v0, v1) and np.array_equal(f0, f1) and read_ply_colors(mcol).shape == v1.shape

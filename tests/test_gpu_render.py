"""GPU checks of the forward-only view renderer (neuraludf_b200/render.py, nudf_render_view_forward): against render()
on the same rays, independence of the chunk size, the workspace budget, and the CLI's files.  Golden scene networks,
the DTU conf's sampling (64 + 50 samples in 5 rounds, 32 NeRF++ samples), a 32 x 24 view of a synthetic DTU-layout scan
with 8 source views."""
import os

import numpy as np
import pytest
import torch

from tests.gpu_util import build_modules, report
from tests.runner_env import write_synthetic_dtu

pytestmark = pytest.mark.gpu
DEV = "cuda"
LEVEL = 3


@pytest.fixture(scope="module")
def scan(tmp_path_factory):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from neuraludf_b200 import render as R
    d = write_synthetic_dtu(str(tmp_path_factory.mktemp("scan")), n_images=12, width=96, height=72)
    return R.load_scan(d, device=DEV)


def _renderer(golden, h_patch=3):
    from neuraludf_b200.models.udf_renderer_blending import UDFRendererBlending
    udf, col, nerf, var, beta = build_modules(golden, DEV)
    return UDFRendererBlending(nerf, udf, var, col, beta, n_samples=64, n_importance=50, n_outside=32, up_sample_steps=5,
                               perturb=0.0, h_patch_size=h_patch)


def _view(scan, idx=2):
    rays_o, rays_d, near, far = scan.rays_at(idx, LEVEL)
    cmaps, w2cs, intr = scan.source_info(idx)
    rot = np.linalg.inv(scan.pose_all[idx, :3, :3].cpu().numpy())
    return rays_o, rays_d, near, far, dict(color_maps=cmaps, w2cs=w2cs, intrinsics=intr, rot=rot)


@pytest.mark.parametrize("h_patch", [3, 5])
def test_render_view_matches_render(golden, scan, h_patch):
    """color / depth: the same bits as one render() call on the same rays; color_pixel and validate()'s normal
    expression (summed in another order by torch) within 1e-6 of their maximum"""
    from neuraludf_b200 import render as R
    ren = _renderer(golden, h_patch)
    rays_o, rays_d, near, far, kw = _view(scan)
    H, W = rays_o.shape[:2]
    out = R.render_view(ren, rays_o, rays_d, near, far, cos_anneal_ratio=0.7, **kw)
    o, d = rays_o.reshape(-1, 3), rays_d.reshape(-1, 3)
    c2w = scan.pose_all[2]
    with torch.no_grad():
        ref = ren.render(o, d, near.reshape(-1, 1), far.reshape(-1, 1), cos_anneal_ratio=0.7, perturb_overwrite=0,
                         color_maps=kw["color_maps"], w2cs=kw["w2cs"], intrinsics=kw["intrinsics"], query_c2w=c2w)
    assert torch.equal(out["color"].reshape(-1, 3), ref["color"]), "color differs from render()"
    assert torch.equal(out["depth"].reshape(-1, 1), ref["depth"]), "depth differs from render()"
    S = ref["gradients_flip"].shape[1]
    nrm = (ref["gradients_flip"] * ref["weights"][:, :S, None] * ref["inside_sphere"][..., None]).sum(dim=1)
    nrm = (torch.from_numpy(kw["rot"]).float().to(DEV) @ nrm.T).T
    for k, r in (("color_pixel", ref["color_pixel"]), ("normal", nrm), ("weight_sum", ref["weight_sum"])):
        a = out[k].reshape(r.shape)
        err = float((a - r).abs().max())
        scale = float(r.abs().max())
        report("render_view.h%d.%s" % (h_patch, k), err=err, rel=err / scale)
        assert err <= 1e-6 * scale, (k, err, scale)
    assert out["color"].shape == (H, W, 3) and out["depth"].shape == (H, W, 1)


def test_render_view_chunk_size_independent(golden, scan):
    """chunks of 1, 511, 4096 rays and the whole view give the same bits (every stage is per ray or per point)"""
    from neuraludf_b200 import render as R
    ren = _renderer(golden)
    rays_o, rays_d, near, far, kw = _view(scan, 5)
    outs = [R.render_view(ren, rays_o, rays_d, near, far, cos_anneal_ratio=0.3, max_chunk=c, **kw)
            for c in (None, 1, 511, 4096)]
    for c, o in zip((1, 511, 4096), outs[1:]):
        for k in outs[0]:
            assert torch.equal(outs[0][k], o[k]), "chunk %d changes %s" % (c, k)


def test_render_view_workspace_budget(golden, scan):
    """peak device memory of a view stays under the workspace budget plus the image buffers"""
    from neuraludf_b200 import render as R
    ren = _renderer(golden)
    rays_o, rays_d, near, far, kw = _view(scan)
    budget = 24 << 20
    R.render_view(ren, rays_o, rays_d, near, far, workspace_bytes=budget, **kw)      # folds the weights once
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = R.render_view(ren, rays_o, rays_d, near, far, workspace_bytes=budget, **kw)
    torch.cuda.synchronize()
    images = sum(v.numel() * 4 for v in out.values())
    peak = torch.cuda.max_memory_allocated() - base
    report("render_view.memory", peak=peak, budget=budget, images=images)
    assert peak <= budget + images, (peak, budget, images)
    ws = R.ViewWorkspace(ren, rays_o.shape[0] * rays_o.shape[1], budget, rays_o.device, 8)
    assert ws.chunk < rays_o.shape[0] * rays_o.shape[1]           # the budget forces several chunks


def test_render_view_perturb_draws_once_per_view(golden, scan):
    from neuraludf_b200 import render as R
    ren = _renderer(golden)
    rays_o, rays_d, near, far, kw = _view(scan)
    res = []
    for c in (None, 100):
        torch.manual_seed(7)
        res.append(R.render_view(ren, rays_o, rays_d, near, far, perturb=1.0, max_chunk=c, **kw))
    for k in res[0]:
        assert torch.equal(res[0][k], res[1][k]), k
    assert torch.isfinite(res[0]["color"]).all()


def test_cli_writes_the_runner_files(golden, scan, tmp_path):
    import cv2
    from neuraludf_b200 import render as R
    udf, col, nerf, var, beta = build_modules(golden, "cpu")
    ck = {"udf_network_fine": udf.state_dict(), "color_network_fine": col.state_dict(), "nerf": nerf.state_dict(),
          "variance_network_fine": var.state_dict(), "beta_network": beta.state_dict(), "iter_step": 1234}
    ckp = str(tmp_path / "ckpt.pth")
    torch.save(ck, ckp)
    out = str(tmp_path / "out")
    files = R.main(["--ckpt", ckp, "--scan_dir", scan.data_dir, "--views", "0", "3", "--between", "0", "1",
                    "--frames", "2", "--level", str(LEVEL), "--out_dir", out])
    H, W = 72 // LEVEL, 96 // LEVEL
    for idx in (0, 3):
        v = cv2.imread(os.path.join(out, "validations_fine", "00001234_%d.png" % idx))
        assert v.shape == (3 * H, W, 3)
        assert cv2.imread(os.path.join(out, "normals", "00001234_%d.png" % idx)).shape == (H, W, 3)
        assert np.load(os.path.join(out, "depth", "00001234_%d.npy" % idx)).shape == (H, W)
    for k in range(2):
        assert cv2.imread(os.path.join(out, "render", "%d.png" % k)).shape == (H, W, 3)
    assert len(files) == 2 * 2 + 2 + sum(1 for f in files if f.endswith(".png") and "/depth/" in f)
    # the CLI's networks equal the golden ones: its colour image is the one render_view gives
    ren = _renderer(golden)
    rays_o, rays_d, near, far, kw = _view(scan, 3)
    ref = R.render_view(ren, rays_o, rays_d, near, far, cos_anneal_ratio=1234 / 25000.0, **kw)
    img = cv2.imread(os.path.join(out, "validations_fine", "00001234_3.png"))[:H]
    p = str(tmp_path / "ref.png")
    cv2.imwrite(p, R.color_image(ref["color"].cpu().numpy()))
    np.testing.assert_array_equal(img, cv2.imread(p))


# ---- against the unmodified reference (tests/golden/render_view.*.npz, oracle/make_golden_render.py) ----
@pytest.fixture(scope="module")
def gfx():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from tests.golden_util import Fixtures
    return Fixtures("render_view")


@pytest.fixture(scope="module")
def gscan(tmp_path_factory, gfx):
    from neuraludf_b200 import render as R
    from oracle.make_golden_render import HEIGHT, N_IMAGES, WIDTH
    d = write_synthetic_dtu(str(tmp_path_factory.mktemp("gscan")), n_images=N_IMAGES, width=WIDTH, height=HEIGHT)
    return R.load_scan(d, device=DEV)


def _golden_view(gfx, gscan):
    from oracle.make_golden_render import IDX
    H, W = (int(x) for x in gfx["hw"])
    t = lambda k, c: torch.from_numpy(gfx[k]).to(DEV).reshape(H, W, c)
    cmaps, w2cs, intr = gscan.source_info(IDX)
    rot = np.linalg.inv(gscan.pose_all[IDX, :3, :3].cpu().numpy())
    return (t("rays_o", 3), t("rays_d", 3), t("near", 1), t("far", 1),
            dict(color_maps=cmaps, w2cs=w2cs, intrinsics=intr, rot=rot))


def test_render_view_strict_parity_on_reference_samples(golden, gfx, gscan):
    """on the reference's own fine samples: color, color_pixel, depth and the normal map within SURVEY 8(c)'s bound,
    max|err| <= max(1e-4 max|ref64|, 2 max|ref32 - ref64|)"""
    from neuraludf_b200 import render as R
    from oracle.make_golden_render import COS_ANNEAL
    from tests.gpu_util import parity
    ren = _renderer(golden)
    rays_o, rays_d, near, far, kw = _golden_view(gfx, gscan)
    z = torch.from_numpy(gfx["z_vals"]).to(DEV)
    out = R.render_view(ren, rays_o, rays_d, near, far, cos_anneal_ratio=COS_ANNEAL, z_vals=z, **kw)
    for k in ("color", "color_pixel", "depth", "normal"):
        r64 = torch.from_numpy(gfx["strict_%s_f64" % k])
        parity("render_view.strict." + k, out[k].reshape(r64.shape), r64, torch.from_numpy(gfx["strict_%s_f32" % k]))


def test_render_view_end_to_end_against_reference(golden, gfx, gscan):
    """with its own sampling: the same bound on every ray whose fine samples equal the reference's fp32 ones"""
    from neuraludf_b200 import render as R
    from oracle.make_golden_render import COS_ANNEAL
    from tests.gpu_util import parity
    ren = _renderer(golden)
    rays_o, rays_d, near, far, kw = _golden_view(gfx, gscan)
    out = R.render_view(ren, rays_o, rays_d, near, far, cos_anneal_ratio=COS_ANNEAL, **kw)
    # render_view's sampling stage is renderer.importance_sample on per-ray work, so one call over the view gives its z
    o, d = rays_o.reshape(-1, 3).contiguous(), rays_d.reshape(-1, 3).contiguous()
    nr, fr = near.reshape(-1, 1), far.reshape(-1, 1)
    sd = float(((fr - nr) / ren.n_samples).mean())
    with torch.no_grad():
        z0 = (nr + (fr - nr) * torch.linspace(0.0, 1.0, ren.n_samples, device=DEV)[None, :]).contiguous()
        z = ren.importance_sample(o, d, z0, sd).cpu()
    # the device and the reference's CPU scans round differently in the last bits; a ray "differs" when one of its
    # samples moved by more than 1e-4 (the scene spans ~2 along a ray: a sample drawn in another interval moves by far
    # more than that)
    zdiff = (z - torch.from_numpy(gfx["z_vals"])).abs().max(dim=1).values
    same = zdiff <= 1e-4
    n_diff = int((~same).sum())
    report("render_view.e2e.rays_with_other_samples", count=n_diff, of=int(same.numel()),
           median_z_diff=float(zdiff.median()), max_z_diff=float(zdiff.max()))
    assert n_diff <= same.numel() // 4, n_diff
    for k in ("color", "color_pixel", "depth", "normal"):
        r64 = torch.from_numpy(gfx["e2e_%s_f64" % k])
        r32 = torch.from_numpy(gfx["e2e_%s_f32" % k])
        new = out[k].reshape(r64.shape).cpu()
        parity("render_view.e2e." + k, new[same], r64[same], r32[same])


def test_rays_between_matches_reference(gfx, gscan):
    from neuraludf_b200 import render as R
    from oracle.make_golden_render import LEVEL
    for k in range(2):
        o, d, near, far, _ = R.rays_between(gscan, 0, 1, float(gfx["between%d_ratio" % k]), LEVEL)
        np.testing.assert_allclose(d.cpu().numpy(), gfx["between%d_rays_d" % k], atol=1e-5)
        np.testing.assert_allclose(o.cpu().numpy(), gfx["between%d_rays_o" % k], atol=1e-5)


def test_render_view_perturb_draws_as_render(golden, scan):
    """under one seed, render_view(perturb=1) and one render() call with perturb_overwrite=1 draw the same jitter:
    color and depth are the same bits"""
    from neuraludf_b200 import render as R
    ren = _renderer(golden)
    rays_o, rays_d, near, far, kw = _view(scan)
    torch.manual_seed(11)
    out = R.render_view(ren, rays_o, rays_d, near, far, perturb=1.0, cos_anneal_ratio=0.7, **kw)
    torch.manual_seed(11)
    with torch.no_grad():
        ref = ren.render(rays_o.reshape(-1, 3), rays_d.reshape(-1, 3), near.reshape(-1, 1), far.reshape(-1, 1),
                         cos_anneal_ratio=0.7, perturb_overwrite=1.0, color_maps=kw["color_maps"], w2cs=kw["w2cs"],
                         intrinsics=kw["intrinsics"], query_c2w=scan.pose_all[2])
    assert torch.equal(out["color"].reshape(-1, 3), ref["color"])
    assert torch.equal(out["depth"].reshape(-1, 1), ref["depth"])


# ---- against the unmodified runner's validate() ----
RUNNER_DRIVER = """
import sys
sys.path.insert(0, {root!r})
from tests import runner_env
runner_env.install_stubs()
import torch
_load = torch.load
torch.load = lambda *a, **k: _load(*a, **dict(dict(weights_only=False), **k))
from neuraludf_b200 import launch
try:
    rc = launch.main({argv!r})
except NotImplementedError as e:
    if "custom_mc" not in str(e):
        raise
    rc = 0
sys.exit(rc)
"""


def test_cli_matches_the_runner_validate(tmp_path):
    """the unmodified runner (conf perturb = 0) saves a checkpoint and runs validate() at the same iteration; the CLI
    renders that view from the checkpoint: its colour / blended colour and normal PNGs differ from the runner's by at
    most one level per channel"""
    import subprocess
    import sys
    import cv2
    from oracle import refshim
    from tests import runner_env
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if not refshim.available():
        pytest.skip("no staged reference copy (oracle/make_ref.py)")
    from neuraludf_b200 import render as R
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    ref = refshim.REFERENCE_ROOT
    tmp = str(tmp_path)
    data = runner_env.write_synthetic_dtu(os.path.join(tmp, "data", "synth"), n_images=12, width=96, height=72)
    exp = os.path.join(tmp, "exp", "CASE_NAME") + "/"
    conf = runner_env.write_conf(ref, os.path.join(tmp, "synth.conf"), os.path.join(tmp, "data", "CASE_NAME") + "/", exp,
                                 end_iter=3, batch_size=256, save_freq=3, val_freq=3, extra_replace=(("perturb", 0.0),))
    drv = os.path.join(tmp, "drive.py")
    with open(drv, "w") as f:
        f.write(RUNNER_DRIVER.format(root=root, argv=[os.path.join(ref, "exp_runner_blending.py"), "--mode", "train",
                                                      "--conf", conf, "--case", "synth", "--gpu", "0"]))
    r = subprocess.run([sys.executable, drv], cwd=tmp, capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, PYTHONUNBUFFERED="1"))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    exp_dir = os.path.join(tmp, "exp", "synth", "udf_dtu")
    runner_pngs = sorted(os.listdir(os.path.join(exp_dir, "validations_fine")))
    assert len(runner_pngs) == 1, runner_pngs
    name = runner_pngs[0]
    idx = int(name[:-4].split("_")[1])
    out = os.path.join(tmp, "cli")
    R.main(["--ckpt", os.path.join(exp_dir, "checkpoints", "ckpt_000003.pth"), "--scan_dir", data, "--views", str(idx),
            "--level", "4", "--out_dir", out])
    total = 0
    for sub in ("validations_fine", "normals"):
        a = cv2.imread(os.path.join(exp_dir, sub, name)).astype(np.int32)
        b = cv2.imread(os.path.join(out, sub, name)).astype(np.int32)
        assert a.shape == b.shape, (sub, a.shape, b.shape)
        diff = np.abs(a - b)
        n = int((diff.max(axis=-1) > 0).sum())
        total += n
        report("render_view.cli_vs_runner." + sub, differing_pixels=n, pixels=int(a.shape[0] * a.shape[1]),
               max_level_diff=int(diff.max()))
        assert diff.max() <= 1, (sub, int(diff.max()), n)

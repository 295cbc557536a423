"""The device colour loss (neuraludf_b200/loss.py, csrc/color_loss.cu) against the reference's ColorLoss: the goldens of
oracle/make_golden_loss.py, the unmodified loss/loss.py on fresh inputs at the runner's shapes, determinism, no host
synchronisation, CUDA-graph replay, and the unmodified runner's fine-tuning steps under NUDF_DEVICE_LOSS=1."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import refshim
from tests.gpu_util import parity
from tests.test_loss_proto import CASES, INPUTS, PREDS, assert_same_kept, load

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
KEYS = ["loss", "color_base_loss", "color_loss", "color_pixel_loss", "color_patch_loss"]
TYPES = ["l1", "ssd", "ssim", "ncc"]


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _device_run(fx, dev, bars=None):
    """five scalars, kept mask and gradients of the device ColorLoss on the fixture's inputs"""
    from neuraludf_b200.loss import ColorLoss
    w = fx["weights"]
    fn = ColorLoss(*w, pixel_loss_type="l1", patch_loss_type=TYPES[int(fx["patch_type"])], h_patch_size=int(fx["h"]))
    t = {k: torch.from_numpy(np.asarray(fx[k])).to(dev) for k in INPUTS if k in fx}
    for k in PREDS:
        if k in t:
            t[k].requires_grad_(True)
    out = fn(*[t.get(k) for k in INPUTS])
    vals = torch.stack([out[k] if torch.is_tensor(out[k]) else torch.zeros((), device=dev) for k in KEYS])
    if bars is None:
        out["loss"].backward()
    else:
        sum(b * out[k] for b, k in zip(bars, KEYS) if torch.is_tensor(out[k])).backward()
    kept = None if fn.kept is None else fn.kept.cpu().numpy()
    return vals.detach().cpu(), kept, {k: t[k].grad.cpu() for k in PREDS if k in t}, out


@pytest.mark.parametrize("case", CASES)
def test_matches_reference_goldens(case):
    dev = _dev()
    fx = load(case)
    vals, kept, grads, out = _device_run(fx, dev)
    for i, k in enumerate(KEYS):
        parity("loss[%s].%s" % (case, k), vals[i:i + 1], torch.from_numpy(fx["losses64"][i:i + 1]),
               torch.from_numpy(fx["losses32"][i:i + 1]))
    if "kept" in fx:
        assert_same_kept(kept, fx["kept"], fx)
    for k in PREDS:
        if k in fx:
            parity("loss[%s].d_%s" % (case, k), grads[k], torch.from_numpy(fx["d_" + k + "64"]),
                   torch.from_numpy(fx["d_" + k + "32"]))
    for i, k in enumerate(("color_base", "color", "color_pixel", "patch_colors")):
        if k not in fx:
            assert out[KEYS[1 + i]] == 0.0 and not torch.is_tensor(out[KEYS[1 + i]])


def _reference_fixture(mod, spec, x):
    """the unmodified reference's outputs for inputs x in fp32 and fp64, laid out like a golden fixture"""
    from oracle.make_golden_loss import run
    N, h, ptype, w, *_ = spec
    l32, k32, g32 = run(mod, spec, x, torch.float32)
    l64, k64, g64 = run(mod, spec, x, torch.float64)
    fx = dict(x, weights=np.array(w), h=np.array(h), patch_type=np.array(TYPES.index(ptype)), losses32=l32, losses64=l64,
              kept=k64, kept32=k32)
    fx.update({"d_%s32" % k[2:]: v for k, v in g32.items()})
    fx.update({"d_%s64" % k[2:]: v for k, v in g64.items()})
    return fx


def _fresh_inputs(N, h, ptype, seed, mod):
    """runner-shaped inputs, screened so that the k-th and (k+1)-th errors are more than 1e-4 apart (relative)"""
    from oracle.make_golden_loss import make_inputs, separated
    spec = (N, h, ptype, (0.01, 1.0, 0.1, 0.1), True, True, 0.8, seed)
    s = seed
    x = make_inputs("fresh", s, spec)
    while not separated("fresh", x, mod, spec):
        s += 1000
        x = make_inputs("fresh", s, spec)
    return _reference_fixture(mod, spec, x)


@pytest.fixture(scope="module")
def ref_loss():
    if not refshim.available():
        pytest.skip("no staged reference copy (oracle/make_ref.py)")
    from oracle.make_golden_loss import load_reference_loss
    return load_reference_loss()


@pytest.mark.parametrize("N,h,ptype", [(512, 5, "ssim"), (512, 3, "ncc"), (512, 5, "l1"), (512, 3, "ssd"), (8192, 5, "ssim")])
def test_matches_staged_reference_at_runner_shapes(ref_loss, N, h, ptype):
    dev = _dev()
    fx = _fresh_inputs(N, h, ptype, 100 + N + h, ref_loss)
    vals, kept, grads, _ = _device_run(fx, dev)
    for i, k in enumerate(KEYS):
        parity("loss_ref[%d,%d,%s].%s" % (N, h, ptype, k), vals[i:i + 1], torch.from_numpy(fx["losses64"][i:i + 1]),
               torch.from_numpy(fx["losses32"][i:i + 1]))
    assert np.array_equal(kept, fx["kept"])
    for k in PREDS:
        parity("loss_ref[%d,%d,%s].d_%s" % (N, h, ptype, k), grads[k], torch.from_numpy(fx["d_" + k + "64"]),
               torch.from_numpy(fx["d_" + k + "32"]))


@pytest.mark.parametrize("case", ["ssim_h5", "ncc_h3", "l1_h3", "coarse"])
def test_upstream_gradients_of_every_output(case):
    from tests.proto import color_loss as R
    dev = _dev()
    fx = load(case)
    bars = tuple(np.random.default_rng(3).standard_normal(5))
    _, _, grads, _ = _device_run(fx, dev, bars=bars)
    want = R.backward(fx, bars)
    for k in PREDS:
        if k in fx:
            g = torch.from_numpy(want["d_" + k])
            assert float((grads[k].double() - g).abs().max()) <= 1e-5 * float(g.abs().max()), k


def test_deterministic_bits():
    dev = _dev()
    fx = load("ssim_h5")
    a = _device_run(fx, dev)
    b = _device_run(fx, dev)
    assert torch.equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert all(torch.equal(a[2][k], b[2][k]) for k in a[2])


def _tensors(fx, dev):
    t = {k: torch.from_numpy(np.asarray(fx[k])).to(dev) for k in INPUTS if k in fx}
    for k in PREDS:
        t[k].requires_grad_(True)
    return t


def test_no_host_synchronisation():
    from neuraludf_b200.loss import ColorLoss
    dev = _dev()
    fx = load("ssim_h5")
    fn = ColorLoss(*fx["weights"], patch_loss_type="ssim", h_patch_size=5)
    t = _tensors(fx, dev)
    fn(*[t.get(k) for k in INPUTS])["loss"].backward()           # uploads the window
    torch.cuda.synchronize()
    t = _tensors(fx, dev)
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = fn(*[t.get(k) for k in INPUTS])
        out["loss"].backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(out["loss"]).item()


def test_cuda_graph_replay_equals_eager():
    from neuraludf_b200.loss import ColorLoss
    dev = _dev()
    fx = load("ncc_h5")
    fn = ColorLoss(*fx["weights"], patch_loss_type="ncc", h_patch_size=5)
    eager = _tensors(fx, dev)
    e_out = fn(*[eager.get(k) for k in INPUTS])
    e_out["loss"].backward()
    t = _tensors(fx, dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fn(*[t.get(k) for k in INPUTS])["loss"].backward()
    torch.cuda.current_stream().wait_stream(s)
    for k in PREDS:
        t[k].grad = None
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = fn(*[t.get(k) for k in INPUTS])
        out["loss"].backward()
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(out[k], e_out[k]) for k in KEYS)
    assert all(torch.equal(t[k].grad, eager[k].grad) for k in PREDS)


def test_empty_kept_set_gives_nan():
    from neuraludf_b200.loss import ColorLoss
    dev = _dev()
    fx = dict(load("ssim_h3"))
    fx["patch_mask"] = np.zeros_like(fx["patch_mask"])
    vals, kept, grads, _ = _device_run(fx, dev)
    assert torch.isnan(vals[4]) and torch.isnan(vals[0]) and not kept.any()
    assert torch.count_nonzero(grads["patch_colors"]) == 0
    with pytest.raises(RuntimeError, match="CPU"):
        ColorLoss(1, 1, 1, 1)(torch.zeros(4, 3), None, torch.zeros(4, 3), None, None, None, None, None)
    with pytest.raises(ValueError, match="shape"):
        ColorLoss(1, 1, 1, 1, h_patch_size=5)(None, None, None, None, None, torch.zeros(4, 49, 3, device=dev),
                                              torch.zeros(4, 49, 3, device=dev), torch.ones(4, 1, dtype=torch.bool, device=dev))


def test_strided_pixel_mask():
    """a float pixel mask that is a column slice (the runner's rays[:, 9:10]) gives the contiguous mask's bits"""
    dev = _dev()
    fx = load("ssim_h3")
    want = _device_run(fx, dev)
    rays = torch.rand(fx["pixel_mask"].shape[0], 10, device=dev)
    rays[:, 9:10] = torch.from_numpy(fx["pixel_mask"]).to(dev)
    from neuraludf_b200.loss import ColorLoss
    fn = ColorLoss(*fx["weights"], patch_loss_type="ssim", h_patch_size=3)
    t = {k: torch.from_numpy(np.asarray(fx[k])).to(dev) for k in INPUTS if k in fx}
    t["pixel_mask"] = rays[:, 9:10]
    assert not t["pixel_mask"].reshape(-1).is_contiguous()
    for k in PREDS:
        t[k].requires_grad_(True)
    out = fn(*[t.get(k) for k in INPUTS])
    out["loss"].backward()
    assert all(torch.equal(out[k].detach().cpu(), want[0][i]) for i, k in enumerate(KEYS))
    assert all(torch.equal(t[k].grad.cpu(), want[2][k]) for k in PREDS)


def test_nan_errors_rank_largest(ref_loss):
    """a NaN patch error ranks above every finite one on the device as in the reference's torch.sort, on a masked ray
    (excluded) and on an unmasked ray (NaN * 0 is NaN: it takes one of the k exclusion slots)"""
    dev = _dev()
    fx = {k: np.array(v) for k, v in load("ssim_h3").items() if k in INPUTS}
    mask = fx["patch_mask"][:, 0]
    on, off = int(np.flatnonzero(mask)[3]), int(np.flatnonzero(~mask)[0])
    for r in (on, off):
        fx["patch_colors"][r, 5, 1] = np.nan
    spec = (len(mask), 3, "ssim", tuple(load("ssim_h3")["weights"]), True, True, 0.8, 0)
    ref = _reference_fixture(ref_loss, spec, fx)
    vals, kept, grads, _ = _device_run(ref, dev)
    k = int(np.float32(0.3) * np.float32(mask.sum()))
    assert k >= 2 and not kept[on] and not ref["kept"][on]
    assert np.array_equal(kept, ref["kept"]) and np.array_equal(ref["kept"], ref["kept32"])
    # the unmasked NaN ray used a slot: k - 1 masked rays were excluded (the NaN one and the k - 2 largest finite errors)
    assert int(mask.sum() - kept.sum()) == k - 1
    assert torch.isfinite(vals).all()
    for i, key in enumerate(KEYS):
        parity("loss_nan.%s" % key, vals[i:i + 1], torch.from_numpy(ref["losses64"][i:i + 1]),
               torch.from_numpy(ref["losses32"][i:i + 1]))
    rows = np.ones(len(mask), bool)
    rows[[on, off]] = False                          # the reference's gradient is NaN there (0 * NaN partials); ours is 0
    for key in PREDS:
        r64, r32 = ref["d_" + key + "64"], ref["d_" + key + "32"]
        if key == "patch_colors":
            assert torch.count_nonzero(grads[key][[on, off]]) == 0
            r64, r32, g = r64[rows], r32[rows], grads[key][torch.from_numpy(rows)]
        else:
            g = grads[key]
        parity("loss_nan.d_" + key, g, torch.from_numpy(r64), torch.from_numpy(r32))


DRIVER = """
import atexit, json, sys
sys.path.insert(0, {root!r})
sys.path.insert(1, {ref!r})
from tests import runner_env
runner_env.install_stubs()
import numpy as np, torch
from torch.optim.optimizer import register_optimizer_step_pre_hook
torch.manual_seed(0)
np.random.seed(0)
from neuraludf_b200 import launch
launch.install_shadow_modules({ref!r})
import loss.loss as LM
seen = []
_fwd = LM.ColorLoss.forward
def forward(self, *a):
    out = _fwd(self, *a)
    seen.append(float(out["color_patch_loss"]))
    return out
LM.ColorLoss.forward = forward
steps = []
def pre_step(opt, args, kwargs):
    steps.append([(p.detach().cpu().clone(), None if p.grad is None else p.grad.detach().cpu().clone())
                  for g in opt.param_groups for p in g["params"]])
register_optimizer_step_pre_hook(pre_step)
def dump():
    json.dump(dict(module=LM.__file__, color_patch_loss=seen), open({log!r}, "w"))
    torch.save(steps, {log!r} + ".steps.pt")
atexit.register(dump)
try:
    rc = launch.main({argv!r})
except NotImplementedError as e:
    if "custom_mc" not in str(e):
        raise
    rc = 0
sys.exit(rc)
"""


def _run_runner(tmp, tag, device_loss, steps):
    import json
    from tests import runner_env
    ref = refshim.REFERENCE_ROOT
    root = os.path.join(tmp, tag)
    os.makedirs(root)
    data = os.path.join(root, "data", "synth")
    runner_env.write_synthetic_dtu(data, n_images=12, width=96, height=72)
    exp = os.path.join(root, "exp", "CASE_NAME") + "/"
    conf = runner_env.write_conf(ref, os.path.join(root, "ft.conf"), os.path.join(root, "data", "CASE_NAME") + "/", exp,
                                 end_iter=steps, batch_size=512, save_freq=steps, val_freq=1000,
                                 conf_name="confs/udf_dtu_blending_ft.conf")
    log = os.path.join(root, "log.json")
    drv = os.path.join(root, "drive.py")
    argv = [os.path.join(ref, "exp_runner_blending.py"), "--mode", "train", "--conf", conf, "--case", "synth", "--gpu", "0",
            "--is_finetune"]
    with open(drv, "w") as f:
        f.write(DRIVER.format(root=ROOT, ref=ref, log=log, argv=argv))
    env = dict(os.environ, PYTHONUNBUFFERED="1")
    env.pop("NUDF_DEVICE_LOSS", None)
    if device_loss:
        env["NUDF_DEVICE_LOSS"] = "1"
    r = subprocess.run([sys.executable, drv], cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + "\n---- stderr ----\n" + r.stderr[-3000:]
    return json.load(open(log)), torch.load(log + ".steps.pt", weights_only=False), r.stdout


@pytest.mark.skipif(not refshim.available(), reason="no staged reference copy (oracle/make_ref.py)")
def test_unmodified_runner_finetunes_with_device_loss(tmp_path):
    _dev()
    steps = 3
    dev_log, dev_steps, out = _run_runner(str(tmp_path), "device", True, steps)
    ref_log, ref_steps, _ = _run_runner(str(tmp_path), "reference", False, steps)
    assert dev_log["module"].startswith(os.path.join(ROOT, "neuraludf_b200"))
    assert ref_log["module"].startswith(refshim.REFERENCE_ROOT)
    assert len(dev_log["color_patch_loss"]) == len(ref_log["color_patch_loss"]) == steps
    assert len(dev_steps) == len(ref_steps) == steps
    assert re.search(r"c_patch_loss = [0-9.]+", out)
    a, b = np.array(dev_log["color_patch_loss"]), np.array(ref_log["color_patch_loss"])
    assert np.all(a > 0) and np.abs(a - b).max() <= 1e-4 * np.abs(b).max(), (a, b)
    # The runner's warm-up gives the first step a learning rate of 0, so the first two steps start from the same parameters in
    # both runs (checked bit for bit).  Their parameter gradients then differ only through the loss's gradients w.r.t. the
    # rendered colours, carried through the same renderer backward: each tensor within 1e-4 of its own max |ref|, with a
    # floor of 1e-6 of the largest gradient for tensors whose gradient is tiny.  A wrong scale, sign or ray selection in the
    # device backward breaks this; the noise of an fp32 loss gradient does not.
    worst, checked = 0.0, 0
    for i in range(2):
        assert len(dev_steps[i]) == len(ref_steps[i])
        assert all(torch.equal(pd, pr) for (pd, _), (pr, _) in zip(dev_steps[i], ref_steps[i])), "step %d" % i
        gmax = max(float(g.abs().max()) for _, g in ref_steps[i] if g is not None)
        assert gmax > 0
        for j, ((_, gd), (_, gr)) in enumerate(zip(dev_steps[i], ref_steps[i])):
            assert (gd is None) == (gr is None), (i, j)
            if gr is None:
                continue
            err = float((gd.double() - gr.double()).abs().max())
            bound = max(1e-4 * float(gr.double().abs().max()), 1e-6 * gmax)
            worst = max(worst, err / bound)
            checked += 1
            assert err <= bound, (i, j, tuple(gr.shape), err, bound)
    assert checked > 10
    from tests.gpu_util import report
    report("loss_runner_e2e", patch_loss_err=float(np.abs(a - b).max()), worst_grad_err_over_bound=worst, tensors=checked)

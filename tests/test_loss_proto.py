"""The NumPy restatement of the device colour loss (tests/proto/color_loss.py) and the op-by-op mirrors of
neuraludf_b200/loss.py against the reference's own ColorLoss (fixtures: oracle/make_golden_loss.py); CPU only."""
import glob
import os

import numpy as np
import pytest
import torch

from tests.golden_util import GOLDEN, Fixtures
from tests.proto import color_loss as R

CASES = sorted(os.path.basename(p)[len("loss_"):-len(".00.npz")] for p in glob.glob(os.path.join(GOLDEN, "loss_*.00.npz")))
INPUTS = ["color_base", "color", "gt_color", "color_pixel", "pixel_mask", "patch_colors", "gt_patch_colors", "patch_mask"]
PREDS = ["color_base", "color", "color_pixel", "patch_colors"]


def load(case):
    fx = Fixtures("loss_" + case)
    return {k: fx[k] for k in fx.files}


def rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


def test_fixture_set_covers_the_issue_cases():
    assert len(CASES) == 13
    types_h = {(int(load(c)["patch_type"]), int(load(c)["h"])) for c in CASES if "patch_colors" in load(c)}
    assert {(t, h) for t in range(4) for h in (3, 5)} <= types_h
    assert "pixel_mask" not in load("nomask_ssim_h5") and "patch_colors" not in load("coarse")
    assert load("single_ssim_h3")["gt_color"].shape[0] == 1
    assert load("sparse_ncc_h3")["patch_mask"].sum() <= 8


@pytest.mark.parametrize("case", CASES)
def test_restatement_forward_matches_reference(case):
    fx = load(case)
    losses, kept, _ = R.forward(fx)
    assert rel(losses, fx["losses64"]) < 1e-10, (losses, fx["losses64"])
    if "kept" in fx:
        assert_same_kept(kept, fx["kept"], fx)
    # fp32 reference within its own rounding of the fp64 one
    assert rel(fx["losses32"], fx["losses64"]) < 1e-4


def assert_same_kept(kept, ref, fx):
    """kept masks equal; in `zero_tie` the reference's unstable sort picks which of the tied zero-error rays it excludes,
    so there the count and every ray outside the tie must agree"""
    if "zero_tie" not in fx:
        assert np.array_equal(kept, ref)
        return
    tie = fx["zero_tie"]
    assert kept.sum() == ref.sum() and np.array_equal(kept[~tie], ref[~tie])


def test_zero_tie_lands_among_zero_errors():
    fx = load("zero_tie")
    _, kept, err = R.forward(fx)
    mask = fx["patch_mask"].reshape(-1)
    k = int(np.float32(0.3) * np.float32(mask.sum()))
    assert (err[mask] > 0).sum() < k < mask.sum()
    assert np.array_equal(fx["zero_tie"], mask & (err == 0)) and 0 < (fx["kept"] & fx["zero_tie"]).sum() < fx["zero_tie"].sum()
    assert_same_kept(kept, fx["kept"], fx)


@pytest.mark.parametrize("case", CASES)
def test_restatement_backward_matches_reference_autograd(case):
    fx = load(case)
    g = R.backward(fx)
    for k in PREDS:
        if k in fx:
            assert rel(g["d_" + k], fx["d_" + k + "64"]) < 1e-10, k


def _mirror_losses(fx, dtype=torch.float64):
    """the five scalars through the op-by-op mirrors, with autograd inputs"""
    from neuraludf_b200.loss import ColorPatchLoss, ColorPixelLoss
    t = {k: torch.from_numpy(np.asarray(fx[k])) for k in INPUTS if k in fx}
    for k in list(t):
        if t[k].dtype == torch.float32:
            t[k] = t[k].to(dtype)
            if k in PREDS:
                t[k].requires_grad_(True)
    pix = ColorPixelLoss("l1")
    z = torch.zeros((), dtype=dtype)
    terms = [pix(t[k], t["gt_color"], t.get("pixel_mask") if k != "color_pixel" else t.get("patch_mask")) if k in t else z
             for k in ("color_base", "color", "color_pixel")]
    patch = z
    if "patch_colors" in t:
        pf = ColorPatchLoss(R.PATCH_TYPES[int(fx["patch_type"])], int(fx["h"])).to(dtype)
        patch = pf(t["patch_colors"], t["gt_patch_colors"], t["patch_mask"])
    w = fx["weights"]
    total = (terms[0] * w[0] + terms[1] * w[1] + terms[2] * w[2]) / (w[0] + w[1] + w[2]) + patch * w[3]
    return torch.stack([total] + terms + [patch]), t


@pytest.mark.parametrize("case", CASES)
def test_mirror_modules_match_reference(case):
    fx = load(case)
    losses, _ = _mirror_losses(fx)
    assert rel(losses.detach().numpy(), fx["losses64"]) < 1e-10


@pytest.mark.parametrize("case", CASES)
def test_restatement_backward_matches_autograd_for_every_output(case):
    """hand-derived backward of sum_i bars_i losses_i == fp64 autograd through the op-by-op reference formulas"""
    fx = load(case)
    bars = np.random.default_rng(7).standard_normal(5)
    losses, t = _mirror_losses(fx)
    (losses * torch.from_numpy(bars)).sum().backward()
    g = R.backward(fx, tuple(bars))
    for k in PREDS:
        if k in fx:
            assert rel(g["d_" + k], t[k].grad.numpy()) < 1e-10, k


def test_create_window_matches_reference_construction():
    from neuraludf_b200.loss import create_window, gaussian
    for size in (7, 11):
        g = gaussian(size, 1.5)
        assert g.dtype == torch.float32 and abs(float(g.sum()) - 1.0) < 1e-6
        w = create_window(size, 3)
        assert w.shape == (3, 1, size, size) and torch.equal(w[0, 0], g[:, None] * g[None, :])


def test_rejection_order_rules():
    key = np.array([0.5, np.nan, 0.5, -0.0, 0.0, 1.0, -1e-7])
    assert list(R.order_rank(key)) == [2, 0, 3, 4, 5, 1, 6]

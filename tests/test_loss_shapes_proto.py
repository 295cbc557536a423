"""Pins tests/proto/color_loss.py at every configuration of the colour-loss sweep (tests/test_gpu_loss_shapes.py) against the
UNMODIFIED reference's ColorLoss (loss/loss.py with loss/patch_metric.py, run by oracle/make_golden_loss.run), in fp64 and
in fp32, on the sweep's own inputs and upstream gradients.  CPU only; skipped without a staged reference copy.

Same tolerances as tests/test_oracle_shapes_pinned.py: the fp64 proto agrees with the fp64 reference run to round-off and
the fp32 proto with the fp32 run to fp32 noise, except `const_ncc` in fp32 (below).  The five scalars, the kept mask and the
gradient of every prediction are compared.  Where the reference cannot decide, the port's documented rule is checked
instead:
  * equal keys straddling the k-th position: the reference's torch.sort is unstable and excludes any of the tied rays; the
    proto takes them in ray order.  Every ray outside the tie and the loss must agree, and the gradient rows of the tied
    rays agree up to which of the (identical) rays carries them.
  * an unmasked ray's key is 0, so when the tie is at 0 (`zero`) unmasked rays share it and take some of the k exclusion
    slots: how many masked rays the reference then excludes depends on its sort (the kept count itself is undecided).  The
    proto excludes the first k rays of the tie in ray order, masked or not."""
import numpy as np
import pytest
import torch

from oracle import refshim
from tests.proto import color_loss as R
from tests.test_gpu_loss_shapes import BARS, CFGS, TYPES, _keys, make_case
from tests.test_loss_proto import INPUTS, PREDS

TOL = {torch.float64: 1e-8, torch.float32: 2e-5}
# A constant patch leaves sigma^2 = xx - mu^2 as the cancellation residue of two values near mu^2: ~1e-7 of mu^2 in fp32,
# against SSIM's C2 = 9e-4 and NCC's 1e-4 floor.  The fp32 gradients of those rays then carry ~1e-4 (SSIM) and ~1e-3 (NCC)
# of noise in either implementation; the fp64 ones do not.
TOL32_OVERRIDE = {"const_ssim": 5e-4, "const_ncc": 1e-2}


@pytest.fixture(scope="module")
def ref_loss():
    if not refshim.available():
        pytest.skip("no staged reference copy (oracle/make_ref.py)")
    from oracle.make_golden_loss import load_reference_loss
    return load_reference_loss()


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)) if a.size else 0.0


def _ties_straddle(fx, kept):
    return "tie" in fx and 0 < int((kept & fx["tie"]).sum()) < int((fx["tie"] & fx["patch_mask"].reshape(-1)).sum())


def _ray_order_rule(fx):
    """the kept mask when equal keys are taken in ray order: a tied ray is excluded when fewer than k rays precede it
    (rays with a larger key, then tied rays with a lower number), masked or not"""
    key, k = _keys(fx)
    mask = fx["patch_mask"].reshape(-1)
    ahead = np.array([(key > v).sum() + (key[:i] == v).sum() for i, v in enumerate(key)])
    return mask & (ahead >= k)


@pytest.mark.parametrize("dtype", [torch.float64, torch.float32], ids=["f64", "f32"])
@pytest.mark.parametrize("name", list(CFGS))
def test_proto_matches_reference_at_sweep(ref_loss, name, dtype):
    from oracle.make_golden_loss import run
    N, h, ptype, *_ = CFGS[name]
    fx = make_case(name)
    x = {k: fx[k] for k in INPUTS if k in fx}
    losses, kept, grads = run(ref_loss, (N, h, ptype, tuple(fx["weights"])), x, dtype, bars=BARS)
    npdt = np.float64 if dtype == torch.float64 else np.float32
    p_losses, p_kept, _ = R.forward(fx, npdt)
    p_grads = R.backward(fx, BARS, npdt)
    tol = TOL[dtype] if dtype == torch.float64 else TOL32_OVERRIDE.get(name, TOL[dtype])
    nan = np.isnan(losses)
    assert np.array_equal(nan, np.isnan(p_losses)), (losses, p_losses)
    assert not nan.any() or (CFGS[name][5] == 0 and nan.tolist() == [True, False, False, False, True])
    assert _rel(p_losses[~nan], losses[~nan]) < TOL[dtype], (p_losses, losses)
    assert (kept is None) == (p_kept is None)
    perm = np.arange(N)
    if kept is not None:
        if _ties_straddle(fx, p_kept):
            tie = fx["tie"]
            assert np.array_equal(kept[~tie], p_kept[~tie])
            if fx["patch_mask"][tie].all():
                assert kept.sum() == p_kept.sum()
            t = np.flatnonzero(tie)
            assert np.array_equal(p_kept[t], _ray_order_rule(fx)[t])
            # map the reference's kept tied rays onto the proto's, for the row-wise gradient comparison
            if kept.sum() == p_kept.sum():
                perm[t[p_kept[t]]] = t[kept[t]]
                perm[t[~p_kept[t]]] = t[~kept[t]]
            else:                               # every tied ray has error 0: so has every gradient row (checked exactly)
                assert not grads["d_patch_colors"][t].any() and not p_grads["d_patch_colors"][t].any()
        else:
            assert np.array_equal(kept, p_kept), np.flatnonzero(kept != p_kept)
    for k in PREDS:
        if k in fx:
            g = grads["d_" + k][perm] if k == "patch_colors" else grads["d_" + k]
            assert not np.isnan(g).any(), k
            assert _rel(p_grads["d_" + k], g) < tol, (k, _rel(p_grads["d_" + k], g))


def test_sweep_reaches_the_ties_it_names():
    """the tie configurations straddle the k-th position as named, and in `zero` (every key 0, unmasked rays included)
    the first k rays in ray order are excluded"""
    for name, straddle in (("tie_km3", False), ("tie_km2", True), ("tie_km1", True), ("tie_k", False), ("zero", True)):
        fx = make_case(name)
        _, kept, err = R.forward(fx)
        assert _ties_straddle(fx, kept) == straddle, name
        assert len(set(err[fx["tie"]].tolist())) == 1, name
        assert np.array_equal(kept, _ray_order_rule(fx)), name
    fx = make_case("zero")
    _, kept, _ = R.forward(fx)
    mask = fx["patch_mask"].reshape(-1)
    assert fx["tie"].all() and not mask.all() and not mask[:12].all()
    assert np.array_equal(kept, mask & (np.arange(len(mask)) >= 12))


def test_sweep_spans_the_issue_grid():
    """every patch type at h = 1 and h = 15, every h of the sweep for ssim and ncc, the named ray counts and patch-mask
    counts"""
    cf = list(CFGS.values())
    th = {(c[2], c[1]) for c in cf if "q" in c[3]}
    for t in TYPES:
        assert {(t, 1), (t, 15)} <= th, t
    for t in ("ssim", "ncc"):
        assert {(t, h) for h in (1, 2, 4, 7, 10, 15)} <= th, t
    assert {1, 7, 31, 33, 1000, 1025, 12288, 12289, 16384} <= {c[0] for c in cf}
    counts = set()
    for name, c in CFGS.items():
        if c[5] is not None and "q" in c[3]:
            counts.add("N" if c[5] == 1.0 and isinstance(c[5], float) else int(make_case(name)["patch_mask"].sum()))
    assert {0, 1, 3, 4, 10, 20, "N"} <= counts

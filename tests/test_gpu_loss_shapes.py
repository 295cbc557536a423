"""GPU tests of the device colour loss away from the runner's shapes: a configuration sweep against the fp64 restatement.

tests/test_gpu_loss.py runs csrc/color_loss.cu at the goldens' and the runner's shapes (h = 3 and 5, N up to 8192).  The
kernels branch on much more: the per-ray warp loops `p = lane; p < npx; p += 32` (npx = 9 … 961), one warp per ray in
8-warp blocks with `ray >= N` returns, one 1024-thread rejection CTA with strided loops and block sums over partial warps,
4 N bytes of sort keys in dynamic shared memory (with the 256-byte static buffer above 48 KB from N = 12225, which needs
an opt-in, up to N = 16384), k = int(0.3f * count) at its
edges, equal keys at the k-th position, the terms each present or absent, and patches on which SSIM / NCC and their
hand-derived backward are fragile.  Each configuration below names the branch it is there for.

Every configuration is compared with tests/proto/color_loss.py in fp64 (the arbiter; tests/test_loss_shapes_proto.py pins
it against the unmodified reference at these same inputs), with the proto's own fp32 evaluation as the noise yardstick of
parity(): the five scalars, the kept mask, and the gradient of every prediction under upstream gradients on all five
outputs at once.  Inputs are built on the host from a seeded NumPy generator, so the proto and the device read the same
fp32 values; random configurations are screened so that the k-th and (k+1)-th keys are more than 1e-4 apart (relative), and
the tie configurations hold exactly equal keys, so the device must give the proto's kept mask exactly (equal keys in ray
order on both sides)."""
import time

import numpy as np
import pytest
import torch

from tests.gpu_util import parity, report
from tests.proto import color_loss as R
from tests.test_loss_proto import INPUTS, PREDS

pytestmark = pytest.mark.gpu
KEYS = ["loss", "color_base_loss", "color_loss", "color_pixel_loss", "color_patch_loss"]
TYPES = ["l1", "ssd", "ssim", "ncc"]
WEIGHTS = (0.25, 1.0, 0.5, 0.75)                     # every term visible in `loss`
BARS = (0.75, -1.25, 0.5, 2.0, -1.5)                 # upstream gradients of the five scalars (exact in fp32)
SMEM_DEFAULT = 48 * 1024                             # static + dynamic shared memory a block gets without the opt-in
SMEM_STATIC = 32 * 8                                 # reject_kernel's own: the block_sum buffer of 32 doubles
SEP = 1e-4                                           # relative gap kept between the k-th and (k+1)-th keys

# name: (N, h, patch type, terms, pixel_mask, patch-mask count, data, branch)
#   terms      b color_base, c color, p color_pixel, q patch_colors (gt_color comes with any of b, c, p)
#   pixel_mask None, "f01" float 0 / 1, "bool", "frac" float in [0, 2)
#   count      masked rays of patch_mask: an int, a fraction of N, or None for no patch_mask
#   data       "rand"; "const" constant pred patches on two rays in three (gt constant too on one of them), the third
#              ray's pred anti-correlated with its gt; "same" pred == gt on even rays;
#              "x1000" patches scaled by 1000; "zero" pred == gt on every ray; "tie<d>" three identical patches at order
#              positions k + d, k + d + 1, k + d + 2 (0-based; positions 0 .. k - 1 are excluded)
CFGS = {
    # patch sizes: the per-ray warp loops over npx = (2h + 1)^2 pixels
    "l1_h1": (40, 1, "l1", "bcpq", "f01", 0.8, "rand", "npx = 9 < 32: 23 idle lanes in every per-ray loop (L1)"),
    "ssd_h1": (40, 1, "ssd", "bcpq", "f01", 0.8, "rand", "npx = 9 < 32: idle lanes (SSD)"),
    "ssim_h1": (40, 1, "ssim", "bcpq", "f01", 0.8, "rand", "npx = 9 < 32: idle lanes in the moment and gradient loops"),
    "ncc_h1": (40, 1, "ncc", "bcpq", "f01", 0.8, "rand", "npx = 9 < 32: idle lanes in both NCC passes"),
    "ssim_h2": (64, 2, "ssim", "bcpq", "f01", 0.8, "rand", "npx = 25: one pass, 7 lanes idle"),
    "ncc_h2": (64, 2, "ncc", "bcpq", "f01", 0.8, "rand", "npx = 25: one pass, 7 lanes idle"),
    "ssim_h4": (64, 4, "ssim", "bcpq", "f01", 0.8, "rand", "npx = 81: three passes, the last with 17 lanes"),
    "ncc_h4": (64, 4, "ncc", "bcpq", "f01", 0.8, "rand", "npx = 81: three passes, the last with 17 lanes"),
    "ssim_h7": (48, 7, "ssim", "bcpq", "f01", 0.8, "rand", "npx = 225 = 7 * 32 + 1: eight passes, the last with one lane"),
    "ncc_h7": (48, 7, "ncc", "bcpq", "f01", 0.8, "rand", "npx = 225: eight passes, the last with one lane"),
    "ssim_h10": (40, 10, "ssim", "bcpq", "f01", 0.8, "rand", "npx = 441 = 13 * 32 + 25: fourteen passes"),
    "ncc_h10": (40, 10, "ncc", "bcpq", "f01", 0.8, "rand", "npx = 441: fourteen passes"),
    "l1_h15": (33, 15, "l1", "bcpq", "f01", 0.8, "rand", "npx = 961 = 30 * 32 + 1: 31 passes, the largest h accepted"),
    "ssd_h15": (33, 15, "ssd", "bcpq", "f01", 0.8, "rand", "npx = 961: 31 passes (SSD)"),
    "ssim_h15": (33, 15, "ssim", "bcpq", "f01", 0.8, "rand", "npx = 961: 31 passes of every SSIM loop"),
    "ncc_h15": (33, 15, "ncc", "bcpq", "f01", 0.8, "rand", "npx = 961: 31 passes of every NCC loop"),
    # ray counts: one warp per ray in 8-warp blocks; one 1024-thread rejection CTA
    "n1": (1, 3, "ssim", "bcpq", "f01", 1, "rand", "N = 1: one warp, 31 rejection warps idle; count 1, k = 0, one ray kept"),
    "n7": (7, 2, "ncc", "bcpq", "f01", 7, "rand", "N = 7 < 8: the block's last warp returns at ray >= N; k = 2"),
    "n31": (31, 3, "l1", "bcpq", "f01", 0.8, "rand", "N = 31 < 32: one partial warp in every rejection block sum"),
    "n33": (33, 4, "ssd", "bcpq", "f01", 0.8, "rand", "N = 33: a second rejection warp with one lane; a last block of one ray"),
    "n1000": (1000, 3, "ssim", "bcpq", "f01", 0.8, "rand", "N = 1000 < 1024: 24 rejection threads idle, 125 full ray blocks"),
    "n1025": (1025, 2, "ncc", "bcpq", "f01", 0.8, "rand", "N = 1025: rejection thread 0 strides to a second ray; a ragged "
                                                         "last ray block"),
    "n12224": (12224, 1, "l1", "bcpq", "f01", 0.8, "rand", "4 N + 256 = 48 KB: the largest N launched without the opt-in"),
    "n12225": (12225, 2, "ncc", "bcpq", "f01", 0.8, "rand", "4 N + 256 = 48 KB + 4: the first N with the opt-in"),
    "n12288": (12288, 2, "ssim", "bcpq", "f01", 0.8, "rand", "4 N = 48 KB of keys, 48 KB + 256 with the block_sum buffer: "
                                                            "launched without the opt-in, this failed (invalid argument)"),
    "n12289": (12289, 1, "ncc", "bcpq", "f01", 0.8, "rand", "4 N = 48 KB + 4 of keys alone past the default"),
    "n16384": (16384, 3, "ssim", "bcpq", "f01", 0.8, "rand", "N = kMaxRays: 64 KB of keys, the largest N accepted"),
    # rejection: k = int(0.3f * count(patch_mask))
    "q0": (64, 3, "ssim", "bcpq", "f01", 0, "rand", "no masked ray: k = 0, an empty kept set (NaN patch term and loss), "
                                                     "color_pixel over 0 + 1e-4"),
    "q1": (64, 2, "ncc", "bcpq", "f01", 1, "rand", "one masked ray: k = 0, exactly one ray kept"),
    "q3": (64, 3, "l1", "bcpq", "f01", 3, "rand", "count 3: 0.3f * 3 < 1, k = 0"),
    "q4": (64, 3, "ssd", "bcpq", "f01", 4, "rand", "count 4: k = 1"),
    "q10": (64, 3, "ssim", "bcpq", "f01", 10, "rand", "count 10: 0.3f * 10 rounds to 3 exactly in fp32, k = 3"),
    "q20": (64, 2, "ncc", "bcpq", "f01", 20, "rand", "count 20: 0.3f * 20 = 6 in fp32, k = 6"),
    "qN": (100, 2, "ssim", "bcpq", "f01", 1.0, "rand", "every ray masked: count = N, k = 30"),
    "tie_km3": (50, 3, "ssim", "bcpq", "f01", 1.0, "tie-3", "three equal keys at positions k-3 .. k-1: all excluded, "
                                                            "the boundary right after them"),
    "tie_km2": (50, 3, "ncc", "bcpq", "f01", 1.0, "tie-2", "equal keys at k-2 .. k: two excluded, one kept, by ray order"),
    "tie_km1": (50, 2, "l1", "bcpq", "f01", 1.0, "tie-1", "equal keys at k-1 .. k+1: one excluded, two kept, by ray order"),
    "tie_k": (50, 3, "ssd", "bcpq", "f01", 1.0, "tie+0", "equal keys at k .. k+2: all kept, the boundary right before them"),
    "zero": (48, 2, "l1", "bcpq", "f01", 40, "zero", "every error 0: all keys equal, unmasked ones too; the first k rays in "
                                                     "ray order take the exclusion slots; L1 gradient sign(0) = 0"),
    # term subsets
    "patch_only": (300, 3, "ssim", "q", None, 0.7, "rand", "the patch term alone: gt_color null, no pixel term"),
    "pixel_only": (300, 3, "ssim", "bcp", "f01", 0.7, "rand", "pixel terms alone: patch_mask only in color_pixel's "
                                                             "denominator, kept never written, k = 0"),
    "no_color_pixel": (300, 2, "ncc", "bcq", "f01", 0.7, "rand", "color_pixel absent with the patch term present"),
    "pm_none": (300, 3, "l1", "bcpq", None, 0.7, "rand", "pixel_mask absent: color_base / color are means over N x 3"),
    "pm_bool": (300, 3, "ssd", "bcpq", "bool", 0.7, "rand", "a bool pixel_mask, converted to float on the host"),
    "pm_frac": (300, 3, "ssim", "bcpq", "frac", 0.7, "rand", "a float pixel_mask in [0, 2): the denominator is no count"),
    "no_masks": (77, 3, "ssim", "bc", None, None, "rand", "no mask at all: both pixel terms are means"),
    # degenerate patches
    "const_ssim": (64, 3, "ssim", "bcpq", "f01", 0.8, "const", "constant patches: sigma ~ 0, SSIM on C1 / C2"),
    "const_ncc": (64, 4, "ncc", "bcpq", "f01", 0.8, "const", "constant patches: NCC on its sqrt(. + 1e-4) floor"),
    "same_ssim": (64, 3, "ssim", "bcpq", "f01", 0.8, "same", "pred == gt on half the rays: error exactly 0, gradient 0"),
    "same_ncc": (64, 2, "ncc", "bcpq", "f01", 0.8, "same", "pred == gt on half the rays: NCC below 1 by the floor only"),
    "x1000_ssim": (64, 3, "ssim", "bcpq", "f01", 0.8, "x1000", "values x 1000: xx - mu^2 cancels, C1 / C2 negligible"),
    "x1000_ncc": (64, 2, "ncc", "bcpq", "f01", 0.8, "x1000", "values x 1000: xx - mu^2 cancels, the floor negligible"),
}


def _keys(fx):
    """fp64 proto errors * mask and k of the case's patch term"""
    err = R.patch_errors(TYPES[int(fx["patch_type"])], fx["patch_colors"].astype(np.float64),
                         fx["gt_patch_colors"].astype(np.float64), R.window(int(fx["h"])))
    mask = fx["patch_mask"].reshape(-1)
    return err * mask, int(np.float32(0.3) * np.float32(mask.sum()))


def _apart(a, b):
    return abs(a - b) > SEP * max(abs(a), abs(b))


def _draw(name, seed):
    N, h, ptype, terms, pm_kind, count, data, _ = CFGS[name]
    rng = np.random.default_rng(seed)
    P = (2 * h + 1) ** 2
    f = lambda *s: rng.random(s, dtype=np.float64).astype(np.float32)  # noqa: E731
    fx = {"weights": np.array(WEIGHTS), "h": np.array(h), "patch_type": np.array(TYPES.index(ptype))}
    if set("bcp") & set(terms):
        fx["gt_color"] = f(N, 3)
    for c, k in zip("bcp", R.TERMS):
        if c in terms:
            fx[k] = f(N, 3)
    if pm_kind is not None:
        u = rng.random((N, 1))
        fx["pixel_mask"] = {"f01": (u > 0.3).astype(np.float32), "bool": u > 0.3, "frac": (2 * u).astype(np.float32)}[pm_kind]
    if count is not None:
        n = count if isinstance(count, int) else int(round(count * N))
        pm = np.zeros((N, 1), bool)
        pm[rng.choice(N, n, replace=False)] = True
        fx["patch_mask"] = pm
    if "q" not in terms:
        return fx
    gt = f(N, P, 3)
    scale = (0.02 + 0.5 * rng.random((N, 1, 1))).astype(np.float32)
    pred = np.clip(gt + scale * (f(N, P, 3) - 0.5), 0.0, 1.0).astype(np.float32)
    if data == "const":
        # a constant patch has NCC ~ 0 (error ~ 1, all within 1e-8 of each other): the anti-correlated third of the rays
        # (error > 1) holds the k-th boundary, so the constant rays are kept and their gradients checked
        pred[0::3] = pred[0::3].mean(axis=1, keepdims=True)
        pred[1::3] = pred[1::3].mean(axis=1, keepdims=True)
        gt[0::3] = gt[0::3].mean(axis=1, keepdims=True)
        pred[2::3] = np.float32(1) - pred[2::3]
    elif data == "same":
        pred[::2] = gt[::2]
    elif data == "zero":
        pred[:] = gt
    elif data == "x1000":
        pred, gt = pred * np.float32(1000), gt * np.float32(1000)
    fx["patch_colors"], fx["gt_patch_colors"] = pred, gt
    if data.startswith("tie"):
        key, k = _keys(fx)
        order = np.argsort(R.order_rank(key))
        s = k + int(data[3:])
        tie = np.zeros(N, bool)
        tie[order[s]] = tie[order[-1]] = tie[order[-2]] = True         # two rays from the bottom take the k-th's patch
        for r in (order[-1], order[-2]):
            pred[r], gt[r] = pred[order[s]], gt[order[s]]
        fx["tie"] = tie
    elif data == "zero":
        fx["tie"] = np.ones(N, bool)                                    # unmasked rays' keys are 0 as well
    return fx


def _screened(fx):
    """no key within SEP of the k-th boundary, except the exactly equal keys a tie configuration places there"""
    if "patch_colors" not in fx:
        return True
    key, k = _keys(fx)
    srt = key[np.argsort(R.order_rank(key))]
    if "tie" in fx:
        v = key[fx["tie"]]
        assert (v == v[0]).all(), "identical patches with different fp64 errors"
        s = int(np.flatnonzero(srt == v[0])[0])
        return (s == 0 or _apart(srt[s - 1], v[0])) and (s + len(v) >= len(srt) or _apart(srt[s + len(v)], v[0]))
    if k == 0 or k >= len(srt):
        return True
    return _apart(srt[k - 1], srt[k])


def make_case(name):
    """seeded fp32 inputs of configuration `name`, laid out like a golden fixture (plus `tie`: the rays of equal keys)"""
    seed = 1000 + sum(map(ord, name))
    for _ in range(50):
        fx = _draw(name, seed)
        if CFGS[name][6] == "zero" or _screened(fx):
            return fx
        seed += 7919
    raise AssertionError("no seed keeps %s's k-th key apart from its neighbours" % name)


def proto_reference(fx, bars=BARS):
    """(losses, kept, gradients) of the proto in fp64 and in fp32"""
    out = {}
    for dt in (np.float64, np.float32):
        losses, kept, _ = R.forward(fx, dt)
        out[dt] = losses, kept, R.backward(fx, bars, dt)
    return out[np.float64], out[np.float32]


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


def _run(fx, dev, bars=BARS):
    from tests.test_gpu_loss import _device_run
    return _device_run(fx, dev, bars=bars)


@pytest.mark.parametrize("name", list(CFGS))
def test_loss_shapes_vs_fp64(name):
    N, h, ptype, terms, pm_kind, count, data, why = CFGS[name]
    dev = _dev()
    fx = make_case(name)
    (l64, k64, g64), (l32, _, g32) = proto_reference(fx)
    t0 = time.perf_counter()
    vals, kept, grads, out = _run(fx, dev)
    torch.cuda.synchronize()
    seconds = time.perf_counter() - t0
    tag = "loss_shapes[%s]" % name
    for i, key in enumerate(KEYS):
        if np.isnan(l64[i]):                     # the empty kept set: the reference's mean of nothing
            assert data == "rand" and count == 0 and torch.isnan(vals[i]), (key, vals[i])
            continue
        parity(tag + "." + key, vals[i:i + 1], torch.from_numpy(l64[i:i + 1]), torch.from_numpy(l32[i:i + 1]))
    for i, (c, key) in enumerate(zip("bcpq", KEYS[1:])):
        if c not in terms:
            assert out[key] == 0.0 and not torch.is_tensor(out[key]), key
    if "q" in terms:
        # equal keys are taken in ray order on both sides, and no other key lies within SEP of the boundary
        assert np.array_equal(kept, k64), np.flatnonzero(kept != k64)
        # excluded and unmasked rays: exactly zero rows
        assert torch.count_nonzero(grads["patch_colors"][torch.from_numpy(~kept)]) == 0
    else:
        assert kept is None
    for key in PREDS:
        if key in fx:
            parity(tag + ".d_" + key, grads[key], torch.from_numpy(g64["d_" + key]), torch.from_numpy(g32["d_" + key]))
    if data == "same" or data == "zero":
        # pred == gt: the analytic gradient of those rows is 0 (SSIM and L1: round-off of it, or exactly 0)
        rows = np.zeros(N, bool)
        rows[::1 if data == "zero" else 2] = True
        rows &= fx["patch_mask"].reshape(-1)
        g = grads["patch_colors"][torch.from_numpy(rows)].double()
        if ptype == "l1":
            assert torch.count_nonzero(g) == 0
        elif ptype == "ssim":
            assert float(g.abs().max()) <= 1e-9 * max(float(grads["patch_colors"].double().abs().max()), 1e-30)
    smem = 4 * N + SMEM_STATIC if "q" in terms else 0
    if N > 12224:
        assert smem > SMEM_DEFAULT                # the forward raises the kernel's shared-memory limit
    report(tag, why=why, N=N, h=h, type=ptype, smem_bytes=smem, smem_opt_in=bool(smem > SMEM_DEFAULT),
           kept=None if kept is None else int(kept.sum()), seconds_with_copies=seconds)


def test_refusals_before_any_launch():
    """N = 16385, h = 0 and h = 16 raise through ColorLoss without a launch"""
    from neuraludf_b200 import _lib as L
    from neuraludf_b200.loss import ColorLoss
    dev = _dev()
    lib = L.lib()
    for N, h, match in ((16385, 1, "n_rays"), (4, 0, "h_patch"), (4, 16, "h_patch")):
        P = (2 * h + 1) ** 2
        x = torch.rand(N, P, 3, device=dev)
        c = torch.rand(N, 3, device=dev)
        mask = torch.ones(N, 1, dtype=torch.bool, device=dev)
        fn = ColorLoss(*WEIGHTS, patch_loss_type="ssim", h_patch_size=h)
        torch.cuda.synchronize()
        before = lib.nudf_launch_count()
        with pytest.raises(RuntimeError, match=match):
            fn(c, c, c, c, None, x.requires_grad_(True), x, mask)
        assert lib.nudf_launch_count() == before, (N, h)
    torch.cuda.synchronize()


def test_max_rays_deterministic_bits():
    """two runs at N = 16384 (keys above 48 KB of shared memory) give the same bits; the forward + backward time is
    reported (the rejection CTA's rank loop is O(N^2))"""
    from neuraludf_b200.loss import ColorLoss
    dev = _dev()
    fx = make_case("n16384")
    a = _run(fx, dev)
    b = _run(fx, dev)
    assert all(torch.equal(a[0][i], b[0][i]) or (torch.isnan(a[0][i]) and torch.isnan(b[0][i])) for i in range(5))
    assert np.array_equal(a[1], b[1])
    assert all(torch.equal(a[2][k], b[2][k]) for k in a[2])
    fn = ColorLoss(*WEIGHTS, patch_loss_type="ssim", h_patch_size=int(fx["h"]))
    t = {k: torch.from_numpy(np.asarray(fx[k])).to(dev) for k in INPUTS if k in fx}
    for k in PREDS:
        t[k].requires_grad_(True)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times = []
    for _ in range(4):
        ev[0].record()
        fn(*[t.get(k) for k in INPUTS])["loss"].backward()
        ev[1].record()
        torch.cuda.synchronize()
        times.append(ev[0].elapsed_time(ev[1]))
    report("loss_shapes.n16384_timing", ms_forward_backward=min(times[1:]), gpu=torch.cuda.get_device_name(dev))


@pytest.mark.parametrize("name", ["n1025", "pm_frac", "n16384"])
def test_pixel_gradient_rows_are_per_ray(name):
    """new pixel predictions and gt_color on the odd rays leave the even rows of every pixel-term gradient, and the whole
    patch gradient, bit for bit unchanged (the masks, and so the denominators, are kept)"""
    dev = _dev()
    fx = make_case(name)
    a = _run(fx, dev)
    fx2 = dict(fx)
    rng = np.random.default_rng(5)
    for k in ("color_base", "color", "color_pixel", "gt_color"):
        fx2[k] = fx[k].copy()
        fx2[k][1::2] = rng.random(fx2[k][1::2].shape).astype(np.float32)
    b = _run(fx2, dev)
    for k in ("color_base", "color", "color_pixel"):
        assert torch.equal(a[2][k][0::2], b[2][k][0::2]), k
        assert not torch.equal(a[2][k][1::2], b[2][k][1::2]), k
    assert torch.equal(a[2]["patch_colors"], b[2]["patch_colors"])

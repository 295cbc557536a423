"""Golden outputs of the reference's colour loss -- tests/golden/loss_<case>.NN.npz.

    python oracle/make_golden_loss.py       # needs the reference checkout or its staged copy (oracle/make_ref.py)

Each case runs the UNMODIFIED `loss/loss.py` ColorLoss (with `loss/patch_metric.py`; `icecream` and `termcolor` stubbed) on
seeded inputs, once in fp32 and once in fp64 (the same values; the module's window buffers cast with `.double()`), on the
CPU.  Stored: the inputs (`color_base`, `color`, `gt_color`, `color_pixel`, `pixel_mask`, `patch_colors`, `gt_patch_colors`,
`patch_mask`; absent ones are missing), `weights`, `h`, `patch_type`; per precision the five scalars `losses32/64` (an absent
term as 0), the kept-ray mask after the rejection `kept` (read from the reference's own sorted mask and sort indices; equal
in both precisions) and the gradients `d_<name>32/64` of `loss` w.r.t. every predicted input.

The kept set is a hard threshold of the reference (SURVEY 8(c)): the seeded inputs are screened so that the k-th and
(k+1)-th largest errors differ by more than 1e-4 relative, except in `zero_tie`, where k lands among exact zero errors on
purpose (masked rays with pred == gt; `zero_tie` marks them: the reference's unstable sort decides which of them it
excludes).
"""
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import refshim  # noqa: E402
from tests.golden_util import save_fixtures  # noqa: E402

PATCH_TYPES = ["l1", "ssd", "ssim", "ncc"]          # codes 0..3, as NUDF_PATCH_*
FT_WEIGHTS = (0.01, 1.0, 0.1, 0.1)                 # confs/udf_dtu_blending_ft.conf color_loss


def load_reference_loss():
    refshim._stub("icecream", ic=lambda *a, **k: None)
    refshim._stub("termcolor", colored=lambda s, *a, **k: s)
    for k in [k for k in sys.modules if k == "loss" or k.startswith("loss.")]:
        del sys.modules[k]
    if refshim.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, refshim.REFERENCE_ROOT)
    mod = importlib.import_module("loss.loss")
    assert mod.__file__.startswith(refshim.REFERENCE_ROOT), mod.__file__
    return mod


class _Recorder:
    """Stands in for the `torch` global of loss.py during one call and keeps the sort indices and the sorted mask (which
    the reference then edits in place, loss.py:80-82)."""

    def __init__(self):
        self.rec = {}

    def __getattr__(self, name):
        return getattr(torch, name)

    def sort(self, *a, **k):
        r = torch.sort(*a, **k)
        self.rec["indices"] = r[1]
        return r

    def index_select(self, *a, **k):
        r = torch.index_select(*a, **k)
        self.rec["mask"] = r
        return r


CASES = {
    # name: (N, h, type, weights, pixel_mask, color_pixel and patch inputs, patch-mask density, seed)
    "l1_h3": (48, 3, "l1", FT_WEIGHTS, True, True, 0.8, 1),
    "ssd_h3": (48, 3, "ssd", FT_WEIGHTS, True, True, 0.8, 2),
    "ssim_h3": (48, 3, "ssim", FT_WEIGHTS, True, True, 0.8, 3),
    "ncc_h3": (48, 3, "ncc", FT_WEIGHTS, True, True, 0.8, 4),
    "l1_h5": (48, 5, "l1", FT_WEIGHTS, True, True, 0.8, 5),
    "ssd_h5": (48, 5, "ssd", FT_WEIGHTS, True, True, 0.8, 6),
    "ssim_h5": (48, 5, "ssim", FT_WEIGHTS, True, True, 0.8, 7),
    "ncc_h5": (48, 5, "ncc", FT_WEIGHTS, True, True, 0.8, 8),
    "nomask_ssim_h5": (40, 5, "ssim", (0.5, 1.0, 0.25, 0.3), False, True, 0.7, 9),
    "coarse": (64, 3, "ssim", (0.01, 1.0, 0.0, 0.0), True, False, 0.0, 10),
    "sparse_ncc_h3": (64, 3, "ncc", FT_WEIGHTS, True, True, 0.1, 11),
    "single_ssim_h3": (1, 3, "ssim", FT_WEIGHTS, True, True, 1.0, 12),
    "zero_tie": (40, 3, "l1", FT_WEIGHTS, False, True, 1.0, 13),
}


def make_inputs(name, seed, spec=None):
    """seeded inputs of case `name` (spec: its CASES tuple, for cases outside CASES)"""
    N, h, ptype, _, has_pm, has_patch, density, _ = spec or CASES[name]
    rng = np.random.default_rng(seed)
    P = (2 * h + 1) ** 2
    f = lambda *s: rng.random(s, dtype=np.float64).astype(np.float32)  # noqa: E731
    x = {"gt_color": f(N, 3), "color_base": f(N, 3), "color": f(N, 3)}
    if has_pm:
        x["pixel_mask"] = (rng.random((N, 1)) > 0.3).astype(np.float32)
    if has_patch:
        x["color_pixel"] = f(N, 3)
        gt = f(N, P, 3)
        scale = (0.02 + 0.5 * rng.random((N, 1, 1))).astype(np.float32)
        x["gt_patch_colors"] = gt
        x["patch_colors"] = np.clip(gt + scale * (f(N, P, 3) - 0.5), 0.0, 1.0).astype(np.float32)
        pm = rng.random((N, 1)) < density
        if name == "zero_tie":
            x["patch_colors"][: 3 * N // 4] = gt[: 3 * N // 4]      # 30 masked rays with error 0; k = 12 > 10 positive ones
        if name == "single_ssim_h3":
            pm[:] = True
        x["patch_mask"] = pm
    return x


def run(mod, spec, x, dtype):
    """the reference's five scalars, kept mask and gradients for inputs x (spec: a CASES tuple)"""
    N, h, ptype, w, *_ = spec
    loss_fn = mod.ColorLoss(*w, pixel_loss_type="l1", patch_loss_type=ptype, h_patch_size=h)
    if dtype == torch.float64:
        loss_fn = loss_fn.double()
    t = {k: torch.from_numpy(v) for k, v in x.items()}
    for k in t:
        if t[k].dtype == torch.float32:
            t[k] = t[k].to(dtype)
    preds = ["color_base", "color", "color_pixel", "patch_colors"]
    for k in preds:
        if k in t:
            t[k].requires_grad_(True)
    rec = _Recorder()
    mod.torch = rec
    try:
        out = loss_fn(t["color_base"], t["color"], t["gt_color"], t.get("color_pixel"), t.get("pixel_mask"),
                      t.get("patch_colors"), t.get("gt_patch_colors"), t.get("patch_mask"))
    finally:
        mod.torch = torch
    out["loss"].backward()
    keys = ["loss", "color_base_loss", "color_loss", "color_pixel_loss", "color_patch_loss"]
    losses = np.array([float(out[k]) for k in keys], np.float64)
    kept = None
    if "patch_colors" in t:
        kept = np.zeros(N, bool)
        kept[rec.rec["indices"].numpy()] = rec.rec["mask"].reshape(N).numpy()
    grads = {"d_" + k: t[k].grad.numpy() for k in preds if k in t}
    return losses, kept, grads


def separated(name, x, mod, spec=None):
    """the k-th and (k+1)-th largest error * mask differ by more than 1e-4 relative"""
    N, h, ptype, *_ = spec or CASES[name]
    if "patch_colors" not in x or name == "zero_tie":
        return True
    pf = mod.ColorPatchLoss(ptype, h).double()
    pred, gt = torch.from_numpy(x["patch_colors"]).double(), torch.from_numpy(x["gt_patch_colors"]).double()
    e = {"l1": lambda: (pred - gt).abs().mean(-1).sum(-1), "ssd": lambda: ((pred - gt) ** 2).mean(-1).sum(-1),
         "ssim": lambda: pf.ssim(pred[:, None], gt)[:, 0], "ncc": lambda: 1 - pf.ncc(pred[:, None], gt)[:, 0]}[ptype]()
    key = np.sort((e * torch.from_numpy(x["patch_mask"][:, 0]).double()).numpy())[::-1]
    k = int(np.float32(0.3) * np.float32(x["patch_mask"].sum()))
    if k == 0 or k >= N:
        return True
    return abs(key[k - 1] - key[k]) > 1e-4 * max(abs(key[k - 1]), abs(key[k]))


def main():
    mod = load_reference_loss()
    for name, (N, h, ptype, w, *_rest, seed) in CASES.items():
        s = seed
        x = make_inputs(name, s)
        while not separated(name, x, mod):
            s += 1000
            x = make_inputs(name, s)
        l32, k32, g32 = run(mod, CASES[name], x, torch.float32)
        l64, k64, g64 = run(mod, CASES[name], x, torch.float64)
        if k32 is not None:
            assert np.array_equal(k32, k64), name
        arrays = dict(x, weights=np.array(w, np.float64), h=np.array(h), patch_type=np.array(PATCH_TYPES.index(ptype)),
                      losses32=l32, losses64=l64)
        if k64 is not None:
            arrays["kept"] = k64
        if name == "zero_tie":
            err = np.abs(x["patch_colors"].astype(np.float64) - x["gt_patch_colors"]).sum((1, 2))
            arrays["zero_tie"] = x["patch_mask"][:, 0] & (err == 0)
        for k, v in g32.items():
            arrays[k + "32"] = v
        for k, v in g64.items():
            arrays[k + "64"] = v
        save_fixtures("loss_" + name, arrays)
        print("%-16s N %3d h %d %-4s seed %5d  losses64 %s  kept %s" % (name, N, h, ptype, s, np.array2string(l64, precision=5),
                                                                        None if k64 is None else int(k64.sum())))


if __name__ == "__main__":
    main()

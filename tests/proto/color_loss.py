"""NumPy fp64 restatement of the device colour loss (csrc/color_loss.cu, neuraludf_b200/loss.py): the forward of the
reference's ColorLoss (loss/loss.py, loss/patch_metric.py) and its hand-derived backward.  The kernels follow it step by
step: per-ray Gaussian-window moments, the per-ray error, the rejection order (error * mask descending, NaN largest, equal
keys in ray order), and per-pixel gradients of the form w_p (k0 + 2 x_p k1 + y_p k2) (SSIM) or
w_p (k1 (x_p - mu1) + k0 ((y_p - mu2) - U)) (NCC).

`forward` and `backward` also run in fp32 (`dtype=np.float32`): the same formulas with fp32 arrays, the rounding noise an
fp32 evaluation of the loss has, which the device tests take as their yardstick."""
import numpy as np

PATCH_TYPES = ["l1", "ssd", "ssim", "ncc"]
C1, C2 = 0.01 ** 2, 0.03 ** 2
TERMS = ["color_base", "color", "color_pixel"]


def window(h):
    """fp32 flat Gaussian window of patch_metric.create_window(2h + 1, ., std=1.5), as float64"""
    from neuraludf_b200.loss import create_window
    return create_window(2 * h + 1, 1).reshape(-1).double().numpy()


def _moments(x, y, w):
    """x, y [N,P,3], w [P] -> mu1, mu2, xx, yy, xy, each [N,3]"""
    m = lambda t: np.einsum("npc,p->nc", t, w)  # noqa: E731
    return m(x), m(y), m(x * x), m(y * y), m(x * y)


def patch_errors(ptype, x, y, w):
    """[N] per-ray patch error (loss.py:69-76)"""
    d = x - y
    if ptype == "l1":
        return np.abs(d).mean(-1).sum(-1)
    if ptype == "ssd":
        return (d * d).mean(-1).sum(-1)
    mu1, mu2, xx, yy, xy = _moments(x, y, w)
    if ptype == "ssim":
        s1, s2, s12 = xx - mu1 ** 2, yy - mu2 ** 2, xy - mu1 * mu2
        v = 1 - ((2 * mu1 * mu2 + C1) * (2 * s12 + C2)) / ((mu1 ** 2 + mu2 ** 2 + C1) * (s1 + s2 + C2))
        return v.sum(-1) / 2
    sig1, sig2 = np.sqrt(xx - mu1 ** 2 + 1e-4), np.sqrt(yy - mu2 ** 2 + 1e-4)
    T = np.einsum("npc,p->nc", (x - mu1[:, None]) * (y - mu2[:, None]), w)
    return 1 - (T / ((sig1 + 1e-8) * (sig2 + 1e-8))).mean(-1)


def order_rank(key):
    """position of every ray in the descending order of key (NaN largest, equal keys in ray order)"""
    k = np.where(np.isnan(key), np.inf, key)
    nan = np.isnan(key)
    order = np.lexsort((np.arange(len(key)), -k, ~nan))      # NaN first, then descending, then ray index
    rank = np.empty(len(key), np.int64)
    rank[order] = np.arange(len(key))
    return rank


def kept_mask(err, mask):
    """rays left after excluding the first int(0.3f * count) of the descending order of err * mask (loss.py:78-82)"""
    key = err * mask.astype(err.dtype)
    k = int(np.float32(0.3) * np.float32(mask.sum()))
    return mask & (order_rank(key) >= k)


def n_rays(fx):
    return next(fx[k].shape[0] for k in ("gt_color", "patch_colors") if k in fx)


def _count_den(mask, dt):
    """mask.sum() + 1e-4: a bool mask's sum is an integer tensor, so torch forms count + 1e-4 in fp32 whatever the
    precision of the predictions; a float mask's in its own precision"""
    if mask.dtype == bool:
        return float(np.float32(np.float32(mask.sum()) + np.float32(1e-4)))
    return float(mask.astype(dt).sum() + dt.type(1e-4))


def denominators(fx, dtype=np.float64):
    """L1-sum denominators of the three pixel terms: mask.sum() + 1e-4, or N * 3"""
    n, dt = n_rays(fx), np.dtype(dtype)
    pm, qm = fx.get("pixel_mask"), fx.get("patch_mask")
    d = _count_den(pm, dt) if pm is not None else 3.0 * n
    dq = _count_den(qm, dt) if qm is not None else 3.0 * n
    return [d, d, dq]


def forward(fx, dtype=np.float64):
    """fx: dict of the golden's inputs (absent terms missing).  Returns losses [5], kept [N] or None, err [N] or None."""
    dt = np.dtype(dtype)
    w = np.asarray(fx["weights"], np.float64).astype(dt)
    ptype = PATCH_TYPES[int(fx["patch_type"])]
    den = denominators(fx, dt)
    gt = fx["gt_color"].astype(dt) if "gt_color" in fx else None
    terms = [np.abs(fx[t].astype(dt) - gt).sum() / den[i] if t in fx else 0.0 for i, t in enumerate(TERMS)]
    kept = err = None
    patch = 0.0
    if "patch_colors" in fx:
        err = patch_errors(ptype, fx["patch_colors"].astype(dt), fx["gt_patch_colors"].astype(dt),
                           window(int(fx["h"])).astype(dt))
        kept = kept_mask(err, fx["patch_mask"].reshape(-1))
        patch = err[kept].mean() if kept.any() else np.nan
    total = (terms[0] * w[0] + terms[1] * w[1] + terms[2] * w[2]) / (w[0] + w[1] + w[2]) + patch * w[3]
    return np.array([total] + terms + [patch], np.float64), kept, err


def backward(fx, bars=(1.0, 0.0, 0.0, 0.0, 0.0), dtype=np.float64):
    """gradients of sum_i bars[i] * losses[i] w.r.t. each present prediction, {'d_<name>': array}"""
    dt = np.dtype(dtype)
    w = np.asarray(fx["weights"], np.float64).astype(dt)
    bars = np.asarray(bars, np.float64).astype(dt)
    ws = w[0] + w[1] + w[2]
    den = denominators(fx, dt)
    gt = fx["gt_color"].astype(dt) if "gt_color" in fx else None
    out = {}
    for i, t in enumerate(TERMS):
        if t in fx:
            out["d_" + t] = np.sign(fx[t].astype(dt) - gt) * ((bars[1 + i] + bars[0] * w[i] / ws) / den[i])
    if "patch_colors" not in fx:
        return out
    ptype = PATCH_TYPES[int(fx["patch_type"])]
    x, y = fx["patch_colors"].astype(dt), fx["gt_patch_colors"].astype(dt)
    _, kept, _ = forward(fx, dt)
    g = np.where(kept, (bars[4] + bars[0] * w[3]) / max(int(kept.sum()), 1), 0.0).astype(dt)[:, None, None]   # d / d error
    if ptype == "l1":
        out["d_patch_colors"] = g * np.sign(x - y) / 3
        return out
    if ptype == "ssd":
        out["d_patch_colors"] = g * 2 * (x - y) / 3
        return out
    wp = window(int(fx["h"])).astype(dt)[None, :, None]
    mu1, mu2, xx, yy, xy = _moments(x, y, wp[0, :, 0])
    g = g[:, :, 0]
    if ptype == "ssim":
        m12, m11, m22 = mu1 * mu2, mu1 * mu1, mu2 * mu2
        A, B = 2 * m12 + C1, 2 * (xy - m12) + C2
        C, D = m11 + m22 + C1, (xx - m11) + (yy - m22) + C2
        S = A * B / (C * D)
        sA, sB, sC, sD = B / (C * D), A / (C * D), -S / C, -S / D
        h = -0.5 * g
        k0 = h * (2 * mu2 * (sA - sB) + 2 * mu1 * (sC - sD))
        k1, k2 = h * sD, h * 2 * sB
        out["d_patch_colors"] = wp * (k0[:, None] + 2 * x * k1[:, None] + y * k2[:, None])
        return out
    s1, s2 = np.sqrt(xx - mu1 ** 2 + 1e-4), np.sqrt(yy - mu2 ** 2 + 1e-4)
    ia, ib = 1 / (s1 + 1e-8), 1 / (s2 + 1e-8)
    T = np.einsum("npc,p->nc", (x - mu1[:, None]) * (y - mu2[:, None]), wp[0, :, 0])
    U = np.einsum("npc,p->nc", y - mu2[:, None], wp[0, :, 0])
    h = -g / 3
    k0, k1 = h * ib * ia, -h * ib * T * ia * ia / s1
    out["d_patch_colors"] = wp * (k1[:, None] * (x - mu1[:, None]) + k0[:, None] * ((y - mu2[:, None]) - U[:, None]))
    return out

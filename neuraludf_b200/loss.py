"""The runner's colour loss on the device: API mirror of the reference's `loss/loss.py` (`ColorLoss`, `ColorPixelLoss`,
`ColorPatchLoss`, `Normalize`) and `loss/patch_metric.py` (`gaussian`, `create_window`, `SSIM`, `NCC`).

`ColorLoss.forward` runs as one autograd function over the four predictions (`color_base`, `color`, `color_pixel`,
`patch_colors`): two launches forward (`nudf_color_loss_forward`, csrc/color_loss.cu) and one backward, with no host
synchronisation, so a training step that ends in this loss can be captured in a CUDA graph.  It computes what the reference
computes (loss.py:29-45, 59-84, 105-133; patch_metric.py:21-66):

  * a pixel term (`color_base`, `color`: `pixel_mask`; `color_pixel`: `patch_mask`) is the L1 SUM over the N x 3 errors of
    ALL rays divided by `mask.sum() + 1e-4` -- the mask enters the denominator only; without a mask it is the mean over
    N x 3.  `patch_mask` is bool, so that denominator is fp32(count) + 1e-4 in fp32;
  * the patch error of a ray is, for `patch_loss_type` l1 / ssd, the sum over the patch of the channel mean of |d| / d^2; for
    ssim, sum_c (1 - SSIM_c) / 2; for ncc, 1 - mean_c NCC_c, with the Gaussian window `create_window(2h + 1, 3, std=1.5)`
    over the whole (2h + 1)^2 patch (padding 0: each moment is a single weighted sum per channel; NCC normalises with
    sqrt(sigma^2 + 1e-4) + 1e-8);
  * rejection: k = int(0.3 * count(patch_mask)) in fp32, the first k rays of the descending order of error * mask are
    excluded, and `color_patch_loss` is the mean error of the masked rays left (NaN when none is left, as an empty mean);
  * `loss` = (sum of the weighted pixel terms) / (color_base_weight + color_weight + color_pixel_weight) +
    color_patch_loss * color_patch_weight.  A term whose input is None stays the Python float 0.0.

Deviations: equal keys of the rejection order are taken in ray order (the reference's `torch.sort` is unstable and may
exclude any of them -- unmasked rays too when the tie is at 0, so there even how many masked rays it excludes is undecided;
the loss and its gradients do not depend on which, when the tied errors are equal); NaN ranks largest as there; the
per-ray moments and formulas are evaluated in fp64 and rounded to fp32 once per ray; a bool `pixel_mask`'s count + 1e-4
is formed in fp64 (the reference forms it in fp32: a relative difference below 2^-24); no gradient flows to `gt_color` /
`gt_patch_colors`.  Inputs must be fp32 CUDA tensors (masks: any float / bool tensor for `pixel_mask`, bool for
`patch_mask`); anything else raises -- there is no fallback.

`ColorPixelLoss`, `ColorPatchLoss`, `SSIM`, `NCC` and `Normalize` are kept in the op-by-op torch form as importable
mirrors (any device); the fused path does not use them.
"""
import ctypes
import math

import torch
import torch.nn as nn

from neuraludf_b200 import _lib as L

PENALIZE_RATIO = 0.3


def gaussian(window_size, sigma):
    """fp32 [window_size]: exp(-(x - c)^2 / (2 sigma^2)) in double, rounded to fp32, normalised in fp32 (c = size // 2)."""
    c = window_size // 2
    g = torch.tensor([math.exp(-((x - c) ** 2) / float(2 * sigma ** 2)) for x in range(window_size)], dtype=torch.float32)
    return g / g.sum()


def create_window(window_size, channel, std=1.5):
    """fp32 [channel, 1, window_size, window_size]: the outer product of `gaussian` with itself, per channel."""
    g = gaussian(window_size, std)[:, None]
    w2 = torch.mm(g, g.t())
    return w2[None, None].expand(channel, 1, window_size, window_size).contiguous()


def _patch_moments(pred, gt, window):
    """pred [N,V,P,C], gt [N,P,C], window [P] -> Gaussian-weighted means and second moments, [N,V,C] (gt terms [N,1,C])."""
    w = window.to(pred.dtype)
    g = gt[:, None]
    m = lambda t: torch.einsum("nvpc,p->nvc", t, w)  # noqa: E731
    return m(pred), m(g), m(pred * pred), m(g * g), m(pred * g)


class SSIM(nn.Module):
    """1 - SSIM per channel, summed and halved: [N,V] from img_pred [N,V,P,C] and img_gt [N,P,C] (P = (2h+1)^2)."""

    def __init__(self, h_patch_size):
        super().__init__()
        self.window_size = 2 * h_patch_size + 1
        self.channel = 3
        self.register_buffer("window", create_window(self.window_size, self.channel))

    def forward(self, img_pred, img_gt):
        mu1, mu2, xx, yy, xy = _patch_moments(img_pred, img_gt, self.window[0, 0].reshape(-1))
        c1, c2 = 0.01 ** 2, 0.03 ** 2
        s1, s2, s12 = xx - mu1 ** 2, yy - mu2 ** 2, xy - mu1 * mu2
        v = 1 - ((2 * mu1 * mu2 + c1) * (2 * s12 + c2)) / ((mu1 ** 2 + mu2 ** 2 + c1) * (s1 + s2 + c2))
        return v.sum(dim=2) / 2


class NCC(nn.Module):
    """Gaussian-weighted normalised cross-correlation, mean over channels: [N,V] from img_pred [N,V,P,C], img_gt [N,P,C]."""

    def __init__(self, h_patch_size, mode='rgb'):
        super().__init__()
        self.window_size = 2 * h_patch_size + 1
        self.mode = mode
        self.channel = 3
        self.register_buffer("window", create_window(self.window_size, self.channel))

    def forward(self, img_pred, img_gt):
        w = self.window[0, 0].reshape(-1)
        mu1, mu2, xx, yy, _ = _patch_moments(img_pred, img_gt, w)
        sig1 = torch.sqrt(xx - mu1 ** 2 + 1e-4)
        sig2 = torch.sqrt(yy - mu2 ** 2 + 1e-4)
        a = (img_pred - mu1[:, :, None]) / (sig1[:, :, None] + 1e-8)
        b = (img_gt[:, None] - mu2[:, :, None]) / (sig2[:, :, None] + 1e-8)
        return torch.einsum("nvpc,p->nvc", a * b, w.to(a.dtype)).mean(dim=2)


class Normalize(nn.Module):
    def forward(self, bottom):
        return bottom / (torch.norm(bottom, p=2, dim=1, keepdim=True) + 1e-12)


class ColorPixelLoss(nn.Module):
    """L1: sum |pred - gt| / (mask.sum() + 1e-4) with a mask, the mean without one (the mask enters the denominator only)."""

    def __init__(self, type='mse'):
        super().__init__()
        self.type = type

    def forward(self, pred, gt, mask):
        err = (pred - gt).abs()
        return err.sum() / (mask.sum() + 1e-4) if mask is not None else err.mean()


class ColorPatchLoss(nn.Module):
    """Per-ray patch error with the top-30 % rejection (op by op; reads the kept count on the host)."""

    def __init__(self, type='ssim', h_patch_size=3):
        super().__init__()
        self.type = type
        self.ssim = SSIM(h_patch_size=h_patch_size)
        self.ncc = NCC(h_patch_size=h_patch_size)
        self.eps = 1e-4

    def errors(self, pred, gt):
        """[N] patch error of each ray, before masking."""
        if self.type == 'l1':
            return (pred - gt).abs().mean(dim=-1).sum(dim=-1)
        if self.type == 'ssd':
            return ((pred - gt) ** 2).mean(dim=-1).sum(dim=-1)
        if self.type == 'ssim':
            return self.ssim(pred[:, None], gt)[:, 0]
        if self.type == 'ncc':
            return 1 - self.ncc(pred[:, None], gt)[:, 0]
        raise ValueError("unknown patch loss type %r" % self.type)

    def forward(self, pred, gt, mask, penalize_ratio=PENALIZE_RATIO):
        m = mask.reshape(-1)
        key = self.errors(pred, gt) * m.float()
        order = torch.sort(key, descending=True, stable=True).indices
        kept = m.clone()
        kept[order[:int(penalize_ratio * m.sum())]] = False
        return key[kept].mean()


class _ColorLossFunction(torch.autograd.Function):
    """nudf_color_loss_forward / _backward.  Differentiable w.r.t. color_base, color, color_pixel and patch_colors."""

    @staticmethod
    def forward(ctx, args, keep, color_base, color, color_pixel, patch_colors):
        lib = L.lib()
        dev = keep[0].device
        n = args.n_rays
        losses = torch.empty(5, device=dev)
        kept = torch.empty(n, dtype=torch.bool, device=dev)
        ws = torch.empty(L.color_loss_ws_floats(n), device=dev)
        L.check(lib.nudf_color_loss_forward(ctypes.byref(args), L.ptr(losses), L.ptr(kept), L.ptr(ws), L.stream_ptr()),
                "nudf_color_loss_forward")
        ctx.set_materialize_grads(False)
        ctx.args, ctx.keep = args, keep
        ctx.save_for_backward(kept, ws, color_base, color, color_pixel, patch_colors)
        ctx.mark_non_differentiable(kept)
        return losses[0], losses[1], losses[2], losses[3], losses[4], kept

    @staticmethod
    def backward(ctx, *grads):
        lib = L.lib()
        kept, ws, *preds = ctx.saved_tensors
        bars = (ctypes.c_void_p * 5)(*[None if g is None else g.contiguous().data_ptr() for g in grads[:5]])
        outs = [torch.empty_like(p) if (p is not None and ctx.needs_input_grad[2 + i]) else None for i, p in enumerate(preds)]
        if any(o is not None for o in outs):
            L.check(lib.nudf_color_loss_backward(ctypes.byref(ctx.args), bars, L.ptr(kept), L.ptr(ws), *[L.ptr(o) for o in outs],
                                                 L.stream_ptr()), "nudf_color_loss_backward")
        return (None, None, *outs)


def _rows(t, name, n, cols):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("ColorLoss: %s is on the CPU; the device loss needs CUDA tensors (there is no CPU fallback)" % name)
    if t.dtype != torch.float32:
        raise TypeError("ColorLoss: %s must be float32, got %s" % (name, t.dtype))
    if t.numel() != n * cols or t.shape[0] != n:
        raise ValueError("ColorLoss: %s has shape %s, expected [%d, %s]" % (name, tuple(t.shape), n,
                                                                           "3" if cols == 3 else "%d, 3" % (cols // 3)))
    return t.contiguous()


def _mask(t, name, n):
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError("ColorLoss: %s is on the CPU; the device loss needs CUDA tensors (there is no CPU fallback)" % name)
    if t.numel() != n:
        raise ValueError("ColorLoss: %s has shape %s, expected [%d] or [%d, 1]" % (name, tuple(t.shape), n, n))
    return t.reshape(n).contiguous()                    # a column slice such as rays[:, 9:10] reshapes to a strided view


class ColorLoss(nn.Module):
    """loss/loss.py ColorLoss on the device kernels (module docstring).  After a forward with a patch term, `kept` is the
    device bool [N] mask of the rays the patch term averaged."""

    def __init__(self, color_base_weight, color_weight, color_pixel_weight, color_patch_weight,
                 pixel_loss_type='l1', patch_loss_type='ssim', h_patch_size=3):
        super().__init__()
        if patch_loss_type not in L.PATCH_TYPES:
            raise ValueError("unknown patch_loss_type %r (l1, ssd, ssim, ncc)" % patch_loss_type)
        self.set_color_weights(color_base_weight, color_weight, color_pixel_weight, color_patch_weight)
        self.pixel_func = ColorPixelLoss(pixel_loss_type)
        self.patch_func = ColorPatchLoss(patch_loss_type, h_patch_size)
        self.h_patch_size = h_patch_size
        self.patch_loss_type = patch_loss_type
        self.kept = None
        self._windows = {}

    def set_color_weights(self, color_base_weight, color_weight, color_pixel_weight, color_patch_weight):
        self.color_base_weight = color_base_weight
        self.color_weight = color_weight
        self.color_pixel_weight = color_pixel_weight
        self.color_patch_weight = color_patch_weight

    def _window(self, device):
        """the flat fp32 window on `device`, uploaded once (a CUDA-graph capture must follow one eager call)"""
        w = self._windows.get(device)
        if w is None:
            side = 2 * self.h_patch_size + 1
            w = self._windows[device] = create_window(side, 1).reshape(-1).to(device)
        return w

    def forward(self, color_base, color, gt_color, color_pixel, pixel_mask, patch_colors, gt_patch_colors, patch_mask):
        wb, wc, wp, wq = self.color_base_weight, self.color_weight, self.color_pixel_weight, self.color_patch_weight
        preds = (color_base, color, color_pixel, patch_colors)
        if all(p is None for p in preds):
            return {'loss': (0.0 * wb + 0.0 * wc + 0.0 * wp) / (wb + wc + wp) + 0.0 * wq, 'color_base_loss': 0.0,
                    'color_loss': 0.0, 'color_pixel_loss': 0.0, 'color_patch_loss': 0.0}
        n = next(p for p in preds if p is not None).shape[0]
        h = self.h_patch_size
        npx = (2 * h + 1) ** 2
        pix = [_rows(t, nm, n, 3) for t, nm in ((color_base, "color_base"), (color, "color"), (color_pixel, "color_pixel"))]
        gt = _rows(gt_color, "gt_color", n, 3) if any(p is not None for p in pix) else None
        if any(p is not None for p in pix) and gt is None:
            raise ValueError("ColorLoss: the pixel terms need gt_color")
        pm = _mask(pixel_mask, "pixel_mask", n)
        if pm is not None and pm.dtype != torch.float32:
            pm = pm.float()
        qm = _mask(patch_mask, "patch_mask", n)
        if qm is not None and qm.dtype != torch.bool:
            raise TypeError("ColorLoss: patch_mask must be a bool tensor (the reference indexes with it)")
        pat = _rows(patch_colors, "patch_colors", n, 3 * npx)
        gpat = None
        if pat is not None:
            if gt_patch_colors is None or qm is None:
                raise ValueError("ColorLoss: the patch term needs gt_patch_colors and patch_mask")
            gpat = _rows(gt_patch_colors, "gt_patch_colors", n, 3 * npx)
        qm8 = None if qm is None else qm.view(torch.uint8)
        dev = next(t for t in pix + [pat] if t is not None).device
        window = self._window(dev) if pat is not None else None
        args = L.ColorLossArgs(n, h, L.PATCH_TYPES[self.patch_loss_type], (ctypes.c_float * 4)(wb, wc, wp, wq),
                               *[L.ptr(t) for t in (pix[0], pix[1], pix[2], gt, pm, pat, gpat, qm8, window)])
        keep = [t for t in (gt, pm, gpat, qm8, window) if t is not None]     # alive until the backward reads them
        out = _ColorLossFunction.apply(args, keep, pix[0], pix[1], pix[2], pat)
        self.kept = out[5] if pat is not None else None
        terms = [out[1 + i] if preds[i] is not None else 0.0 for i in range(4)]
        return {'loss': out[0], 'color_base_loss': terms[0], 'color_loss': terms[1], 'color_pixel_loss': terms[2],
                'color_patch_loss': terms[3]}

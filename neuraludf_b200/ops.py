"""torch.autograd.Function wrappers over the libnudf C-ABI.

PyTorch is plumbing here: it owns the device buffers (parameters, activations, workspaces), the stream and the
autograd graph between the three kernel groups (UDF net -> colour net -> compositing).  All arithmetic is in
libnudf.so; there is no eager fallback.
"""
import ctypes

import torch

from . import _lib as L


def _require_cuda(*ts):
    """Every libnudf call launches on the CURRENT device's current stream: tensors must live there.  (One process per GPU --
    `torch.cuda.set_device(local_rank)` -- is the supported arrangement; a tensor on another device would otherwise be touched
    by kernels of the wrong device without any stream ordering.)"""
    cur = None
    for t in ts:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError("neuraludf_b200 runs on CUDA tensors only (got a %s tensor); there is no CPU path"
                               % t.device)
        if cur is None:
            cur = torch.cuda.current_device()
        if t.device.index != cur:
            raise RuntimeError("neuraludf_b200: tensor on %s but the current CUDA device is cuda:%d; call "
                               "torch.cuda.set_device(...) (one process per GPU)" % (t.device, cur))


def _f32c(t):
    if t is None:
        return None
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


_STATUS = {}


def status_word(device):
    """Per-device int32 status word the ray kernels OR their NUDF_STATUS_* bits into (device memory, never read here)."""
    key = (device.type, device.index)
    if key not in _STATUS:
        _STATUS[key] = torch.zeros(1, dtype=torch.int32, device=device)
    return _STATUS[key]


def check_status(device, extra=None):
    """ONE host read of the status word (plus `extra`, a 0-d / 1-element tensor the caller wanted on the host anyway,
    returned as a float).  Raises RuntimeError if a kernel flagged a non-finite result since the last check -- the
    reference drops into pdb at these places (udf_renderer_blending.py:97-101, 265-269, 543-544)."""
    st = status_word(device)
    if extra is None:
        bits, val = int(st.item()), None
    else:
        both = torch.cat([extra.reshape(1).double(), st.double()]).tolist()
        val, bits = both[0], int(both[1])
    if bits:
        st.zero_()
        what = []
        if bits & L.STATUS_NONFINITE_SAMPLES:
            what.append("importance sampling produced non-finite sample positions")
        if bits & L.STATUS_NONFINITE_RENDER:
            what.append("compositing produced non-finite colour / depth / regulariser values")
        raise RuntimeError("neuraludf_b200: " + "; ".join(what) + " (status bits %d)" % bits)
    return val


def _ptr_array(tensors):
    arr = (ctypes.c_void_p * len(tensors))()
    for i, t in enumerate(tensors):
        arr[i] = t.data_ptr()
    return arr


# ---------------------------------------------------------------------------------------------------------------
# UDF network
# ---------------------------------------------------------------------------------------------------------------
class UdfHandle:
    """Per-module state: C descriptor, folded-weight buffer (re-folded whenever a parameter changed)."""

    def __init__(self, layers, d_in, multires, d_out, skip_layer, scale):
        # layers: list of modules with .weight_g [out,1], .weight_v [out,in], .bias [out]
        self.layers = layers
        self.meta = (d_in, multires, d_out, skip_layer, float(scale))
        self._key = None
        self.desc = None
        self.wfold = None
        self.grad_sink = None        # dp.GradBucket region: backward writes the parameter gradients in place there

    def params(self):
        ps = []
        for m in self.layers:
            ps += [m.weight_g, m.weight_v, m.bias]
        return ps

    def sink_layout(self):
        """parameter groups in the order a gradient bucket must lay them out: the biases first, contiguous and in layer
        order (nudf_udf_backward writes dbias as ONE array), then g / v of every layer"""
        return [[m.bias for m in self.layers], [p for m in self.layers for p in (m.weight_g, m.weight_v)]]

    def invalidate(self):
        """Forget the folded weights.  The cache is keyed on (data_ptr, Tensor._version) of every parameter: optimisers and
        `load_state_dict` bump the version, writes through `param.data` do NOT -- call this after such an update."""
        self._key = None

    def refresh(self):
        ps = self.params()
        _require_cuda(*ps)
        lib_ = L.lib()
        # the folded images depend on the engine and on which chains run fused (chain mask)
        key = tuple((p.data_ptr(), p._version) for p in ps) + (lib_.nudf_get_engine(), lib_.nudf_get_tc_mask())
        if key == self._key:
            return
        d = L.UdfDesc()
        d.n_lin = len(self.layers)
        d.d_in, d.multires, d.d_out, d.skip_layer, d.scale = self.meta
        for l, m in enumerate(self.layers):
            for p in (m.weight_g, m.weight_v, m.bias):
                if p.dtype != torch.float32 or not p.is_contiguous():
                    raise RuntimeError("UDFNetwork parameters must be contiguous float32")
            d.out_dim[l], d.in_dim[l] = m.weight_v.shape
            d.weight_g[l] = m.weight_g.data_ptr()
            d.weight_v[l] = m.weight_v.data_ptr()
            d.bias[l] = m.bias.data_ptr()
        lib = L.lib()
        n = lib.nudf_udf_folded_floats(ctypes.byref(d))
        if n < 0:
            L.check(-1, "nudf_udf_folded_floats")
        dev = ps[0].device
        if self.wfold is None or self.wfold.numel() != n or self.wfold.device != dev:
            self.wfold = torch.empty(n, dtype=torch.float32, device=dev)
        L.check(lib.nudf_udf_fold_weights(ctypes.byref(d), L.ptr(self.wfold), L.stream_ptr()), "nudf_udf_fold_weights")
        self.desc = d
        self._key = key


class _UdfFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pts, handle, with_grad, split, *params):
        """split = False: (out [P, d_out], empty, grad);  split = True: (udf [P, 1], feat [P, d_out - 1], grad) as SEPARATE tensors
        (the renderer's form: no slicing of an odd-width [P, 257] tensor and no zero-fill / copy / add to reassemble its gradient)"""
        lib = L.lib()
        handle.refresh()
        pts = _f32c(pts)
        _require_cuda(pts)
        P = pts.shape[0]
        d_out = handle.meta[2]
        dev = pts.device
        grad = torch.empty(P, 3, dtype=torch.float32, device=dev) if with_grad else None
        nctx = lib.nudf_udf_ctx_floats(ctypes.byref(handle.desc), P, 1 if with_grad else 0)
        buf = torch.empty(max(nctx, 1), dtype=torch.float32, device=dev)
        if split:
            a = torch.empty(P, 1, dtype=torch.float32, device=dev)
            b = torch.empty(P, d_out - 1, dtype=torch.float32, device=dev)
            L.check(lib.nudf_udf_forward_split(ctypes.byref(handle.desc), L.ptr(handle.wfold), L.ptr(pts), P, L.ptr(a), L.ptr(b), d_out - 1,
                                               L.ptr(grad), L.ptr(buf), L.stream_ptr()), "nudf_udf_forward_split")
        else:
            a = torch.empty(P, d_out, dtype=torch.float32, device=dev)
            b = torch.empty(0, device=dev)
            L.check(lib.nudf_udf_forward(ctypes.byref(handle.desc), L.ptr(handle.wfold), L.ptr(pts), P, L.ptr(a), d_out,
                                         L.ptr(grad), L.ptr(buf), L.stream_ptr()), "nudf_udf_forward")
        ctx.handle, ctx.with_grad, ctx.P, ctx.split = handle, with_grad, P, split
        ctx.save_for_backward(pts, buf)
        ctx.key = handle._key
        ctx.set_materialize_grads(False)            # unused outputs arrive as None: a null pointer = zero gradient for the kernels
        return a, b, (grad if with_grad else torch.empty(0, device=dev))

    @staticmethod
    def backward(ctx, a_bar, b_bar, grad_bar):
        lib = L.lib()
        h = ctx.handle
        pts, buf = ctx.saved_tensors
        if h._key != ctx.key:
            raise RuntimeError("UDFNetwork parameters were modified between forward and backward")
        P = ctx.P
        if not ctx.with_grad:
            grad_bar = None
        a_bar = _f32c(a_bar)
        b_bar = _f32c(b_bar) if ctx.split else None
        grad_bar = _f32c(grad_bar)
        dev = pts.device
        nscr = lib.nudf_udf_scratch_floats(ctypes.byref(h.desc), P)
        scratch = torch.empty(max(nscr, 1), dtype=torch.float32, device=dev)
        dw = torch.empty_like(h.wfold)
        sink = h.grad_sink if (h.grad_sink is not None and h.grad_sink.begin()) else None
        if sink is not None:                  # gradients land directly in the data-parallel bucket (dp.GradBucket)
            db = sink.block([m.bias for m in h.layers])
            dgs = [sink.view(m.weight_g) for m in h.layers]
            dvs = [sink.view(m.weight_v) for m in h.layers]
            dbs = [sink.view(m.bias) for m in h.layers]
        else:
            nb = sum(int(m.bias.numel()) for m in h.layers)
            db = torch.empty(nb, dtype=torch.float32, device=dev)
            dgs = [torch.empty_like(m.weight_g) for m in h.layers]
            dvs = [torch.empty_like(m.weight_v) for m in h.layers]
            dbs, off = [], 0
            for m in h.layers:
                n = m.bias.numel()
                dbs.append(db[off:off + n])
                off += n
        if ctx.split:
            L.check(lib.nudf_udf_backward_split(ctypes.byref(h.desc), L.ptr(h.wfold), L.ptr(pts), P, L.ptr(a_bar), L.ptr(b_bar),
                                                b_bar.shape[1] if b_bar is not None else 0, L.ptr(grad_bar), L.ptr(buf),
                                                L.ptr(scratch), L.ptr(dw), L.ptr(db), L.stream_ptr()), "nudf_udf_backward_split")
        else:
            L.check(lib.nudf_udf_backward(ctypes.byref(h.desc), L.ptr(h.wfold), L.ptr(pts), P, L.ptr(a_bar),
                                          a_bar.shape[1] if a_bar is not None else 0, L.ptr(grad_bar), L.ptr(buf),
                                          L.ptr(scratch), L.ptr(dw), L.ptr(db), L.stream_ptr()), "nudf_udf_backward")
        L.check(lib.nudf_udf_unfold_grads(ctypes.byref(h.desc), L.ptr(dw), _ptr_array(dgs), _ptr_array(dvs),
                                          L.stream_ptr()), "nudf_udf_unfold_grads")
        if sink is not None:
            sink.ready()
        grads = []
        for l in range(len(h.layers)):
            grads += [dgs[l], dvs[l], dbs[l]]
        return (None, None, None, None) + tuple(grads)


def udf_forward(handle, pts, with_grad):
    """(out [P,d_out], grad [P,3] or None); differentiable w.r.t. the module parameters (not w.r.t. pts)."""
    out, _, grad = _UdfFunction.apply(pts, handle, with_grad, False, *handle.params())
    return out, (grad if with_grad else None)


def udf_forward_split(handle, pts, with_grad=True):
    """(udf [P,1], feature [P,d_out-1], grad [P,3] or None) as separate tensors -- what render_core consumes."""
    udf, feat, grad = _UdfFunction.apply(pts, handle, with_grad, True, *handle.params())
    return udf, feat, (grad if with_grad else None)


def udf_value(handle, pts):
    """udf [P] without autograd and without keeping activations (sampling / grid queries)."""
    lib = L.lib()
    handle.refresh()
    pts = _f32c(pts)
    _require_cuda(pts)
    P = pts.shape[0]
    udf = torch.empty(P, dtype=torch.float32, device=pts.device)
    n = lib.nudf_udf_ctx_floats(ctypes.byref(handle.desc), P, 0)
    work = torch.empty(max(n, 1), dtype=torch.float32, device=pts.device)
    L.check(lib.nudf_udf_value(ctypes.byref(handle.desc), L.ptr(handle.wfold), L.ptr(pts), P, L.ptr(udf), L.ptr(work),
                               L.stream_ptr()), "nudf_udf_value")
    return udf


# ---------------------------------------------------------------------------------------------------------------
# colour network
# ---------------------------------------------------------------------------------------------------------------
class ColorHandle:
    def __init__(self, base_layers, main_layers, d_feature, d_hidden, d_out, n_blend, multires_view):
        self.base, self.main = base_layers, main_layers
        self.meta = (d_feature, d_hidden, d_out, n_blend, multires_view)
        self._key = None
        self.desc = None
        self.wfold = None
        self.grad_sink = None

    def params(self):
        ps = []
        for m in list(self.main) + list(self.base):
            ps += [m.weight_g, m.weight_v, m.bias]
        return ps

    def sink_layout(self):
        """biases first in the library's order (base layers, then main layers: nudf_color_backward's dbias), then g / v"""
        mods = list(self.base) + list(self.main)
        return [[m.bias for m in mods], [p for m in mods for p in (m.weight_g, m.weight_v)]]

    def invalidate(self):
        """see UdfHandle.invalidate"""
        self._key = None

    def refresh(self):
        ps = self.params()
        _require_cuda(*ps)
        key = tuple((p.data_ptr(), p._version) for p in ps) + (L.lib().nudf_get_engine(),)
        if key == self._key:
            return
        d = L.ColorDesc()
        d.n_lin = len(self.base)
        d.d_feature, d.d_hidden, d.d_out, d.n_blend, d.multires_view = self.meta
        for l, m in enumerate(self.base):
            d.base_g[l], d.base_v[l], d.base_b[l] = m.weight_g.data_ptr(), m.weight_v.data_ptr(), m.bias.data_ptr()
        for l, m in enumerate(self.main):
            d.main_g[l], d.main_v[l], d.main_b[l] = m.weight_g.data_ptr(), m.weight_v.data_ptr(), m.bias.data_ptr()
        lib = L.lib()
        n = lib.nudf_color_folded_floats(ctypes.byref(d))
        if n < 0:
            L.check(-1, "nudf_color_folded_floats")
        dev = ps[0].device
        if self.wfold is None or self.wfold.numel() != n or self.wfold.device != dev:
            self.wfold = torch.empty(n, dtype=torch.float32, device=dev)
        L.check(lib.nudf_color_fold_weights(ctypes.byref(d), L.ptr(self.wfold), L.stream_ptr()), "nudf_color_fold_weights")
        self.desc = d
        self._key = key


class _ColorFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pts, dirs, feat, handle, samples_per_ray, *params):
        lib = L.lib()
        handle.refresh()
        pts, dirs = _f32c(pts), _f32c(dirs)
        if feat.dtype != torch.float32 or feat.stride(-1) != 1:
            feat = _f32c(feat)
        _require_cuda(pts, dirs, feat)
        P = pts.shape[0]
        d_feature, d_hidden, d_out, n_blend, _ = handle.meta
        dev = pts.device
        cb = torch.empty(P, d_out, dtype=torch.float32, device=dev)
        c = torch.empty(P, d_out, dtype=torch.float32, device=dev)
        bl = torch.empty(P, n_blend, dtype=torch.float32, device=dev)
        n = lib.nudf_color_ctx_floats(ctypes.byref(handle.desc), P)
        buf = torch.empty(max(n, 1), dtype=torch.float32, device=dev)
        L.check(lib.nudf_color_forward(ctypes.byref(handle.desc), L.ptr(handle.wfold), L.ptr(pts), L.ptr(dirs),
                                       int(samples_per_ray), L.ptr(feat), feat.stride(0), P, L.ptr(cb), L.ptr(c),
                                       L.ptr(bl), L.ptr(buf), L.stream_ptr()), "nudf_color_forward")
        ctx.handle, ctx.P, ctx.key = handle, P, handle._key
        ctx.save_for_backward(buf)
        return cb, c, bl

    @staticmethod
    def backward(ctx, cb_bar, c_bar, bl_bar):
        lib = L.lib()
        h = ctx.handle
        (buf,) = ctx.saved_tensors
        if h._key != ctx.key:
            raise RuntimeError("colour-network parameters were modified between forward and backward")
        P = ctx.P
        dev = buf.device
        cb_bar, c_bar, bl_bar = _f32c(cb_bar), _f32c(c_bar), _f32c(bl_bar)
        d_feature = h.meta[0]
        nscr = lib.nudf_color_scratch_floats(ctypes.byref(h.desc), P)
        scratch = torch.empty(max(nscr, 1), dtype=torch.float32, device=dev)
        dfeat = torch.empty(P, d_feature, dtype=torch.float32, device=dev)
        dw = torch.empty_like(h.wfold)
        mods = list(h.base) + list(h.main)
        sink = h.grad_sink if (h.grad_sink is not None and h.grad_sink.begin()) else None
        if sink is not None:
            db = sink.block([m.bias for m in mods])
            new_g = lambda m: sink.view(m.weight_g)
            new_v = lambda m: sink.view(m.weight_v)
            bb = [sink.view(m.bias) for m in h.base]
            bm = [sink.view(m.bias) for m in h.main]
        else:
            nb = sum(int(m.bias.numel()) for m in mods)
            db = torch.empty(nb, dtype=torch.float32, device=dev)
            new_g = lambda m: torch.empty_like(m.weight_g)
            new_v = lambda m: torch.empty_like(m.weight_v)
            off = 0            # bias layout in the library: base layers first, then main layers
            bb, bm = [], []
            for m in h.base:
                n = m.bias.numel(); bb.append(db[off:off + n]); off += n
            for m in h.main:
                n = m.bias.numel(); bm.append(db[off:off + n]); off += n
        L.check(lib.nudf_color_backward(ctypes.byref(h.desc), L.ptr(h.wfold), P, L.ptr(cb_bar), L.ptr(c_bar),
                                        L.ptr(bl_bar), L.ptr(buf), L.ptr(scratch), L.ptr(dfeat), d_feature, L.ptr(dw),
                                        L.ptr(db), L.stream_ptr()), "nudf_color_backward")
        dgb = [new_g(m) for m in h.base]
        dvb = [new_v(m) for m in h.base]
        dgm = [new_g(m) for m in h.main]
        dvm = [new_v(m) for m in h.main]
        L.check(lib.nudf_color_unfold_grads(ctypes.byref(h.desc), L.ptr(dw), _ptr_array(dgb), _ptr_array(dvb),
                                            _ptr_array(dgm), _ptr_array(dvm), L.stream_ptr()), "nudf_color_unfold_grads")
        if sink is not None:
            sink.ready()
        grads = []
        for l in range(len(h.main)):
            grads += [dgm[l], dvm[l], bm[l]]
        for l in range(len(h.base)):
            grads += [dgb[l], dvb[l], bb[l]]
        return (None, None, dfeat, None, None) + tuple(grads)


def color_forward(handle, pts, dirs, feat, samples_per_ray=0):
    return _ColorFunction.apply(pts, dirs, feat, handle, samples_per_ray, *handle.params())


# ---------------------------------------------------------------------------------------------------------------
# NeRF++ background network
# ---------------------------------------------------------------------------------------------------------------
class NerfHandle:
    def __init__(self, module, D, W, d_in, multires, multires_view, skip):
        self.m = module
        self.meta = (D, W, d_in, multires, multires_view, skip)
        self._key = None
        self.wimg = None
        self.grad_sink = None

    def sink_layout(self):
        return [self.params()]

    def images(self):
        """bf16 hi/lo weight images for the tensor engine, rebuilt when a parameter changed (None on the fp32 engine, or
        when neither the NeRF++ backward (chain bit 64) nor the ReLU-network forward (bit 128) runs on the tensor cores)."""
        lib = L.lib()
        if lib.nudf_get_engine() != 1 or not (lib.nudf_get_tc_mask() & (64 | 128)):
            return None
        ps = self.params()
        key = tuple((p.data_ptr(), p._version) for p in ps)
        if key != self._key:
            d = self.desc()
            n = lib.nudf_nerf_image_floats(ctypes.byref(d))
            if self.wimg is None or self.wimg.numel() != n or self.wimg.device != ps[0].device:
                self.wimg = torch.empty(n, dtype=torch.float32, device=ps[0].device)
            L.check(lib.nudf_nerf_prepare(ctypes.byref(d), L.ptr(self.wimg), L.stream_ptr()), "nudf_nerf_prepare")
            self._key = key
        return self.wimg

    def params(self):
        m = self.m
        ps = []
        for lin in m.pts_linears:
            ps += [lin.weight, lin.bias]
        for lin in (m.views_linears[0], m.feature_linear, m.alpha_linear, m.rgb_linear):
            ps += [lin.weight, lin.bias]
        return ps

    def desc(self):
        m = self.m
        d = L.NerfDesc()
        d.D, d.W, d.d_in, d.multires, d.multires_view, d.skip = self.meta
        for i, lin in enumerate(m.pts_linears):
            d.pts_w[i], d.pts_b[i] = lin.weight.data_ptr(), lin.bias.data_ptr()
        d.views_w, d.views_b = m.views_linears[0].weight.data_ptr(), m.views_linears[0].bias.data_ptr()
        d.feature_w, d.feature_b = m.feature_linear.weight.data_ptr(), m.feature_linear.bias.data_ptr()
        d.alpha_w, d.alpha_b = m.alpha_linear.weight.data_ptr(), m.alpha_linear.bias.data_ptr()
        d.rgb_w, d.rgb_b = m.rgb_linear.weight.data_ptr(), m.rgb_linear.bias.data_ptr()
        return d


class _NerfFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pts, dirs, handle, samples_per_ray, *params):
        lib = L.lib()
        _require_cuda(pts, dirs, *params)
        for p in params:
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise RuntimeError("NeRF parameters must be contiguous float32")
        pts, dirs = _f32c(pts), _f32c(dirs)
        P = pts.shape[0]
        dev = pts.device
        d = handle.desc()
        sigma = torch.empty(P, 1, dtype=torch.float32, device=dev)
        rgb = torch.empty(P, 3, dtype=torch.float32, device=dev)
        n = lib.nudf_nerf_ctx_floats(ctypes.byref(d), P)
        buf = torch.empty(max(n, 1), dtype=torch.float32, device=dev)
        wimg = handle.images()
        L.check(lib.nudf_nerf_forward(ctypes.byref(d), L.ptr(wimg), L.ptr(pts), L.ptr(dirs), int(samples_per_ray), P,
                                      L.ptr(sigma), L.ptr(rgb), L.ptr(buf), L.stream_ptr()), "nudf_nerf_forward")
        ctx.handle, ctx.P, ctx.wimg = handle, P, wimg
        ctx.save_for_backward(buf, *params)
        return sigma, rgb

    @staticmethod
    def backward(ctx, sigma_bar, rgb_bar):
        lib = L.lib()
        buf = ctx.saved_tensors[0]
        params = ctx.saved_tensors[1:]
        P = ctx.P
        dev = buf.device
        d = ctx.handle.desc()
        sigma_bar, rgb_bar = _f32c(sigma_bar), _f32c(rgb_bar)
        n = lib.nudf_nerf_scratch_floats(ctypes.byref(d), P)
        scratch = torch.empty(max(n, 1), dtype=torch.float32, device=dev)
        sink = ctx.handle.grad_sink if (ctx.handle.grad_sink is not None and ctx.handle.grad_sink.begin()) else None
        live = ctx.handle.params()
        grads = [sink.view(q) for q in live] if sink is not None else [torch.empty_like(p) for p in params]
        L.check(lib.nudf_nerf_backward(ctypes.byref(d), L.ptr(ctx.wimg), P, L.ptr(sigma_bar), L.ptr(rgb_bar), L.ptr(buf),
                                       L.ptr(scratch), _ptr_array(grads), L.stream_ptr()), "nudf_nerf_backward")
        if sink is not None:
            sink.ready()
        return (None, None, None, None) + tuple(grads)


def nerf_forward(handle, pts, dirs, samples_per_ray=0):
    return _NerfFunction.apply(pts, dirs, handle, samples_per_ray, *handle.params())


# ---------------------------------------------------------------------------------------------------------------
# ray geometry + compositing
# ---------------------------------------------------------------------------------------------------------------
def ray_points(rays_o, rays_d, z_vals, sample_dist):
    lib = L.lib()
    rays_o, rays_d, z_vals = _f32c(rays_o), _f32c(rays_d), _f32c(z_vals)
    _require_cuda(rays_o, rays_d, z_vals)
    N, S = z_vals.shape
    dev = z_vals.device
    pts = torch.empty(N * S, 3, dtype=torch.float32, device=dev)
    mid = torch.empty(N, S, dtype=torch.float32, device=dev)
    dists = torch.empty(N, S, dtype=torch.float32, device=dev)
    L.check(lib.nudf_ray_points(L.ptr(rays_o), L.ptr(rays_d), L.ptr(z_vals), N, S, float(sample_dist), L.ptr(pts),
                                L.ptr(mid), L.ptr(dists), L.stream_ptr()), "nudf_ray_points")
    return pts, mid, dists


DIAG_KEYS = ["gradient_mag", "true_cos", "vis_prob", "alpha", "alpha_plus", "alpha_minus", "alpha_occ", "raw_occ",
             "inside_sphere"]


def _make_cfg(N, S, O, sample_dist, cos_anneal_ratio, flip_saturation, sparse_scale_factor, use_norm, background_rgb):
    cfg = L.RenderCfg()
    cfg.n_rays, cfg.n_samples, cfg.n_outside = N, S, O
    cfg.sample_dist = float(sample_dist)
    cfg.has_cos_anneal = 0 if cos_anneal_ratio is None else 1
    cfg.cos_anneal_ratio = 0.0 if cos_anneal_ratio is None else float(cos_anneal_ratio)
    cfg.flip_saturation = float(flip_saturation)
    cfg.sparse_scale_factor = float(sparse_scale_factor)
    cfg.use_norm_grad_for_cosine = 1 if use_norm else 0
    cfg.has_background_rgb = 0
    if background_rgb is not None:
        cfg.has_background_rgb = 1
        vals = [float(v) for v in torch.as_tensor(background_rgb).reshape(-1).tolist()]
        if len(vals) == 1:
            vals = vals * 3
        for i in range(3):
            cfg.background_rgb[i] = vals[i]
    return cfg


class _CompositeFunction(torch.autograd.Function):
    """differentiable inputs: udf [P], grads [P,3], scb [P,3], sc [P,3], bg_alpha [N,S+O], bg_color [N,S+O,3], heads [3]"""

    @staticmethod
    def forward(ctx, udf, grads, scb, sc, bg_alpha, bg_color, heads, geom, cfg, want_diag):
        lib = L.lib()
        rays_d, pts, mid, dists = geom
        N, S, O = cfg.n_rays, cfg.n_samples, cfg.n_outside
        dev = grads.device
        if udf.dtype != torch.float32:
            udf = udf.float()
        ld_udf = udf.stride(0) if udf.dim() >= 1 and udf.numel() > 1 else 1
        grads, scb, sc, heads = _f32c(grads), _f32c(scb), _f32c(sc), _f32c(heads)
        bg_alpha, bg_color = _f32c(bg_alpha), _f32c(bg_color)
        _require_cuda(udf, grads, scb, sc, heads, rays_d, pts, mid, dists)
        f = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
        outs = {"color_base": f(N, 3), "color": f(N, 3), "depth": f(N, 1), "normals": f(N, 3), "weights": f(N, S + O),
                "weight_sum": f(N, 1), "weight_sum_fg_bg": f(N, 1), "ray_sums": f(N, 5)}
        if want_diag:
            for k in DIAG_KEYS:
                outs[k] = f(N, S)
            outs["gradients_flip"] = f(N, S, 3)
        ro = L.RenderOut()
        for k in L.RENDER_OUT_FIELDS:
            setattr(ro, k, outs[k].data_ptr() if k in outs else None)
        ro.status = status_word(dev).data_ptr()
        L.check(lib.nudf_render_composite_forward(ctypes.byref(cfg), L.ptr(heads), L.ptr(rays_d), L.ptr(pts), L.ptr(mid),
                                                  L.ptr(dists), L.ptr(udf), ld_udf, L.ptr(grads), L.ptr(scb), L.ptr(sc),
                                                  L.ptr(bg_alpha), L.ptr(bg_color), ctypes.byref(ro), L.stream_ptr()),
                "nudf_render_composite_forward")
        ctx.cfg, ctx.geom, ctx.ld_udf = cfg, geom, ld_udf
        ctx.has_bg = bg_alpha is not None
        ctx.save_for_backward(udf, grads, scb, sc, bg_alpha, bg_color, heads)
        diff = ("color_base", "color", "depth", "weight_sum", "weight_sum_fg_bg", "ray_sums", "weights")
        nondiff = [outs[k] for k in outs if k not in diff]
        ctx.mark_non_differentiable(*nondiff)
        ctx.n_extra = len(nondiff)
        ctx.extra_keys = [k for k in outs if k not in diff]
        return tuple(outs[k] for k in diff) + tuple(nondiff)

    @staticmethod
    def backward(ctx, cb_bar, c_bar, depth_bar, ws_bar, wsa_bar, rs_bar, w_bar, *unused):
        lib = L.lib()
        udf, grads, scb, sc, bg_alpha, bg_color, heads = ctx.saved_tensors
        cfg = ctx.cfg
        rays_d, pts, mid, dists = ctx.geom
        N, S, O = cfg.n_rays, cfg.n_samples, cfg.n_outside
        dev = grads.device
        P = N * S
        bar = L.RenderBar()
        keep = []
        for name, t in (("color_base", cb_bar), ("color", c_bar), ("depth", depth_bar), ("weight_sum", ws_bar),
                        ("weight_sum_fg_bg", wsa_bar), ("ray_sums", rs_bar), ("weights", w_bar)):
            t = _f32c(t)
            keep.append(t)
            setattr(bar, name, None if t is None else t.data_ptr())
        f = lambda *shape: torch.empty(*shape, dtype=torch.float32, device=dev)
        udf_bar, grads_bar, scb_bar, sc_bar = f(P), f(P, 3), f(P, 3), f(P, 3)
        bga_bar = f(N, S + O) if ctx.has_bg else None
        bgc_bar = f(N, S + O, 3) if ctx.has_bg else None
        if bgc_bar is not None:
            bgc_bar[:, :S].zero_()
        scal = f(N, 3)
        L.check(lib.nudf_render_composite_backward(ctypes.byref(cfg), L.ptr(heads), L.ptr(rays_d), L.ptr(pts), L.ptr(mid),
                                                   L.ptr(dists), L.ptr(udf), ctx.ld_udf, L.ptr(grads), L.ptr(scb),
                                                   L.ptr(sc), L.ptr(bg_alpha), L.ptr(bg_color), ctypes.byref(bar),
                                                   L.ptr(udf_bar), L.ptr(grads_bar), L.ptr(scb_bar), L.ptr(sc_bar),
                                                   L.ptr(bga_bar), L.ptr(bgc_bar), L.ptr(scal), L.stream_ptr()),
                "nudf_render_composite_backward")
        # udf came in as a (possibly strided) [P] view
        return (udf_bar.reshape(udf.shape), grads_bar, scb_bar, sc_bar, bga_bar, bgc_bar, scal.sum(dim=0),
                None, None, None)


def composite(udf, grads, scb, sc, bg_alpha, bg_color, heads, geom, cfg, want_diag=True):
    res = _CompositeFunction.apply(udf, grads, scb, sc, bg_alpha, bg_color, heads, geom, cfg, want_diag)
    names = ["color_base", "color", "depth", "weight_sum", "weight_sum_fg_bg", "ray_sums", "weights", "normals"]
    if want_diag:
        names += DIAG_KEYS + ["gradients_flip"]
    return dict(zip(names, res))


# ---------------------------------------------------------------------------------------------------------------
# pixel / patch blending (fine-tuning stage)
# ---------------------------------------------------------------------------------------------------------------
class _BlendFunction(torch.autograd.Function):
    """Fused projection + bilinear gathers + masked-softmax view fusion (nudf_blend_forward / _backward).  Differentiable
    w.r.t. the blending logits only; points, projections, homographies and images are constants of the graph."""

    @staticmethod
    def forward(ctx, logits, pts, proj, hom, px, imgs, n_rays, n_samples, h_patch):
        lib = L.lib()
        P = n_rays * n_samples
        V, _, H, W = imgs.shape
        cfg = L.BlendCfg(n_rays, n_samples, V, H, W, h_patch)
        logits = logits.contiguous()
        c_pix = torch.empty(P, 3, device=pts.device)
        npx = (2 * h_patch + 1) ** 2
        c_pat = torch.empty(P, npx, 3, device=pts.device) if hom is not None else None
        m_pat = torch.empty(P, device=pts.device) if hom is not None else None
        L.check(lib.nudf_blend_forward(ctypes.byref(cfg), L.ptr(pts), L.ptr(proj), L.ptr(hom), L.ptr(px), L.ptr(imgs), L.ptr(logits),
                                       logits.stride(0), L.ptr(c_pix), L.ptr(c_pat), L.ptr(m_pat), L.stream_ptr()),
                "nudf_blend_forward")
        ctx.cfg, ctx.has_patch, ctx.n_logits = cfg, hom is not None, logits.shape[1]
        ctx.save_for_backward(logits, pts, proj, hom, px, imgs)
        if hom is None:
            return c_pix, None, None
        ctx.mark_non_differentiable(m_pat)
        return c_pix, c_pat, m_pat

    @staticmethod
    def backward(ctx, g_pix, g_pat, _g_mask):
        lib = L.lib()
        logits, pts, proj, hom, px, imgs = ctx.saved_tensors
        V = ctx.cfg.n_views
        P = pts.shape[0]
        g_pix = g_pix.contiguous() if g_pix is not None else None
        g_pat = g_pat.contiguous() if (g_pat is not None and ctx.has_patch) else None
        g_log = torch.zeros(P, ctx.n_logits, device=pts.device)
        g_v = torch.empty(P, V, device=pts.device)
        L.check(lib.nudf_blend_backward(ctypes.byref(ctx.cfg), L.ptr(pts), L.ptr(proj), L.ptr(hom), L.ptr(px), L.ptr(imgs),
                                        L.ptr(logits), logits.stride(0), L.ptr(g_pix), L.ptr(g_pat), L.ptr(g_v), L.stream_ptr()),
                "nudf_blend_backward")
        g_log[:, :V] = g_v
        return g_log, None, None, None, None, None, None, None, None


def blend_views(logits, pts, proj, hom, px, imgs, n_rays, n_samples, h_patch):
    """logits [P, >=V] (grad), pts [P,3], proj [V,12], hom [V,P,9] or None, px [n_rays,2] or None, imgs [V,3,H,W] ->
    blended pixel colour [P,3], blended patch colours [P,Npx,3] or None, patch-visible mask [P] (0/1) or None."""
    f = lambda t: None if t is None else t.detach().float().contiguous()
    return _BlendFunction.apply(logits, f(pts), f(proj), f(hom), f(px), f(imgs), int(n_rays), int(n_samples), int(h_patch))


# ---------------------------------------------------------------------------------------------------------------
# sampling
# ---------------------------------------------------------------------------------------------------------------
_U_CACHE = {}


def _u_lin(m, device):
    key = (m, str(device))
    if key not in _U_CACHE:
        # computed by torch's CPU linspace (the reference's arithmetic, udf_renderer_blending.py:76), then uploaded
        _U_CACHE[key] = torch.linspace(0.0 + 0.5 / m, 1.0 - 0.5 / m, steps=m, device="cpu").to(device)
    return _U_CACHE[key]


def up_sample(mode, rays_o, rays_d, z, udf, sample_dist, m, inv_s, beta, gamma, return_inds=False):
    lib = L.lib()
    rays_o, rays_d, z, udf = _f32c(rays_o), _f32c(rays_d), _f32c(z), _f32c(udf)
    _require_cuda(rays_o, rays_d, z, udf)
    N, n = z.shape
    new_z = torch.empty(N, m, dtype=torch.float32, device=z.device)
    inds = torch.empty(N, m, dtype=torch.int64, device=z.device) if return_inds else None
    L.check(lib.nudf_up_sample(int(mode), L.ptr(rays_o), L.ptr(rays_d), L.ptr(z), L.ptr(udf), N, n, m, float(sample_dist),
                               float(inv_s), float(beta), float(gamma), L.ptr(_u_lin(m, z.device)), L.ptr(new_z),
                               L.ptr(inds), L.ptr(status_word(z.device)), L.stream_ptr()), "nudf_up_sample")
    return (new_z, inds) if return_inds else new_z


def sample_pdf(bins, weights, m, return_inds=False):
    lib = L.lib()
    bins, weights = _f32c(bins), _f32c(weights)
    _require_cuda(bins, weights)
    N, n = bins.shape
    samples = torch.empty(N, m, dtype=torch.float32, device=bins.device)
    inds = torch.empty(N, m, dtype=torch.int64, device=bins.device) if return_inds else None
    L.check(lib.nudf_sample_pdf(L.ptr(bins), L.ptr(weights), N, n, m, L.ptr(_u_lin(m, bins.device)), L.ptr(samples),
                                L.ptr(inds), L.ptr(status_word(bins.device)), L.stream_ptr()), "nudf_sample_pdf")
    return (samples, inds) if return_inds else samples


def merge_z(z, new_z, udf=None, new_udf=None):
    lib = L.lib()
    z, new_z, udf, new_udf = _f32c(z), _f32c(new_z), _f32c(udf), _f32c(new_udf)
    N, n = z.shape
    m = new_z.shape[1]
    z_out = torch.empty(N, n + m, dtype=torch.float32, device=z.device)
    udf_out = torch.empty(N, n + m, dtype=torch.float32, device=z.device) if udf is not None else None
    L.check(lib.nudf_merge_z(L.ptr(z), L.ptr(new_z), L.ptr(udf), L.ptr(new_udf), N, n, m, L.ptr(z_out), L.ptr(udf_out),
                             L.stream_ptr()), "nudf_merge_z")
    return z_out, udf_out


def points_on_rays(rays_o, rays_d, z):
    lib = L.lib()
    rays_o, rays_d, z = _f32c(rays_o), _f32c(rays_d), _f32c(z)
    N, n = z.shape
    pts = torch.empty(N * n, 3, dtype=torch.float32, device=z.device)
    L.check(lib.nudf_points_on_rays(L.ptr(rays_o), L.ptr(rays_d), L.ptr(z), N, n, L.ptr(pts), L.stream_ptr()),
            "nudf_points_on_rays")
    return pts


def outside_points(rays_o, rays_d, z, col0, sample_dist):
    lib = L.lib()
    rays_o, rays_d, z = _f32c(rays_o), _f32c(rays_d), _f32c(z)
    N, n = z.shape
    m = n - col0
    pts4 = torch.empty(N * m, 4, dtype=torch.float32, device=z.device)
    dists = torch.empty(N, m, dtype=torch.float32, device=z.device)
    L.check(lib.nudf_outside_points(L.ptr(rays_o), L.ptr(rays_d), L.ptr(z), N, n, col0, float(sample_dist), L.ptr(pts4),
                                    L.ptr(dists), L.stream_ptr()), "nudf_outside_points")
    return pts4, dists


# ---------------------------------------------------------------------------------------------------------------
# forward-only view rendering: the network forwards and the compositing pass outside autograd, every per-chunk array
# carved from one caller-owned workspace
# ---------------------------------------------------------------------------------------------------------------
def udf_forward_split_into(handle, pts, udf, feat, grad, ctx):
    """nudf_udf_forward_split into given buffers: udf [P], feat [P, d_out - 1], grad [P,3]; ctx is scratch (no backward)."""
    lib = L.lib()
    handle.refresh()
    L.check(lib.nudf_udf_forward_split(ctypes.byref(handle.desc), L.ptr(handle.wfold), L.ptr(pts), pts.shape[0], L.ptr(udf),
                                       L.ptr(feat), feat.shape[1], L.ptr(grad), L.ptr(ctx), L.stream_ptr()),
            "nudf_udf_forward_split")


def color_forward_into(handle, pts, dirs, samples_per_ray, feat, cb, c, bl, ctx):
    lib = L.lib()
    handle.refresh()
    L.check(lib.nudf_color_forward(ctypes.byref(handle.desc), L.ptr(handle.wfold), L.ptr(pts), L.ptr(dirs),
                                   int(samples_per_ray), L.ptr(feat), feat.stride(0), pts.shape[0], L.ptr(cb), L.ptr(c),
                                   L.ptr(bl), L.ptr(ctx), L.stream_ptr()), "nudf_color_forward")


def nerf_forward_into(handle, pts, dirs, samples_per_ray, sigma, rgb, ctx):
    lib = L.lib()
    L.check(lib.nudf_nerf_forward(ctypes.byref(handle.desc()), L.ptr(handle.images()), L.ptr(pts), L.ptr(dirs),
                                  int(samples_per_ray), pts.shape[0], L.ptr(sigma), L.ptr(rgb), L.ptr(ctx), L.stream_ptr()),
            "nudf_nerf_forward")


def view_composite(cfg, heads, rays_d, pts, mid, dists, udf, grads, sc, c_pix, bg_alpha, bg_color, rot, outs):
    """nudf_render_view_forward: outs maps color / color_pixel / depth / normal / weight_sum to [N, .] tensors (views
    into the image buffers are fine) or None; rot is a host 3x3 (nested sequence or array)."""
    lib = L.lib()
    ro = L.ViewOut()
    for k in L.VIEW_OUT_FIELDS:
        t = outs.get(k)
        setattr(ro, k, None if t is None else t.data_ptr())
    r9 = (ctypes.c_float * 9)(*[float(v) for row in rot for v in row])
    L.check(lib.nudf_render_view_forward(ctypes.byref(cfg), L.ptr(heads), L.ptr(rays_d), L.ptr(pts), L.ptr(mid), L.ptr(dists),
                                         L.ptr(udf), 1, L.ptr(grads), L.ptr(sc), L.ptr(c_pix), L.ptr(bg_alpha),
                                         L.ptr(bg_color), r9, ctypes.byref(ro), L.stream_ptr()), "nudf_render_view_forward")


class ViewWorkspace:
    """One fp32 buffer holding every array of one chunk of the forward-only view pipeline (render.render_view).

    The network forwards keep no state for a backward pass, so their context buffers are scratch: the UDF, colour and
    NeRF++ forwards (and the sampling stage's UDF value queries) share one region sized for the largest of them.  The
    chunk size is the largest ray count whose arrays fit `budget_bytes`, from the library's nudf_*_ctx_floats queries."""

    def __init__(self, renderer, n_rays, budget_bytes, device, n_views=0):
        lib = L.lib()
        udf_h = renderer.udf_network._handle
        udf_h.refresh()
        col_h = renderer.color_network._handle
        col_h.refresh()
        self.S0, self.S = renderer.n_samples, renderer.n_samples + renderer.n_importance
        self.O = renderer.n_outside
        self.F = udf_h.meta[2] - 1
        self.nb = col_h.meta[3]
        self.blend = n_views > 0
        # NeRF++ columns evaluated per ray: all S+O when the pixel blend needs the inside columns too (render() does the same)
        self.m = (self.S + self.O if self.blend else self.O) if self.O > 0 else 0
        nerf_d = renderer.nerf._handle.desc() if self.O > 0 else None
        S, SO, m = self.S, self.S + self.O, self.m

        def ctx(n):
            c = [lib.nudf_udf_ctx_floats(ctypes.byref(udf_h.desc), n * S, 1),
                 lib.nudf_udf_ctx_floats(ctypes.byref(udf_h.desc), n * self.S0, 0),
                 lib.nudf_color_ctx_floats(ctypes.byref(col_h.desc), n * S)]
            if m:
                c.append(lib.nudf_nerf_ctx_floats(ctypes.byref(nerf_d), n * m))
            return max(c)

        # per ray: pts, mid, dists, udf, feat, grad, cb, c, logits (+ c_pix) of S samples; NeRF++ inputs / outputs of m
        # columns and the [S+O] background arrays; sampling and z-sorting temporaries (z, udf, points of each round)
        self._per_ray = (S * (3 + 1 + 1 + 1 + self.F + 3 + 3 + 3 + self.nb + (3 if self.blend else 0))
                         + m * (4 + 1 + 1 + 3) + SO * (1 + 3) + 8 * SO)
        self._ctx = ctx
        # the sampling stage's UDF value queries allocate their own scratch while the workspace is live: counted twice
        total = lambda n: n * self._per_ray + 2 * ctx(n)
        probe = min(4096, n_rays)
        n = max(1, min(n_rays, int(budget_bytes // 4 * probe // total(probe))))
        while n > 1 and total(n) * 4 > budget_bytes:
            n = max(1, n * 15 // 16)
        self.chunk = n
        self.buf = torch.empty(n * (self._per_ray - 8 * SO) + ctx(n) + 64 * 16, dtype=torch.float32, device=device)

    def carve(self, n):
        """views of the workspace for a chunk of n <= self.chunk rays"""
        S, SO, m = self.S, self.S + self.O, self.m
        off = [0]
        buf = self.buf

        def take(*shape):             # every array starts on a 256-byte boundary (vector loads in the kernels)
            k = 1
            for s in shape:
                k *= s
            t = buf[off[0]:off[0] + k].view(*shape)
            off[0] += -(-k // 64) * 64
            return t
        w = {"pts": take(n * S, 3), "mid": take(n, S), "dists": take(n, S), "udf": take(n * S), "feat": take(n * S, self.F),
             "grad": take(n * S, 3), "cb": take(n * S, 3), "c": take(n * S, 3), "bl": take(n * S, self.nb)}
        if self.blend:
            w["c_pix"] = take(n * S, 3)
        if m:
            w.update(pts4=take(n * m, 4), odists=take(n, m), sigma=take(n * m, 1), rgb=take(n * m, 3), bg_alpha=take(n, SO),
                     bg_color=take(n, SO, 3))
        w["ctx"] = buf[off[0]:]
        assert w["ctx"].numel() >= self._ctx(n)
        return w


def blend_pixels_into(pts, proj, imgs, logits, n_rays, n_samples, c_pix):
    """nudf_blend_forward without patches (hom = NULL): pixel-blend colour c_pix [P,3] of every sample.  Pixel blending
    does not depend on the patch size, so this serves any h_patch_size."""
    lib = L.lib()
    V, _, H, W = imgs.shape
    cfg = L.BlendCfg(n_rays, n_samples, V, H, W, 0)
    L.check(lib.nudf_blend_forward(ctypes.byref(cfg), L.ptr(pts), L.ptr(proj), None, None, L.ptr(imgs), L.ptr(logits),
                                   logits.stride(0), L.ptr(c_pix), None, None, L.stream_ptr()), "nudf_blend_forward")


def ray_points_into(rays_o, rays_d, z_vals, sample_dist, pts, mid, dists):
    N, S = z_vals.shape
    L.check(L.lib().nudf_ray_points(L.ptr(rays_o), L.ptr(rays_d), L.ptr(z_vals), N, S, float(sample_dist), L.ptr(pts),
                                    L.ptr(mid), L.ptr(dists), L.stream_ptr()), "nudf_ray_points")


def outside_points_into(rays_o, rays_d, z, col0, sample_dist, pts4, dists):
    N, n = z.shape
    L.check(L.lib().nudf_outside_points(L.ptr(rays_o), L.ptr(rays_d), L.ptr(z), N, n, col0, float(sample_dist), L.ptr(pts4),
                                        L.ptr(dists), L.stream_ptr()), "nudf_outside_points")

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


def _refold(h, ps, extra, make_desc, size_fn, fold_fn):
    """The handles' shared bookkeeping.  h.wfold (folded weights and / or tensor-core weight images) is cached on
    (data_ptr, Tensor._version) of every parameter in ps plus `extra`; on a change it is resized to size_fn's float count
    and rebuilt by fold_fn from a fresh descriptor.  Returns that descriptor, or None when nothing changed."""
    key = tuple((p.data_ptr(), p._version) for p in ps) + extra
    if key == h._key:
        return None
    d = make_desc()
    n = size_fn(ctypes.byref(d))
    if n < 0:
        L.check(-1, size_fn.__name__)
    dev = ps[0].device
    if h.wfold is None or h.wfold.numel() != n or h.wfold.device != dev:
        h.wfold = torch.empty(n, dtype=torch.float32, device=dev)
    L.check(fold_fn(ctypes.byref(d), L.ptr(h.wfold), L.stream_ptr()), fold_fn.__name__)
    h._key = key
    return d


def _grad_targets(h, mods):
    """Where a backward pass writes the gradients of the weight-normed layers `mods` (in the order of the library's
    dbias): (sink, db, dg, dv, dbs).  With an armed gradient sink (dp.GradBucket) they are views of the data-parallel
    bucket, else fresh tensors; db is the ONE contiguous bias block the library writes, dbs its per-layer slices."""
    sink = h.grad_sink if (h.grad_sink is not None and h.grad_sink.begin()) else None
    if sink is not None:
        db = sink.block([m.bias for m in mods])
        return (sink, db, [sink.view(m.weight_g) for m in mods], [sink.view(m.weight_v) for m in mods],
                [sink.view(m.bias) for m in mods])
    nb = sum(int(m.bias.numel()) for m in mods)
    db = torch.empty(nb, dtype=torch.float32, device=mods[0].bias.device)
    dbs, off = [], 0
    for m in mods:
        n = m.bias.numel()
        dbs.append(db[off:off + n])
        off += n
    return None, db, [torch.empty_like(m.weight_g) for m in mods], [torch.empty_like(m.weight_v) for m in mods], dbs


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
        lib = L.lib()
        # the folded images depend on the engine and on which chains run fused (chain mask)
        d = _refold(self, ps, (lib.nudf_get_engine(), lib.nudf_get_tc_mask()), self._make_desc, lib.nudf_udf_folded_floats,
                    lib.nudf_udf_fold_weights)
        if d is not None:
            self.desc = d

    def _make_desc(self):
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
        return d


def _udf_ctx(handle, P, with_grad, dev):
    """the context buffer of a forward over P points (with_grad: also what the gradient and backward chains keep)"""
    n = L.lib().nudf_udf_ctx_floats(ctypes.byref(handle.desc), P, 1 if with_grad else 0)
    return torch.empty(max(n, 1), dtype=torch.float32, device=dev)


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
        buf = _udf_ctx(handle, P, with_grad, dev)
        if split:
            a = torch.empty(P, 1, dtype=torch.float32, device=dev)
            b = torch.empty(P, d_out - 1, dtype=torch.float32, device=dev)
            udf_forward_split_into(handle, pts, a, b, grad, buf)
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
        sink, db, dgs, dvs, dbs = _grad_targets(h, h.layers)
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
    work = _udf_ctx(handle, P, False, pts.device)
    L.check(lib.nudf_udf_value(ctypes.byref(handle.desc), L.ptr(handle.wfold), L.ptr(pts), P, L.ptr(udf), L.ptr(work),
                               L.stream_ptr()), "nudf_udf_value")
    return udf


def udf_value_gradient(handle, pts):
    """(udf [P], d udf/d x [P,3]) without autograd: one nudf_udf_forward_split with no feature output (the feature layer is
    skipped), the udf and gradient bits of udf_forward's"""
    handle.refresh()
    pts = _f32c(pts)
    _require_cuda(pts)
    P = pts.shape[0]
    udf = torch.empty(P, dtype=torch.float32, device=pts.device)
    grad = torch.empty(P, 3, dtype=torch.float32, device=pts.device)
    ctx = _udf_ctx(handle, P, True, pts.device)
    L.check(L.lib().nudf_udf_forward_split(ctypes.byref(handle.desc), L.ptr(handle.wfold), L.ptr(pts), P, L.ptr(udf), None, 0,
                                           L.ptr(grad), L.ptr(ctx), L.stream_ptr()), "nudf_udf_forward_split")
    return udf, grad


# ---------------------------------------------------------------------------------------------------------------
# colour network
# ---------------------------------------------------------------------------------------------------------------
class ColorHandle:
    def __init__(self, base_layers, main_layers, d_feature, d_hidden, d_out, n_blend, multires_view):
        self.base, self.main = base_layers, main_layers
        self.meta = (d_feature, d_hidden, d_out, n_blend, multires_view)
        self._key = None
        self._checked = None         # the parameter pointers whose shapes _check_shapes() accepted
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
        lib = L.lib()
        d = _refold(self, ps, (lib.nudf_get_engine(),), self._make_desc, lib.nudf_color_folded_floats, lib.nudf_color_fold_weights)
        if d is not None:
            self.desc = d

    def layer_shapes(self):
        """[(n_out, n_in)] of the base layers, then of the main layers, as nudf_color_fold_weights reads them"""
        F, H, d_out, n_blend, Lv = self.meta
        n_lin = len(self.base)
        d_view = 3 * (1 + 2 * Lv)
        out = lambda l, head: H if l < n_lin - 1 else head
        return ([(out(l, d_out), 3 + F if l == 0 else H) for l in range(n_lin)] +
                [(out(l, d_out + n_blend), d_view + d_out + H if l == 0 else H) for l in range(n_lin)])

    def _check_shapes(self):
        """every parameter has the shape nudf_color_fold_weights reads it with: any other would be folded with the wrong row
        length"""
        if len(self.main) != len(self.base):
            raise RuntimeError("colour network: %d main layers but %d base layers" % (len(self.main), len(self.base)))
        nb = len(self.base)
        for l, (m, (n_out, n_in)) in enumerate(zip(list(self.base) + list(self.main), self.layer_shapes())):
            if m.weight_v.shape != (n_out, n_in) or m.weight_g.shape != (n_out, 1) or m.bias.shape != (n_out,):
                raise RuntimeError("colour network %s: weight_v %s, weight_g %s, bias %s; the library plans [%d, %d]" % (
                    "lin_base%d" % l if l < nb else "lin%d" % (l - nb), tuple(m.weight_v.shape), tuple(m.weight_g.shape),
                    tuple(m.bias.shape), n_out, n_in))

    def _make_desc(self):
        mods = list(self.base) + list(self.main)
        ptrs = tuple(t.data_ptr() for m in mods for t in (m.weight_g, m.weight_v, m.bias))
        if ptrs != self._checked:                 # the shapes can only have changed with the tensors
            self._check_shapes()
            self._checked = ptrs
        d = L.ColorDesc()
        n = d.n_lin = len(self.base)
        d.d_feature, d.d_hidden, d.d_out, d.n_blend, d.multires_view = self.meta
        for l in range(n):
            d.base_g[l], d.base_v[l], d.base_b[l] = ptrs[3 * l:3 * l + 3]
            d.main_g[l], d.main_v[l], d.main_b[l] = ptrs[3 * (n + l):3 * (n + l) + 3]
        return d


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
        color_forward_into(handle, pts, dirs, samples_per_ray, feat, cb, c, bl, buf)
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
        nbase = len(h.base)             # bias layout in the library: base layers first, then main layers
        sink, db, dg, dv, dbs = _grad_targets(h, list(h.base) + list(h.main))
        L.check(lib.nudf_color_backward(ctypes.byref(h.desc), L.ptr(h.wfold), P, L.ptr(cb_bar), L.ptr(c_bar),
                                        L.ptr(bl_bar), L.ptr(buf), L.ptr(scratch), L.ptr(dfeat), d_feature, L.ptr(dw),
                                        L.ptr(db), L.stream_ptr()), "nudf_color_backward")
        L.check(lib.nudf_color_unfold_grads(ctypes.byref(h.desc), L.ptr(dw), _ptr_array(dg[:nbase]), _ptr_array(dv[:nbase]),
                                            _ptr_array(dg[nbase:]), _ptr_array(dv[nbase:]), L.stream_ptr()),
                "nudf_color_unfold_grads")
        if sink is not None:
            sink.ready()
        grads = []
        for l in list(range(nbase, len(dg))) + list(range(nbase)):     # params() order: main layers, then base layers
            grads += [dg[l], dv[l], dbs[l]]
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
        self._checked = None         # the parameter pointers whose shapes desc() accepted
        self.wfold = None            # NeRF++ has plain weights: the buffer holds the weight images only
        self.grad_sink = None

    def sink_layout(self):
        return [self.params()]

    def images(self):
        """bf16 hi/lo weight images for the tensor engine, rebuilt when a parameter changed (None on the fp32 engine, or
        when neither the NeRF++ backward (chain bit 64) nor the ReLU-network forward (bit 128) runs on the tensor cores)."""
        lib = L.lib()
        if lib.nudf_get_engine() != 1 or not (lib.nudf_get_tc_mask() & (64 | 128)):
            return None
        _refold(self, self.params(), (), self.desc, lib.nudf_nerf_image_floats, lib.nudf_nerf_prepare)
        return self.wfold

    def params(self):
        m = self.m
        ps = []
        for lin in m.pts_linears:
            ps += [lin.weight, lin.bias]
        for lin in (m.views_linears[0], m.feature_linear, m.alpha_linear, m.rgb_linear):
            ps += [lin.weight, lin.bias]
        return ps

    def layer_shapes(self):
        """[(module, (n_out, n_in))] of every layer, in params() order, as nudf_nerf_forward / _backward read the plain
        nn.Linear weights"""
        D, W, d_in, multires, multires_view, skip = self.meta
        ch, chv = d_in * (1 + 2 * multires), 3 * (1 + 2 * multires_view)
        m = self.m
        shapes = [(lin, (W, ch if i == 0 else (W + ch if i - 1 == skip else W))) for i, lin in enumerate(m.pts_linears)]
        return shapes + [(m.views_linears[0], (W // 2, W + chv)), (m.feature_linear, (W, W)), (m.alpha_linear, (1, W)),
                         (m.rgb_linear, (3, W // 2))]

    def desc(self):
        m = self.m
        ptrs = tuple(t.data_ptr() for t in self.params())
        if ptrs != self._checked:                 # the shapes can only have changed with the tensors
            if len(m.pts_linears) != self.meta[0]:
                raise RuntimeError("NeRF: %d pts_linears for D = %d" % (len(m.pts_linears), self.meta[0]))
            for lin, (n_out, n_in) in self.layer_shapes():
                if lin.weight.shape != (n_out, n_in) or lin.bias.shape != (n_out,):
                    raise RuntimeError("NeRF layer of weight %s / bias %s; the library plans [%d, %d]" % (
                        tuple(lin.weight.shape), tuple(lin.bias.shape), n_out, n_in))
            self._checked = ptrs
        d = L.NerfDesc()
        d.D, d.W, d.d_in, d.multires, d.multires_view, d.skip = self.meta
        D = len(m.pts_linears)
        for i in range(D):
            d.pts_w[i], d.pts_b[i] = ptrs[2 * i:2 * i + 2]
        d.views_w, d.views_b, d.feature_w, d.feature_b, d.alpha_w, d.alpha_b, d.rgb_w, d.rgb_b = ptrs[2 * D:]
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
        nerf_forward_into(d, wimg, pts, dirs, samples_per_ray, sigma, rgb, buf)
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
    rays_o, rays_d, z_vals = _f32c(rays_o), _f32c(rays_d), _f32c(z_vals)
    _require_cuda(rays_o, rays_d, z_vals)
    N, S = z_vals.shape
    dev = z_vals.device
    pts = torch.empty(N * S, 3, dtype=torch.float32, device=dev)
    mid = torch.empty(N, S, dtype=torch.float32, device=dev)
    dists = torch.empty(N, S, dtype=torch.float32, device=dev)
    ray_points_into(rays_o, rays_d, z_vals, sample_dist, pts, mid, dists)
    return pts, mid, dists


DIAG_KEYS = ["gradient_mag", "true_cos", "vis_prob", "alpha", "alpha_plus", "alpha_minus", "alpha_occ", "raw_occ",
             "inside_sphere"]


ALPHA_RULES = {"numerical": 0, "theorical": 1}   # sdf2alpha_type -> the kernels' alpha_rule


def alpha_rule(sdf2alpha_type):
    """The kernels' alpha_rule for an sdf2alpha_type string; ValueError for any other string."""
    if sdf2alpha_type not in ALPHA_RULES:
        raise ValueError("sdf2alpha_type %r: expected one of %s" % (sdf2alpha_type, sorted(ALPHA_RULES)))
    return ALPHA_RULES[sdf2alpha_type]


def _make_cfg(N, S, O, sample_dist, cos_anneal_ratio, flip_saturation, sparse_scale_factor, use_norm, background_rgb,
              alpha_rule=0):
    """The compositing kernels' nudf_render_cfg; alpha_rule: 0 numerical, 1 theorical."""
    if alpha_rule not in (0, 1):
        raise ValueError("alpha_rule must be 0 (numerical) or 1 (theorical), got %r" % (alpha_rule,))
    cfg = L.RenderCfg()
    cfg.alpha_rule = int(alpha_rule)
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


def _composite_udf(udf, N, S):
    """udf as the kernels read it: (a [P] tensor, P = N*S, element p at p * ld_udf; ld_udf).  Takes [P] (a strided column
    view too), [P, 1] or [N, S]; raises ValueError for any other shape."""
    P = N * S
    if udf.dtype != torch.float32:
        udf = udf.float()
    if tuple(udf.shape) == (N, S):
        udf = udf.reshape(P)                # a copy only when the rows are not evenly strided
    elif tuple(udf.shape) == (P, 1):
        udf = udf[:, 0]
    if tuple(udf.shape) != (P,):
        raise ValueError("composite: udf of shape %s; expected [%d], [%d, 1] or [%d, %d]" % (tuple(udf.shape), P, P, N, S))
    return udf, (udf.stride(0) if P > 1 else 1)


def _check_composite_rows(N, S, O, **ts):
    """Every per-sample tensor has N*S rows, the background ones N*(S+O), rays_d N; vectors are 3 wide.  Checked before
    any launch: the kernels index these by ray and sample with no bound of their own."""
    rows = {"rays_d": N, "bg_alpha": N * (S + O), "bg_color": N * (S + O), "heads": 1}
    width = {"grads": 3, "scb": 3, "sc": 3, "pts": 3, "rays_d": 3, "bg_color": 3, "heads": 3}
    for name, t in ts.items():
        if t is None:
            continue
        r, w = rows.get(name, N * S), width.get(name, 1)
        if t.numel() != r * w or (w > 1 and t.shape[-1] != w):
            raise ValueError("composite: %s of shape %s; expected %d rows%s (N = %d rays, S = %d samples, O = %d)" % (
                name, tuple(t.shape), r, " of %d" % w if w > 1 else "", N, S, O))


class _CompositeFunction(torch.autograd.Function):
    """differentiable inputs: udf [P] / [P,1] / [N,S], grads [P,3], scb [P,3], sc [P,3], bg_alpha [N,S+O],
    bg_color [N,S+O,3], heads [3]"""

    @staticmethod
    def forward(ctx, udf, grads, scb, sc, bg_alpha, bg_color, heads, geom, cfg, want_diag):
        N, S, O = cfg.n_rays, cfg.n_samples, cfg.n_outside
        udf_shape = udf.shape
        udf, ld_udf = _composite_udf(udf, N, S)
        geom = tuple(_f32c(t) for t in geom)
        rays_d, pts, mid, dists = geom
        _check_composite_rows(N, S, O, grads=grads, scb=scb, sc=sc, pts=pts, mid=mid, dists=dists, rays_d=rays_d,
                              heads=heads, bg_alpha=bg_alpha, bg_color=bg_color)
        lib = L.lib()
        dev = grads.device
        grads, scb, sc, heads = _f32c(grads), _f32c(scb), _f32c(sc), _f32c(heads)
        bg_alpha, bg_color = _f32c(bg_alpha), _f32c(bg_color)
        _require_cuda(udf, grads, scb, sc, heads, rays_d, pts, mid, dists, bg_alpha, bg_color)
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
        ctx.cfg, ctx.geom, ctx.ld_udf, ctx.udf_shape = cfg, geom, ld_udf, udf_shape
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
        L.check(lib.nudf_render_composite_backward(ctypes.byref(cfg), L.ptr(heads), L.ptr(rays_d), L.ptr(pts),
                                                   L.ptr(mid), L.ptr(dists), L.ptr(udf), ctx.ld_udf, L.ptr(grads),
                                                   L.ptr(scb), L.ptr(sc), L.ptr(bg_alpha), L.ptr(bg_color),
                                                   ctypes.byref(bar), L.ptr(udf_bar), L.ptr(grads_bar), L.ptr(scb_bar),
                                                   L.ptr(sc_bar), L.ptr(bga_bar), L.ptr(bgc_bar), L.ptr(scal), L.stream_ptr()),
                "nudf_render_composite_backward")
        # in the caller's shape: [P] (possibly a strided view), [P, 1] or [N, S]
        return (udf_bar.reshape(ctx.udf_shape), grads_bar, scb_bar, sc_bar, bga_bar, bgc_bar, scal.sum(dim=0),
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
        P = n_rays * n_samples
        V, _, H, W = imgs.shape
        cfg = L.BlendCfg(n_rays, n_samples, V, H, W, h_patch)
        logits = logits.contiguous()
        c_pix = torch.empty(P, 3, device=pts.device)
        npx = (2 * h_patch + 1) ** 2
        c_pat = torch.empty(P, npx, 3, device=pts.device) if hom is not None else None
        m_pat = torch.empty(P, device=pts.device) if hom is not None else None
        blend_forward_into(cfg, pts, proj, hom, px, imgs, logits, c_pix, c_pat, m_pat)
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


def up_sample(mode, rays_o, rays_d, z, udf, sample_dist, m, inv_s, beta, gamma, return_inds=False, alpha_rule=0):
    """One nudf_up_sample round.  mode 0 up_sample_unbias, 1 up_sample_no_occ_aware, 2 up_sample_unbias under the
    'theorical' alpha; alpha_rule=1 turns mode 0 into mode 2 (mode 1 has no alpha to choose)."""
    if mode == 0 and alpha_rule == 1:
        mode = 2
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
    rays_o, rays_d, z = _f32c(rays_o), _f32c(rays_d), _f32c(z)
    N, n = z.shape
    m = n - col0
    pts4 = torch.empty(N * m, 4, dtype=torch.float32, device=z.device)
    dists = torch.empty(N, m, dtype=torch.float32, device=z.device)
    outside_points_into(rays_o, rays_d, z, col0, sample_dist, pts4, dists)
    return pts4, dists


# ---------------------------------------------------------------------------------------------------------------
# The library calls that write into caller-owned tensors: the one call site of each entry point.  The allocating wrappers
# and autograd forwards above allocate and call these; the forward-only view renderer (render.render_view) passes views of
# its workspace.  A handle must have been refresh()ed by the caller (the autograd forwards need its descriptor earlier, to
# size the context buffer, and a forward refreshes once).
# ---------------------------------------------------------------------------------------------------------------
def udf_forward_split_into(handle, pts, udf, feat, grad, ctx):
    """nudf_udf_forward_split into given buffers: udf [P] or [P,1], feat [P, d_out - 1], grad [P,3] or None; ctx is the
    context buffer (scratch when there is no backward)."""
    L.check(L.lib().nudf_udf_forward_split(ctypes.byref(handle.desc), L.ptr(handle.wfold), L.ptr(pts), pts.shape[0], L.ptr(udf),
                                           L.ptr(feat), feat.shape[1], L.ptr(grad), L.ptr(ctx), L.stream_ptr()),
            "nudf_udf_forward_split")


def color_forward_into(handle, pts, dirs, samples_per_ray, feat, cb, c, bl, ctx):
    L.check(L.lib().nudf_color_forward(ctypes.byref(handle.desc), L.ptr(handle.wfold), L.ptr(pts), L.ptr(dirs),
                                       int(samples_per_ray), L.ptr(feat), feat.stride(0), pts.shape[0], L.ptr(cb), L.ptr(c),
                                       L.ptr(bl), L.ptr(ctx), L.stream_ptr()), "nudf_color_forward")


def nerf_forward_into(desc, wimg, pts, dirs, samples_per_ray, sigma, rgb, ctx):
    """desc, wimg: NerfHandle.desc() and .images() (None: exact-fp32 engine)"""
    L.check(L.lib().nudf_nerf_forward(ctypes.byref(desc), L.ptr(wimg), L.ptr(pts), L.ptr(dirs), int(samples_per_ray),
                                      pts.shape[0], L.ptr(sigma), L.ptr(rgb), L.ptr(ctx), L.stream_ptr()), "nudf_nerf_forward")


def view_composite(cfg, heads, rays_d, pts, mid, dists, udf, grads, sc, c_pix, bg_alpha, bg_color, rot, outs):
    """nudf_render_view_forward: outs maps color / color_pixel / depth / normal / weight_sum to [N, .] tensors (views
    into the image buffers are fine) or None; rot is a host 3x3 (nested sequence or array)."""
    lib = L.lib()
    ro = L.ViewOut()
    for k in L.VIEW_OUT_FIELDS:
        t = outs.get(k)
        setattr(ro, k, None if t is None else t.data_ptr())
    r9 = (ctypes.c_float * 9)(*[float(v) for row in rot for v in row])
    L.check(lib.nudf_render_view_forward(ctypes.byref(cfg), L.ptr(heads), L.ptr(rays_d), L.ptr(pts), L.ptr(mid),
                                         L.ptr(dists), L.ptr(udf), 1, L.ptr(grads), L.ptr(sc), L.ptr(c_pix),
                                         L.ptr(bg_alpha), L.ptr(bg_color), r9, ctypes.byref(ro), L.stream_ptr()),
            "nudf_render_view_forward")


def blend_forward_into(cfg, pts, proj, hom, px, imgs, logits, c_pix, c_pat, m_pat):
    """nudf_blend_forward; hom / px / c_pat / m_pat None = no patches"""
    L.check(L.lib().nudf_blend_forward(ctypes.byref(cfg), L.ptr(pts), L.ptr(proj), L.ptr(hom), L.ptr(px), L.ptr(imgs), L.ptr(logits),
                                       logits.stride(0), L.ptr(c_pix), L.ptr(c_pat), L.ptr(m_pat), L.stream_ptr()),
            "nudf_blend_forward")


def blend_pixels_into(pts, proj, imgs, logits, n_rays, n_samples, c_pix):
    """The pixel-blend colour c_pix [P,3] of every sample, without patches.  Pixel blending does not depend on the patch
    size, so this serves any h_patch_size."""
    V, _, H, W = imgs.shape
    blend_forward_into(L.BlendCfg(n_rays, n_samples, V, H, W, 0), pts, proj, None, None, imgs, logits, c_pix, None, None)


def ray_points_into(rays_o, rays_d, z_vals, sample_dist, pts, mid, dists):
    N, S = z_vals.shape
    L.check(L.lib().nudf_ray_points(L.ptr(rays_o), L.ptr(rays_d), L.ptr(z_vals), N, S, float(sample_dist), L.ptr(pts),
                                    L.ptr(mid), L.ptr(dists), L.stream_ptr()), "nudf_ray_points")


def outside_points_into(rays_o, rays_d, z, col0, sample_dist, pts4, dists):
    N, n = z.shape
    L.check(L.lib().nudf_outside_points(L.ptr(rays_o), L.ptr(rays_d), L.ptr(z), N, n, col0, float(sample_dist), L.ptr(pts4),
                                        L.ptr(dists), L.stream_ptr()), "nudf_outside_points")

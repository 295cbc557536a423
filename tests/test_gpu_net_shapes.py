"""GPU tests of the UDF, colour and NeRF++ networks away from the shipped shapes: a configuration sweep against fp64.

Every other network test builds the networks at the shapes of the shipped confs.  The planner behind all three networks
(DenseLayer, plan_images and tc_shape_ok in csrc/dense_layer.cuh / gemm_engine.cuh) has branches those shapes never take:
`scale` != 1, layers on both sides of the tensor-core threshold in one network, widths that are no multiple of 4 or 8, the
narrow-head forward kernel against a head that is too wide for it, multires 0 and 16, no skip or a skip on the first or last
layer, 16 layers per stack, and ragged or tiny point counts.  Each configuration below names the branch it is there for.

Every run goes through the real modules (models/fields.py) and is checked against the pinned oracle in fp64 (the arbiter)
with the oracle's own fp32 run as the noise yardstick (parity(), the 1e-4 bound of test_gpu_tc_chains): outputs and every
parameter gradient -- first and second order for the UDF, plus the feature gradient of the colour network.  On the tensor
engine the library's launch counts per kernel family show that the layers whose shape qualifies ran on the tensor cores and
that no other did: layer by layer for the UDF network, as "some" or "none" per family for the ReLU networks.  Forward outputs must not depend on the batch: rows 0..128 of a 4 099-point run equal a 129-point run bit
for bit (no forward contraction reduces over points, so a difference means a ragged tile touched its neighbours' rows)."""
import functools

import pytest
import torch

from neuraludf_b200 import _lib as L
from oracle import oracle_torch as O
from tests.gpu_util import err_inf, parity, report, scale_inf
from tests.test_gpu_chain import _points
from tests.test_gpu_tc_chains import _check_routing, _clear_gates, _grads, _LastWorkload, _run, _udf_loss

pytestmark = pytest.mark.gpu
DEV = "cuda"

# geometric init zeroes the positional-encoding columns of UDF layer 0 and of the skip layer; a perturbation this large
# gives them weight, so an error in the PE part of the skip concatenation is not hidden below the parity bound
UDF_NOISE = 2e-2

# (n_layers, d_hidden, skip_in, multires, d_out, scale); a skip layer's input layer is d_hidden - d_pe wide
UDF_CFGS = {
    "U1": (1, 64, (), 0, 2, 1.0),          # two layers, K = 3 first layer (no frequency bands), 1-wide feature record
    "U2": (3, 100, (1,), 4, 1, 2.5),       # skip at layer 1, no features, widths no multiple of 8, scale > 1
    "U3": (6, 200, (3,), 8, 65, 0.5),      # generic mid-size, scale < 1
    "U4": (8, 512, (4,), 6, 257, 1.0),     # N, K = 512: several column tiles and K slices
    "U5": (5, 33, (5,), 4, 17, 1.7),       # skip on the last layer (its input layer is 6 wide), feature record N = 16
    "U6": (4, 16, (), 16, 9, 3.0),         # multires 16 (99 PE columns), N = 16 / K = 16 layers, no skip
    "U7": (15, 64, (8,), 6, 33, 1.0),      # 16 layers, the most a plan holds
    "U8": (3, 31, (2,), 2, 257, 1.0),      # a hidden K of 31, just below the tensor-core threshold
}
# (n_layers, d_hidden, d_feature, d_out, blending views, multires_view); each stack has n_layers + 1 layers
COLOR_CFGS = {
    "C1": (2, 64, 32, 1, 0, 0),            # three layers per stack, one colour channel, no blending logits, no view PE
    "C2": (4, 256, 256, 3, 29, 6),         # main head of 32 outputs off the narrow-head kernel, wide layers
    "C3": (3, 100, 64, 4, 12, 2),          # main head N = 16 on the narrow-head kernel, 4 colour channels
    "C4": (15, 48, 16, 3, 10, 4),          # 16 layers per stack: a full fold-job table; base layer 0 below the threshold
    "C5": (4, 16, 13, 2, 5, 4),            # every layer at or below the threshold
}
# (D, W, skip or None, d_in, multires, multires_view)
NERF_CFGS = {
    "N1": (2, 64, None, 3, 0, 0),          # two layers, no skip, no PE at all
    "N2": (4, 100, 0, 4, 6, 2),            # skip after the first layer, W no multiple of 4
    "N3": (16, 32, 14, 4, 10, 4),          # 16 layers, the skip at D - 2 (into the last pts layer)
    "N4": (8, 512, 4, 4, 10, 4),           # W = 512
    "N5": (5, 33, 2, 4, 10, 4),            # odd W: W / 2 = 16
}

POINTS = (1, 129, 4099)
BIG = 65499                                # 511 * 128 + 91: a ragged last row tile, several point splits in the weight gradients
BIG_CFGS = ("U3", "U4", "C2", "N4")
SUBSETS = {"all": "ufg", "grad": "g", "uf": "uf"}
# fp32: the exact-fp32 FFMA engine; tc: the tensor engine with the library's default chain mask (and with every chain on,
# when that default is not 255); mN: the tensor engine with the single chain bit N
UDF_BITS = (1, 2, 4, 8, 16)
RELU_BITS = {"color": (16, 32, 128), "nerf": (16, 64, 128)}
BIT_CFGS = {"udf": ("U3", "U4", "U5"), "color": ("C2",), "nerf": ("N5",)}
BIT_P = 4099


def _modes(net, cfg):
    bits = UDF_BITS if net == "udf" else RELU_BITS[net]
    return ["fp32", "tc"] + (["m%d" % b for b in bits] if cfg in BIT_CFGS[net] else [])


def _sizes(cfg):
    return POINTS + ((BIG,) if cfg in BIG_CFGS else ())


UDF_CASES = [(c, P, sub, m) for c in UDF_CFGS for P in _sizes(c) for sub in SUBSETS
             for m in (_modes("udf", c) if P == BIT_P else ["fp32", "tc"])]
COLOR_CASES = [(c, P, m) for c in COLOR_CFGS for P in _sizes(c) for m in (_modes("color", c) if P == BIT_P else ["fp32", "tc"])]
NERF_CASES = [(c, P, m) for c in NERF_CFGS for P in _sizes(c) for m in (_modes("nerf", c) if P == BIT_P else ["fp32", "tc"])]


@pytest.fixture(scope="module", autouse=True)
def _engine():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = L.lib()
    old, old_mask, old_tf32 = lib.nudf_get_engine(), lib.nudf_get_tc_mask(), torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    lib.nudf_set_launch_timing(0)
    lib.nudf_set_engine(old)
    lib.nudf_set_tc_mask(old_mask)
    torch.backends.cuda.matmul.allow_tf32 = old_tf32


@pytest.fixture(scope="module")
def refs():
    return _LastWorkload()


# The weight-norm g gradient of a row is a projection, <dW_row, v_row> / |v_row|, and cancels: the last layer's, when only
# grad_x udf carries an upstream gradient (one non-zero entry, summed over every point and input column), shows an fp32
# oracle noise of 1.9e-5 of its value, 300 times fp32's unit roundoff.  The 2-plane bf16 split of the gradient chains (bits 2,
# 4, 8, 16, 32, 64) carries a unit roundoff of 2^-16, 2^8 times fp32's, so the same cancellation costs it up to 2^8 times the
# oracle's noise; measured on an H100 80GB HBM3 (700 W): 12x (U3, rel 2.2e-4) and 22x (U4, rel 1.1e-4).  Those g
# gradients are held to 64x the oracle's noise; every other tensor, and every g gradient whose noise is small, to 1e-4.
TWO_PLANE_CHAINS = 2 | 4 | 8 | 16 | 32 | 64
TWO_PLANE_G_NOISE = 64.0


def _runs(mode, fn):
    """[(tag, tensors, {family: launches}, engine, mask)] of fn() in `mode` (see the modes above)"""
    lib = L.lib()
    if mode == "fp32":
        lib.nudf_set_engine(0)
        return [("fp32",) + _run(0, fn) + (0, 0)]
    lib.nudf_set_engine(1)
    masks = sorted({lib.nudf_default_tc_mask(), 255}) if mode == "tc" else [int(mode[1:])]
    return [("tc.m%d" % m,) + _run(m, fn) + (1, m) for m in masks]


def _check(tag, new, ref64, ref32, mask):
    """every tensor of `new` within the parity bound of the fp64 oracle; every failure is reported before the test fails"""
    failures = []
    for k in new:
        assert new[k].shape == ref64[k].shape, "%s.%s: shape %s, oracle %s" % (tag, k, tuple(new[k].shape), tuple(ref64[k].shape))
        if new[k].numel() == 0:
            continue
        mult = TWO_PLANE_G_NOISE if (mask & TWO_PLANE_CHAINS and k.endswith(".weight_g")) else 2.0
        try:
            parity("%s.%s" % (tag, k), new[k], ref64[k], ref32[k], tol=1e-4, noise_mult=mult)
        except AssertionError as e:
            failures.append(str(e))
    assert not failures, "\n".join(failures)


# ---------------------------------------------------------------------------------------------------------------
# routing: which layers launch on the tensor cores, from the layer shapes alone
# ---------------------------------------------------------------------------------------------------------------
def tc_shape_ok(N, K):
    """csrc/gemm_engine.cuh: the operand shapes B(N, K) of X W^T (N = out, K = in) and dY W (N = in, K = out) that the
    weights-resident tensor-core kernel takes; any other launch runs on the FFMA kernel"""
    return K >= 32 and N >= 16


def tn_ok(M, N, P):
    """gemm_tn's condition for the tensor-core weight gradient dW [M, N] over P points"""
    return M >= 32 and N >= 32 and P >= 128


def _udf_routing(mask, cfg, sub, P):
    """launches per tensor-core family of one value_feature_gradient + backward (udf_net.cu), layer by layer"""
    layers = cfg["layers"]                                    # (n_in, n_out) of each layer
    hidden, (k_last, _) = layers[:-1], layers[-1]
    d_out, F = cfg["d_out"], cfg["d_out"] - 1
    has_out, has_grad = ("u" in sub or "f" in sub), "g" in sub
    split = has_out and bool(mask & 8) and 64 <= F <= 256 and F % 4 == 0      # the feature rows as their own backward operand
    want = {}
    if mask & 1:     # value chain: the hidden layers, and the feature rows of the last layer (the udf row stays on FFMA)
        want["tc_layer_other"] = sum(tc_shape_ok(n, k) for k, n in hidden) + (F > 0 and tc_shape_ok(F, k_last))
    if mask & 2:     # reverse sweep: dY W of every hidden layer
        want["tc_layer_reverse_sweep"] = sum(tc_shape_ok(k, n) for k, n in hidden)
    if mask & 4:     # tangent chain: X W^T of every hidden layer, only with an upstream gradient of grad_x udf
        want["tc_layer_tangent"] = sum(tc_shape_ok(n, k) for k, n in hidden) if has_grad else 0
    if mask & 8:     # backward chain: the last layer (or its feature rows) with a udf / feature upstream, then layers n_lin-2 .. 1
        top = (tc_shape_ok(k_last, F) if split else tc_shape_ok(k_last, d_out)) if has_out else 0
        want["tc_layer_backward"] = top + sum(tc_shape_ok(k, n) for k, n in hidden[1:])
    if mask & 16:    # weight gradients: every hidden layer for the tangent and for the backward chain, plus the last layer
        n = sum(tn_ok(n, k, P) for k, n in hidden) * (2 if has_grad else 1)
        want["tc_weight_gradient"] = n + (tn_ok(F if split else d_out, k_last, P) if has_out else 0)
    return want


def _some(want, fam, on):
    if on:
        want[fam] = None


def _relu_routing(layers, bwd_layers, P, narrow=lambda k, n: False):
    """colour / NeRF++: 'some' or 'none' per family.  layers: (n_in, n_out) of every layer; bwd_layers: those whose dY W
    the backward pass launches; narrow: the forward layers that run on the narrow-head kernel instead of a layer GEMM"""
    fwd = any(tc_shape_ok(n, k) and not narrow(k, n) for k, n in layers)
    bwd = any(tc_shape_ok(k, n) for k, n in bwd_layers)
    wg = any(n > 16 and tn_ok(n, k, P) for k, n in layers)    # n_out <= 16: the narrow weight-gradient kernel
    return fwd, bwd, wg


def _color_routing(mask, cc, P):
    H, F, d_out, nb = cc["d_hidden"], cc["d_feature"], cc["d_out"], cc["blending_cand_views"]
    n_lin = cc["n_layers"] + 1
    base = [(3 + F, H)] + [(H, H)] * (n_lin - 2) + [(H, d_out)]
    main = [(cc["d_view"] + d_out + H, H)] + [(H, H)] * (n_lin - 2) + [(H, d_out + nb)]
    fwd, bwd, wg = _relu_routing(base + main, main + base, P, narrow=lambda k, n: n <= 16 and k <= 128)
    want = {}
    _some(want, "tc_layer_other", (mask & 128 and fwd) or (mask & 32 and bwd))
    _some(want, "tc_weight_gradient", mask & 16 and wg)
    return want


def _nerf_layers(nc):
    W, ch, chv, skip = nc["W"], nc["input_ch"], nc["input_ch_view"], (nc["skips"] or (None,))[0]
    pts = [(ch, W)] + [(W + ch if i - 1 == skip else W, W) for i in range(1, nc["D"])]
    return pts, [(W + chv, W // 2), (W, W), (W, 1), (W // 2, 3)]       # views, feature, alpha, rgb


def _nerf_routing(mask, nc, P):
    pts, heads = _nerf_layers(nc)
    fwd, bwd, wg = _relu_routing(pts + heads, pts[1:] + heads, P)
    want = {}
    _some(want, "tc_layer_other", (mask & 128 and fwd) or (mask & 64 and bwd))
    _some(want, "tc_weight_gradient", mask & 16 and wg)
    return want


# ---------------------------------------------------------------------------------------------------------------
# UDF network
# ---------------------------------------------------------------------------------------------------------------
def _udf_cfg(name):
    n_layers, d_hidden, skip_in, multires, d_out, scale = UDF_CFGS[name]
    return O.udf_cfg(d_out=d_out, d_hidden=d_hidden, n_layers=n_layers, skip_in=skip_in, multires=multires, scale=scale)


@functools.lru_cache(maxsize=None)
def _udf_params(name):
    cfg = _udf_cfg(name)
    return cfg, O.make_udf_params(cfg, seed=100 + int(name[1:]), noise=UDF_NOISE)


@functools.lru_cache(maxsize=None)
def _udf_scene(name):
    """(cfg, parameters, point pool): the pool holds the points of every run of this config, the P-point run takes its
    first P.  Points where |udf| < 1e-5 are dropped: there sign(y0), and with it grad_x udf, is fp32 rounding noise."""
    cfg, params = _udf_params(name)
    n = max(_sizes(name))
    # on a 2^-20 grid, x * scale is exact in fp32 for every scale of the sweep but 1.7: the fp32 runs then see the inputs of
    # the fp64 oracle, where sin(2^15 x scale) (multires 16) would otherwise turn the input's rounding into a noise of 4e-3
    x = (torch.round(_points(n + n // 4 + 64, 200 + int(name[1:])) * 2 ** 20) / 2 ** 20).float()
    p64 = {k: v.double().to(DEV) for k, v in params.items()}
    with torch.no_grad():
        u64 = O.udf_mlp(p64, cfg, x.double().to(DEV))[:, 0].cpu()
    x = x[u64 >= 1e-5]
    assert x.shape[0] >= n
    return cfg, params, x[:n]


def _udf_module(cfg, params):
    from neuraludf_b200.models import fields as F
    udf = F.UDFNetwork(d_in=3, d_out=cfg["d_out"], d_hidden=cfg["d_hidden"], n_layers=cfg["n_layers"], skip_in=cfg["skip_in"],
                       multires=cfg["multires"], scale=cfg["scale"], bias=cfg["bias"], geometric_init=True, weight_norm=True,
                       udf_type="abs")
    udf.load_state_dict(params)
    return udf.to(DEV)


def _udf_module_run(udf, x, bars, sub):
    for p in udf.parameters():
        p.grad = None
    u, f, grad = udf.value_feature_gradient(x)
    _udf_loss(u, f, grad, bars, sub).backward()
    out = {"udf": u.detach(), "feature": f.detach(), "grad": grad.detach()}
    out.update({"d." + k: (torch.zeros_like(p) if p.grad is None else p.grad.clone()) for k, p in udf.named_parameters()})
    return out


def _udf_oracle(params, cfg, x, bars, sub, dt):
    p = {k: v.to(DEV, dt, copy=True).requires_grad_(True) for k, v in params.items()}
    xg = x.to(DEV, dt).requires_grad_(True)
    out = O.udf_mlp(p, cfg, xg)
    u, f = out[:, :1], out[:, 1:]
    grad = torch.autograd.grad(u, xg, torch.ones_like(u), create_graph=True)[0]
    loss = _udf_loss(u, f, grad, {k: v.to(DEV, dt) for k, v in bars.items()}, sub)
    res = {"udf": u.detach(), "feature": f.detach(), "grad": grad.detach()}
    res.update(_grads(loss, list(p.values()), list(p.keys())))
    return res


def _udf_workload(name, P, sub):
    cfg, params, pool = _udf_scene(name)
    x = pool[:P]
    gen = torch.Generator().manual_seed(7 + P)
    bars = {"u": torch.randn(P, 1, generator=gen), "f": torch.randn(P, cfg["d_out"] - 1, generator=gen),
            "g": torch.randn(P, 3, generator=gen)}
    return dict(udf=_udf_module(cfg, params), cfg=cfg, x=x.to(DEV), bars={k: v.to(DEV) for k, v in bars.items()},
                ref64=_udf_oracle(params, cfg, x.double(), bars, SUBSETS[sub], torch.float64),
                ref32=_udf_oracle(params, cfg, x, bars, SUBSETS[sub], torch.float32))


@pytest.mark.parametrize("name", [c for c in UDF_CFGS if UDF_CFGS[c][3] > 0])
def test_udf_pe_columns_carry_weight(name):
    """the perturbation gives the PE columns that geometric init zeroes (layer 0, the skip layer) real weight"""
    cfg, params = _udf_params(name)
    last = len(cfg["layers"]) - 1
    cols = {0: params["lin0.weight_v"][:, 3:]}
    for s in cfg["skip_in"]:
        if s != last:                                   # the last layer's init does not zero its PE columns
            cols[s] = params["lin%d.weight_v" % s][:, -(cfg["d_pe"] - 3):]
    for l, w in cols.items():
        assert float(w.abs().mean()) > 0.5 * UDF_NOISE, "lin%d: PE columns of mean |w| %.2e" % (l, float(w.abs().mean()))


@pytest.mark.parametrize("name,P,sub,mode", UDF_CASES)
def test_udf_shape(refs, name, P, sub, mode):
    w = refs.get(("udf", name, P, sub), lambda: _udf_workload(name, P, sub))
    for tag, new, counts, engine, mask in _runs(mode, lambda: _udf_module_run(w["udf"], w["x"], w["bars"], SUBSETS[sub])):
        tag = "net_shapes.%s.P%d.%s.%s" % (name, P, sub, tag)
        _check_routing(tag, counts, _udf_routing(mask, w["cfg"], SUBSETS[sub], P) if engine == 1 else {})
        _check(tag, new, w["ref64"], w["ref32"], mask)


# ---------------------------------------------------------------------------------------------------------------
# colour network
# ---------------------------------------------------------------------------------------------------------------
def _color_cfg(name):
    n_layers, d_hidden, d_feature, d_out, views, mv = COLOR_CFGS[name]
    return O.color_cfg(d_feature=d_feature, d_out=d_out, d_hidden=d_hidden, n_layers=n_layers, multires_view=mv,
                       blending_cand_views=views)


def _color_module(cc, params):
    from neuraludf_b200.models import fields as F
    col = F.ResidualRenderingNetwork(d_feature=cc["d_feature"], mode="no_normal", d_in=6, d_out=cc["d_out"],
                                     d_hidden=cc["d_hidden"], n_layers=cc["n_layers"], weight_norm=True,
                                     multires_view=cc["multires_view"], squeeze_out=True,
                                     blending_cand_views=cc["blending_cand_views"])
    col.load_state_dict(params)
    return col.to(DEV)


@functools.lru_cache(maxsize=None)
def _color_params(name):
    cc = _color_cfg(name)
    return cc, O.make_color_params(cc, seed=300 + int(name[1:]))


@functools.lru_cache(maxsize=None)
def _color_scene(name):
    """(cfg, parameters, (pts, dirs, feat) pool) with every ReLU of the fp64 oracle clear of zero (_clear_gates)"""
    cc, params = _color_params(name)
    n = max(_sizes(name))
    gen = torch.Generator().manual_seed(400 + int(name[1:]))
    m = 2 * n + 64
    pts = torch.rand(m, 3, generator=gen) * 2 - 1
    dirs = torch.randn(m, 3, generator=gen)
    dirs = dirs / dirs.norm(dim=1, keepdim=True)
    feat = 0.3 * torch.randn(m, cc["d_feature"], generator=gen)
    p64 = {k: v.double().to(DEV) for k, v in params.items()}
    return cc, params, _clear_gates(n, (pts, dirs, feat), lambda *t: O.color_mlp(p64, cc, *t))


def _color_module_run(col, pts, dirs, feat, bars):
    for p in col.parameters():
        p.grad = None
    featg = feat.clone().requires_grad_(True)
    o = col(pts, None, dirs, featg)
    if len(o) == 2:                                   # no blending views: the module returns (color_base, color)
        o = (o[0], o[1], torch.empty(o[0].shape[0], 0, device=DEV))
    sum((t * b).sum() for t, b in zip(o, bars) if t.numel()).backward()
    out = {"color_base": o[0].detach(), "color": o[1].detach(), "blend": o[2].detach(), "dfeat": featg.grad}
    out.update({"d." + k: p.grad.clone() for k, p in col.named_parameters()})
    return out


def _color_oracle(params, cc, pts, dirs, feat, bars, dt):
    p = {k: v.to(DEV, dt, copy=True).requires_grad_(True) for k, v in params.items()}
    f = feat.to(DEV, dt).requires_grad_(True)
    o = O.color_mlp(p, cc, pts.to(DEV, dt), dirs.to(DEV, dt), f)
    loss = sum((t * b.to(DEV, dt)).sum() for t, b in zip(o, bars))
    res = {"color_base": o[0].detach(), "color": o[1].detach(), "blend": o[2].detach()}
    gr = _grads(loss, list(p.values()) + [f], list(p.keys()) + ["feat"])
    res["dfeat"] = gr.pop("d.feat")
    res.update(gr)
    return res


def _color_workload(name, P):
    cc, params, pool = _color_scene(name)
    pts, dirs, feat = (t[:P] for t in pool)
    gen = torch.Generator().manual_seed(41 + P)
    bars = [torch.randn(P, k, generator=gen) for k in (cc["d_out"], cc["d_out"], cc["blending_cand_views"])]
    return dict(col=_color_module(cc, params), cc=cc, dev=[t.to(DEV) for t in (pts, dirs, feat)],
                bars=[b.to(DEV) for b in bars],
                ref64=_color_oracle(params, cc, pts.double(), dirs.double(), feat.double(), [b.double() for b in bars],
                                    torch.float64),
                ref32=_color_oracle(params, cc, pts, dirs, feat, bars, torch.float32))


@pytest.mark.parametrize("name,P,mode", COLOR_CASES)
def test_color_shape(refs, name, P, mode):
    w = refs.get(("color", name, P), lambda: _color_workload(name, P))
    for tag, new, counts, engine, mask in _runs(mode, lambda: _color_module_run(w["col"], *w["dev"], w["bars"])):
        tag = "net_shapes.%s.P%d.%s" % (name, P, tag)
        _check_routing(tag, counts, _color_routing(mask, w["cc"], P) if engine == 1 else {})
        _check(tag, new, w["ref64"], w["ref32"], mask)


# ---------------------------------------------------------------------------------------------------------------
# NeRF++ background network
# ---------------------------------------------------------------------------------------------------------------
def _nerf_cfg(name):
    D, W, skip, d_in, multires, mv = NERF_CFGS[name]
    return O.nerf_cfg(D=D, W=W, d_in=d_in, multires=multires, multires_view=mv, skips=() if skip is None else (skip,))


def _nerf_module(nc, params):
    from neuraludf_b200.models import fields as F
    nerf = F.NeRF(D=nc["D"], W=nc["W"], d_in=nc["d_in"], d_in_view=3, multires=nc["multires"],
                  multires_view=nc["multires_view"], output_ch=4, skips=list(nc["skips"]), use_viewdirs=True)
    nerf.load_state_dict(params)
    return nerf.to(DEV)


@functools.lru_cache(maxsize=None)
def _nerf_params(name):
    nc = _nerf_cfg(name)
    return nc, O.make_nerf_params(nc, seed=500 + int(name[1:]))


@functools.lru_cache(maxsize=None)
def _nerf_scene(name):
    nc, params = _nerf_params(name)
    n = max(_sizes(name))
    gen = torch.Generator().manual_seed(600 + int(name[1:]))
    m = 2 * n + 64
    pts = torch.randn(m, 4, generator=gen, dtype=torch.float64)
    pts = (pts / pts[:, :3].norm(dim=1, keepdim=True)).float()[:, :nc["d_in"]].contiguous()
    dirs = torch.randn(m, 3, generator=gen)
    dirs = dirs / dirs.norm(dim=1, keepdim=True)
    p64 = {k: v.double().to(DEV) for k, v in params.items()}
    return nc, params, _clear_gates(n, (pts, dirs), lambda *t: O.nerf_mlp(p64, nc, *t))


def _nerf_module_run(nerf, pts, dirs, bars):
    for p in nerf.parameters():
        p.grad = None
    a, rgb = nerf(pts, dirs)
    ((a * bars[0]).sum() + (rgb * bars[1]).sum()).backward()
    out = {"alpha": a.detach(), "rgb": rgb.detach()}
    out.update({"d." + k: p.grad.clone() for k, p in nerf.named_parameters()})
    return out


def _nerf_oracle(params, nc, pts, dirs, bars, dt):
    p = {k: v.to(DEV, dt, copy=True).requires_grad_(True) for k, v in params.items()}
    a, rgb = O.nerf_mlp(p, nc, pts.to(DEV, dt), dirs.to(DEV, dt))
    loss = (a * bars[0].to(DEV, dt)).sum() + (rgb * bars[1].to(DEV, dt)).sum()
    res = {"alpha": a.detach(), "rgb": rgb.detach()}
    res.update(_grads(loss, list(p.values()), list(p.keys())))
    return res


def _nerf_workload(name, P):
    nc, params, pool = _nerf_scene(name)
    pts, dirs = (t[:P] for t in pool)
    gen = torch.Generator().manual_seed(43 + P)
    bars = [torch.randn(P, 1, generator=gen), torch.randn(P, 3, generator=gen)]
    return dict(nerf=_nerf_module(nc, params), nc=nc, dev=[pts.to(DEV), dirs.to(DEV)], bars=[b.to(DEV) for b in bars],
                ref64=_nerf_oracle(params, nc, pts.double(), dirs.double(), [b.double() for b in bars], torch.float64),
                ref32=_nerf_oracle(params, nc, pts, dirs, bars, torch.float32))


@pytest.mark.parametrize("name,P,mode", NERF_CASES)
def test_nerf_shape(refs, name, P, mode):
    w = refs.get(("nerf", name, P), lambda: _nerf_workload(name, P))
    for tag, new, counts, engine, mask in _runs(mode, lambda: _nerf_module_run(w["nerf"], *w["dev"], w["bars"])):
        tag = "net_shapes.%s.P%d.%s" % (name, P, tag)
        _check_routing(tag, counts, _nerf_routing(mask, w["nc"], P) if engine == 1 else {})
        _check(tag, new, w["ref64"], w["ref32"], mask)


# ---------------------------------------------------------------------------------------------------------------
# batch independence of the forward passes
# ---------------------------------------------------------------------------------------------------------------
def _forward(name, P):
    """the forward outputs of config `name` on the first P points of its pool"""
    if name.startswith("U"):
        cfg, params, pool = _udf_scene(name)
        with torch.no_grad():
            return _udf_module(cfg, params).value_feature_gradient(pool[:P].to(DEV))
    if name.startswith("C"):
        cc, params, pool = _color_scene(name)
        pts, dirs, feat = (t[:P].to(DEV) for t in pool)
        with torch.no_grad():
            return _color_module(cc, params)(pts, None, dirs, feat)
    nc, params, pool = _nerf_scene(name)
    with torch.no_grad():
        return _nerf_module(nc, params)(*(t[:P].to(DEV) for t in pool))


@pytest.mark.parametrize("mode", ["fp32", "tc"])
@pytest.mark.parametrize("name", list(UDF_CFGS) + list(COLOR_CFGS) + list(NERF_CFGS))
def test_forward_batch_independent(name, mode):
    lib = L.lib()
    lib.nudf_set_engine(0 if mode == "fp32" else 1)
    lib.nudf_set_tc_mask(lib.nudf_default_tc_mask())
    small, big = _forward(name, 129), _forward(name, 4099)
    for i, (s, b) in enumerate(zip(small, big)):
        assert torch.equal(s, b[:129]), "%s %s: output %d of rows 0..128 changes with the batch (max diff %.3e)" % (
            name, mode, i, err_inf(s, b[:129]) if s.numel() else 0.0)


# ---------------------------------------------------------------------------------------------------------------
# end to end: a 64-wide feature record through the colour network and compositing
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["fp32", "tc"])
def test_render_core_feature_width(mode):
    """render_core forward + backward with U3 (scale 0.5, 64 features) feeding a colour network with d_feature = 64, 64 rays x
    64 samples, against the oracle in fp64 and fp32 on the host with test_c2_full_size_vs_oracle's bounds"""
    from neuraludf_b200.models import fields as F
    from neuraludf_b200.models.udf_renderer_blending import UDFRendererBlending
    lib = L.lib()
    lib.nudf_set_engine(0 if mode == "fp32" else 1)
    lib.nudf_set_tc_mask(lib.nudf_default_tc_mask())
    udf_c, udf_p = _udf_params("U3")
    col_c = O.color_cfg(d_feature=udf_c["d_out"] - 1)
    col_p = O.make_color_params(col_c, seed=1)
    sc = O.make_scalars()
    udf, col = _udf_module(udf_c, udf_p), _color_module(col_c, col_p)
    var = F.SingleVarianceNetwork(init_val=float(sc["variance"])).to(DEV)
    beta = F.BetaNetwork(init_var_beta=float(sc["beta"]), init_var_gamma=float(sc["gamma"]), init_var_zeta=float(sc["zeta"]),
                         beta_min=5e-5, requires_grad_beta=True, requires_grad_gamma=False, requires_grad_zeta=False).to(DEV)
    ren = UDFRendererBlending(None, udf, var, col, beta, n_samples=64, n_importance=0, n_outside=0, up_sample_steps=1,
                              perturb=0.0)
    o, d, near, far = O.make_rays(64, seed=5)
    S = 64
    z = (near + (far - near) * torch.linspace(0.0, 1.0, S)[None, :]).contiguous()
    sd = ((far - near) / S).mean().item()
    refs = {}
    for dt in (torch.float64, torch.float32):
        up, cp, scd = ({k: v.to(dt, copy=True).requires_grad_(True) for k, v in ps.items()} for ps in (udf_p, col_p, sc))
        r = O.render_core(up, udf_c, cp, col_c, scd, o.to(dt), d.to(dt), z.to(dt), sd, cos_anneal_ratio=0.5)
        loss = O.training_loss(r, torch.full((64, 3), 0.4, dtype=dt))
        names = ["udf." + k for k in up] + ["color." + k for k in cp] + ["var.variance", "beta.beta"]
        gr = torch.autograd.grad(loss, list(up.values()) + list(cp.values()) + [scd["variance"], scd["beta"]])
        refs[dt] = ({k: v.detach() for k, v in r.items() if isinstance(v, torch.Tensor)}, loss.detach(), dict(zip(names, gr)))
    (r64, l64, g64), (r32, l32, g32) = refs[torch.float64], refs[torch.float32]
    ret = ren.render_core(o.to(DEV), d.to(DEV), z.to(DEV), sd, udf, var, col, beta_network=beta, cos_anneal_ratio=0.5)
    tag = "net_shapes.render_core.U3_F64.%s" % mode
    for k in ("udf", "gradients", "color", "color_base", "depth", "weights", "normals", "gradient_error", "sparse_error",
              "alpha", "vis_prob"):
        parity("%s.%s" % (tag, k), ret[k].reshape(r64[k].shape), r64[k], r32[k],
               tol=1e-4 if k in ("udf", "gradients") else 2e-4, noise_mult=4.0 if k == "sparse_error" else 2.0)
    loss = O.training_loss(ret, torch.full((64, 3), 0.4, device=DEV))
    parity(tag + ".loss", loss.detach(), l64, l32, tol=2e-4)
    loss.backward()
    n = 0
    for mn, m in (("udf", udf), ("color", col), ("var", var), ("beta", beta)):
        for pn, p in m.named_parameters():
            key = mn + "." + pn
            if key not in g64:
                continue
            e = err_inf(p.grad, g64[key]) / scale_inf(g64[key])
            noise = err_inf(g32[key], g64[key]) / scale_inf(g64[key])
            report("%s.dparam.%s" % (tag, key), rel=e, ref_noise_rel=noise)
            assert e <= max(5e-3, 3.0 * noise), (key, e, noise)
            n += 1
    assert n == 3 * (len(udf_c["layers"]) + 2 * (col_c["n_layers"] + 1)) + 2

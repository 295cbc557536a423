"""GPU tests of each tensor-core chain on its own, at training-size ragged point counts.

One bit of the chain mask (TcChain, csrc/gemm_engine.cuh) moves one chain of the UDF, colour or NeRF++ network onto the
tensor-core layer kernels (csrc/gemm_tc.cuh); every other contraction stays on the exact-fp32 FFMA kernel.  Each run is
checked three ways:
- routing: the library's launch counts per kernel family (nudf_read_launch_timing) show that the chain ran on the tensor
  cores, layer by layer where the count follows from the network's shape, and that no other tensor-core family launched;
- reach: every tensor the chain cannot affect has the bits of the mask-0 run (every contraction on FFMA, same folded
  weights), which also catches a kernel that writes into a context buffer it does not own;
- accuracy: every tensor the chain does reach, parameter gradients included, is within the parity bound of the pinned
  oracle in fp64 (the oracle's own fp32 run is the noise yardstick); its distance from the mask-0 run is reported.
The mask-0 run and both oracle runs are computed once per workload."""
import ctypes

import pytest
import torch

from neuraludf_b200 import _lib as L
from oracle import oracle_torch as O
from tests.gpu_util import build_modules, err_inf, oracle_params, parity, report, scale_inf
from tests.test_gpu_chain import _points

pytestmark = pytest.mark.gpu
DEV = "cuda"

FAM = {name: i for i, name in enumerate(L.LAUNCH_FAMILIES)}
TC_FAMILIES = ("tc_layer_reverse_sweep", "tc_layer_tangent", "tc_layer_backward", "tc_layer_other", "tc_weight_gradient")

# 65 499 = 511 * 128 + 91: a ragged last row tile and several point splits in the weight gradients; 129: one full row tile
# plus one row, and a single split
UDF_POINTS = (65499, 1000, 129)
BIG = 65499
# upstream gradients on (u)df, (f)eature, (g)rad_x udf: an unused output reaches the kernels as a null pointer
SUBSETS = {"all": "ufg", "grad": "g", "uf": "uf"}
UDF_CASES = [(name, P, sub, mask) for name in ("udf", "udf_small") for P in UDF_POINTS for sub in SUBSETS
             for mask in (1, 2, 4, 8, 16, 255)]
COLOR_MASKS = (16, 32, 128, 255)
NERF_MASKS = (16, 64, 128, 64 | 128, 255)


@pytest.fixture(scope="module", autouse=True)
def _engine():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = L.lib()
    old, old_mask, old_tf32 = lib.nudf_get_engine(), lib.nudf_get_tc_mask(), torch.backends.cuda.matmul.allow_tf32
    lib.nudf_set_engine(1)
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    lib.nudf_set_launch_timing(0)
    lib.nudf_set_engine(old)
    lib.nudf_set_tc_mask(old_mask)
    torch.backends.cuda.matmul.allow_tf32 = old_tf32


class _LastWorkload:
    """The references of the workload the previous test used (the tests of one workload are consecutive)."""

    def __init__(self):
        self.key, self.val = None, None

    def get(self, key, make):
        if key != self.key:
            self.key, self.val = None, None
            torch.cuda.empty_cache()
            self.val = make()
            self.key = key
        return self.val


@pytest.fixture(scope="module")
def refs():
    return _LastWorkload()


def _run(mask, fn):
    """fn() with chain mask `mask` and the library's launch timing on: (fn's tensors, {family: launches})"""
    lib = L.lib()
    lib.nudf_set_tc_mask(mask)
    lib.nudf_set_launch_timing(1)
    try:
        out = fn()
        nf = lib.nudf_launch_family_count()
        ms, cnt = (ctypes.c_float * nf)(), (ctypes.c_int32 * nf)()
        L.check(lib.nudf_read_launch_timing(ms, cnt), "nudf_read_launch_timing")
    finally:
        lib.nudf_set_launch_timing(0)
    return out, {name: cnt[FAM[name]] for name in TC_FAMILIES}


def _check_routing(tag, counts, want):
    """want: {family: exact count, or None for 'at least one'}; every other tensor-core family launches nothing"""
    for fam in TC_FAMILIES:
        if fam not in want:
            assert counts[fam] == 0, "%s: %d launches of %s, which this mask does not select" % (tag, counts[fam], fam)
        elif want[fam] is None:
            assert counts[fam] > 0, "%s: the selected chain did not launch %s (fell back to FFMA)" % (tag, fam)
        else:
            assert counts[fam] == want[fam], "%s: %d launches of %s, expected %d" % (tag, counts[fam], fam, want[fam])


def _check_run(tag, new, base, ref64, ref32, reach):
    """reach: the tensors the mask can change; the others must keep the mask-0 run's bits.  One bound for every chain,
    the ReLU networks' forward (bit 128) included: on points whose ReLU gates are clear of rounding (_clear_gates) no
    gate flips between runs, and their worst error measured on an H100 80GB HBM3 (700 W) is 1.8e-5 of max."""
    failures = []                     # every tensor is checked and reported before the test fails
    for k in new:
        name = "%s.%s" % (tag, k)
        if k not in reach:
            if not torch.equal(new[k], base[k]):
                failures.append("%s: changed by a chain that cannot reach it (max diff %.3e)" % (
                    name, err_inf(new[k], base[k])))
            continue
        report(name, rel_vs_mask0=err_inf(new[k], base[k]) / scale_inf(base[k]))
        try:
            parity(name, new[k], ref64[k], ref32[k], tol=1e-4)
        except AssertionError as e:
            failures.append(str(e))
    assert not failures, "\n".join(failures)


def _oracle_params(g, name, dt):
    """the pinned oracle's parameters in dtype dt on the device, as leaves of their own gradients"""
    return {k: v.to(DEV, copy=True).requires_grad_(True) for k, v in oracle_params(g, name, dt).items()}


class _ReluInputs(torch.overrides.TorchFunctionMode):
    """Per row, the smallest |input| of every torch.nn.functional.relu called while the mode is on."""

    def __init__(self):
        super().__init__()
        self.margin = None

    def __torch_function__(self, func, types, args=(), kwargs=None):
        if func is torch.nn.functional.relu:
            m = args[0].detach().abs().min(dim=1).values
            self.margin = m if self.margin is None else torch.minimum(self.margin, m)
        return func(*args, **(kwargs or {}))


def _clear_gates(P, inputs, oracle):
    """The first P rows of `inputs` (one row per point) at which no ReLU of the fp64 oracle has its input within 1e-5 of
    zero.  Closer than that, a gate is decided by fp32 rounding (up to 1.7e-6 in these networks' pre-activations), so
    the fp32 oracle, the FFMA engine and the tensor cores each flip a few gates at different points: unfiltered, one flip
    in the colour network's base layer 2 moves its bias gradient by 1.2e-3 of its max on every engine, mask 0 included,
    while the device's fp32 oracle, flipping other gates, shows a noise of 1.4e-4.  About 8 % (colour) and 18 % (NeRF++)
    of the points are dropped; the UDF points are filtered by the same margin on |udf|."""
    with _ReluInputs() as r, torch.no_grad():
        oracle(*[t.double().to(DEV) for t in inputs])
    keep = (r.margin >= 1e-5).cpu()
    out = [t[keep][:P] for t in inputs]
    assert out[0].shape[0] == P
    return out


def _grads(loss, params, names):
    gr = torch.autograd.grad(loss, params, allow_unused=True)
    return {"d." + k: (torch.zeros_like(p) if d is None else d) for k, p, d in zip(names, params, gr)}


# ---------------------------------------------------------------------------------------------------------------
# UDF network
# ---------------------------------------------------------------------------------------------------------------
def _udf_loss(u, f, grad, bars, sub):
    loss = 0.0
    for key, t in (("u", u), ("f", f), ("g", grad)):
        if key in sub:
            loss = loss + (t * bars[key]).sum()
    return loss


def _udf_module_run(udf, x, bars, sub):
    for p in udf.parameters():
        p.grad = None
    u, f, grad = udf.value_feature_gradient(x)
    _udf_loss(u, f, grad, bars, sub).backward()
    out = {"udf": u.detach(), "feature": f.detach(), "grad": grad.detach()}
    out.update({"d." + k: p.grad.clone() for k, p in udf.named_parameters()})
    return out


def _udf_oracle(g, name, cfg, x, bars, sub, dt):
    p = _oracle_params(g, name, dt)
    xg = x.to(DEV, dt).requires_grad_(True)
    out = O.udf_mlp(p, cfg, xg)
    u, f = out[:, :1], out[:, 1:]
    grad = torch.autograd.grad(u, xg, torch.ones_like(u), create_graph=True)[0]
    loss = _udf_loss(u, f, grad, {k: v.to(DEV, dt) for k, v in bars.items()}, sub)
    res = {"udf": u.detach(), "feature": f.detach(), "grad": grad.detach()}
    res.update(_grads(loss, list(p.values()), list(p.keys())))
    return res


def _udf_points(g, name, cfg, P):
    """P points of test_gpu_chain's mix (a third within 2e-4 of the sphere the scene was initialised to), without those
    where |udf| < 1e-5: there sign(y0), and with it grad_x udf, is fp32 rounding noise (SURVEY 8(c)), in the oracle's fp32
    run and in every engine alike.  Without the filter the 65 499-point set has |y0| down to 1.2e-6, against an fp32
    error of y0 up to 1.2e-6."""
    x = _points(P + P // 8 + 8, 29 + P).float()
    u64 = O.udf_mlp(_oracle_params(g, name, torch.float64), cfg, x.double().to(DEV)).detach()[:, 0].cpu()
    x = x[u64 >= 1e-5][:P]
    assert x.shape[0] == P
    return x


def _udf_workload(g, name, P, sub):
    cfg = g.udf_c if name == "udf" else g.udf_small_c
    udf = build_modules(g, DEV, name)[0]
    x = _udf_points(g, name, cfg, P)
    gen = torch.Generator().manual_seed(7 + P)
    bars = {"u": torch.randn(P, 1, generator=gen), "f": torch.randn(P, cfg["d_out"] - 1, generator=gen),
            "g": torch.randn(P, 3, generator=gen)}
    xd, barsd = x.to(DEV), {k: v.to(DEV) for k, v in bars.items()}
    base, counts0 = _run(0, lambda: _udf_module_run(udf, xd, barsd, SUBSETS[sub]))
    ref64 = _udf_oracle(g, name, cfg, x.double(), bars, SUBSETS[sub], torch.float64)
    ref32 = _udf_oracle(g, name, cfg, x, bars, SUBSETS[sub], torch.float32)
    return dict(udf=udf, cfg=cfg, x=xd, bars=barsd, base=base, counts0=counts0, ref64=ref64, ref32=ref32)


def _udf_routing(mask, n_lin, sub):
    """launches per tensor-core family of one forward (value_feature_gradient) + backward (udf_net.cu)"""
    has_out, has_grad = ("u" in sub or "f" in sub), "g" in sub
    want = {}
    if mask & 1:     # the n_lin - 1 hidden layers and the feature rows of the last layer
        want["tc_layer_other"] = n_lin
    if mask & 2:     # layers n_lin - 2 .. 1 (EpiRev) and layer 0 (EpiRevFinal)
        want["tc_layer_reverse_sweep"] = n_lin - 1
    if mask & 4:     # one per hidden layer, only with an upstream gradient of grad_x udf
        want["tc_layer_tangent"] = n_lin - 1 if has_grad else 0
    if mask & 8:     # the top layer (EpiBwdR1) only with a udf / feature upstream, then layers n_lin - 2 .. 1 (EpiBwd)
        want["tc_layer_backward"] = n_lin - 1 if has_out else n_lin - 2
    if mask & 16:    # per hidden layer for the tangent chain and for the backward chain, plus the top layer's feature rows
        want["tc_weight_gradient"] = (n_lin - 1) * (2 if has_grad else 1) + (1 if has_out else 0)
    return want


def _udf_reach(mask, sub, names):
    if mask & 1:
        return set(names)
    params = {k for k in names if k.startswith("d.")}
    reach = set()
    if mask & 2:                                 # D (the reverse sweep's output) feeds the tangent chain
        reach |= {"grad"} | (params if "g" in sub else set())
    if mask & 4 and "g" in sub:
        reach |= params
    if mask & (8 | 16):
        reach |= params
    return reach


@pytest.mark.parametrize("name,P,sub,mask", UDF_CASES)
def test_udf_chain(golden, refs, name, P, sub, mask):
    w = refs.get(("udf", name, P, sub), lambda: _udf_workload(golden, name, P, sub))
    tag = "tc_chain.%s.P%d.m%d.%s" % (name, P, mask, sub)
    _check_routing(tag + " (mask 0)", w["counts0"], {})
    new, counts = _run(mask, lambda: _udf_module_run(w["udf"], w["x"], w["bars"], SUBSETS[sub]))
    _check_routing(tag, counts, _udf_routing(mask, len(w["cfg"]["layers"]), SUBSETS[sub]))
    _check_run(tag, new, w["base"], w["ref64"], w["ref32"], _udf_reach(mask, SUBSETS[sub], new))


# ---------------------------------------------------------------------------------------------------------------
# colour network
# ---------------------------------------------------------------------------------------------------------------
def _color_module_run(col, pts, dirs, feat, bars):
    for p in col.parameters():
        p.grad = None
    featg = feat.clone().requires_grad_(True)
    o = col(pts, None, dirs, featg)
    sum((t * b).sum() for t, b in zip(o, bars)).backward()
    out = {"color_base": o[0].detach(), "color": o[1].detach(), "blend": o[2].detach(), "dfeat": featg.grad}
    out.update({"d." + k: p.grad.clone() for k, p in col.named_parameters()})
    return out


def _color_oracle(g, pts, dirs, feat, bars, dt):
    p = _oracle_params(g, "color", dt)
    f = feat.to(DEV, dt).requires_grad_(True)
    o = O.color_mlp(p, g.col_c, pts.to(DEV, dt), dirs.to(DEV, dt), f)
    loss = sum((t * b.to(DEV, dt)).sum() for t, b in zip(o, bars))
    res = {"color_base": o[0].detach(), "color": o[1].detach(), "blend": o[2].detach()}
    gr = _grads(loss, list(p.values()) + [f], list(p.keys()) + ["feat"])
    res["dfeat"] = gr.pop("d.feat")
    res.update(gr)
    return res


def _color_workload(g):
    col = build_modules(g, DEV)[1]
    P = BIG
    gen = torch.Generator().manual_seed(41)
    n = P + P // 4
    pts = torch.rand(n, 3, generator=gen) * 2 - 1
    dirs = torch.randn(n, 3, generator=gen)
    dirs = dirs / dirs.norm(dim=1, keepdim=True)
    feat = 0.3 * torch.randn(n, g.col_c["d_feature"], generator=gen)
    p64 = _oracle_params(g, "color", torch.float64)
    pts, dirs, feat = _clear_gates(P, (pts, dirs, feat), lambda *t: O.color_mlp(p64, g.col_c, *t))
    cc = g.col_c
    bars = [torch.randn(P, k, generator=gen) for k in (cc["d_out"], cc["d_out"], cc["blending_cand_views"])]
    dev = [t.to(DEV) for t in (pts, dirs, feat)]
    barsd = [b.to(DEV) for b in bars]
    base, counts0 = _run(0, lambda: _color_module_run(col, *dev, barsd))
    ref64 = _color_oracle(g, pts.double(), dirs.double(), feat.double(), [b.double() for b in bars], torch.float64)
    ref32 = _color_oracle(g, pts, dirs, feat, bars, torch.float32)
    return dict(col=col, dev=dev, bars=barsd, base=base, counts0=counts0, ref64=ref64, ref32=ref32)


@pytest.mark.parametrize("mask", COLOR_MASKS)
def test_color_chain(golden, refs, mask):
    w = refs.get(("color",), lambda: _color_workload(golden))
    tag = "tc_chain.color.P%d.m%d.all" % (BIG, mask)
    _check_routing(tag + " (mask 0)", w["counts0"], {})
    new, counts = _run(mask, lambda: _color_module_run(w["col"], *w["dev"], w["bars"]))
    want = {}
    if mask & (32 | 128):
        want["tc_layer_other"] = None
    if mask & 16:
        want["tc_weight_gradient"] = None
    _check_routing(tag, counts, want)
    params = {k for k in new if k.startswith("d.")}
    if mask & 128:
        reach = set(new)
    else:
        reach = params | ({"dfeat"} if mask & 32 else set())
    _check_run(tag, new, w["base"], w["ref64"], w["ref32"], reach)


# ---------------------------------------------------------------------------------------------------------------
# NeRF++ background network
# ---------------------------------------------------------------------------------------------------------------
def _nerf_module_run(nerf, pts, dirs, bars):
    for p in nerf.parameters():
        p.grad = None
    a, rgb = nerf(pts, dirs)
    ((a * bars[0]).sum() + (rgb * bars[1]).sum()).backward()
    out = {"alpha": a.detach(), "rgb": rgb.detach()}
    out.update({"d." + k: p.grad.clone() for k, p in nerf.named_parameters()})
    return out


def _nerf_oracle(g, pts, dirs, bars, dt):
    p = _oracle_params(g, "nerf", dt)
    a, rgb = O.nerf_mlp(p, g.nerf_c, pts.to(DEV, dt), dirs.to(DEV, dt))
    loss = (a * bars[0].to(DEV, dt)).sum() + (rgb * bars[1].to(DEV, dt)).sum()
    res = {"alpha": a.detach(), "rgb": rgb.detach()}
    res.update(_grads(loss, list(p.values()), list(p.keys())))
    return res


def _nerf_workload(g):
    nerf = build_modules(g, DEV)[2]
    P = BIG
    gen = torch.Generator().manual_seed(43)
    n = P + P // 3
    pts = torch.randn(n, 4, generator=gen, dtype=torch.float64)
    pts = (pts / pts[:, :3].norm(dim=1, keepdim=True)).float()
    dirs = torch.randn(n, 3, generator=gen)
    dirs = dirs / dirs.norm(dim=1, keepdim=True)
    p64 = _oracle_params(g, "nerf", torch.float64)
    pts, dirs = _clear_gates(P, (pts, dirs), lambda *t: O.nerf_mlp(p64, g.nerf_c, *t))
    bars = [torch.randn(P, 1, generator=gen), torch.randn(P, 3, generator=gen)]
    dev = [pts.to(DEV), dirs.to(DEV)]
    barsd = [b.to(DEV) for b in bars]
    base, counts0 = _run(0, lambda: _nerf_module_run(nerf, *dev, barsd))
    ref64 = _nerf_oracle(g, pts.double(), dirs.double(), [b.double() for b in bars], torch.float64)
    ref32 = _nerf_oracle(g, pts, dirs, bars, torch.float32)
    return dict(nerf=nerf, dev=dev, bars=barsd, base=base, counts0=counts0, ref64=ref64, ref32=ref32)


@pytest.mark.parametrize("mask", NERF_MASKS)
def test_nerf_chain(golden, refs, mask):
    w = refs.get(("nerf",), lambda: _nerf_workload(golden))
    tag = "tc_chain.nerf.P%d.m%d.all" % (BIG, mask)
    _check_routing(tag + " (mask 0)", w["counts0"], {})
    new, counts = _run(mask, lambda: _nerf_module_run(w["nerf"], *w["dev"], w["bars"]))
    want = {}
    if mask & (64 | 128):
        want["tc_layer_other"] = None
    if mask & 16:
        want["tc_weight_gradient"] = None
    _check_routing(tag, counts, want)
    reach = set(new) if mask & 128 else {k for k in new if k.startswith("d.")}
    _check_run(tag, new, w["base"], w["ref64"], w["ref32"], reach)

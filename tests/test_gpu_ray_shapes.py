"""GPU tests of the sampling and compositing kernels away from the shipped sample counts: a shape sweep against fp64.

Every other test of csrc/sampling.cu and csrc/ray_kernels.cu runs the shipped confs' counts (DTU 64 + 50 in five rounds of
10, 32 NeRF++ samples; garment 64 + 80, m = 13) or four small synthetic cases.  Those kernels branch on exactly these counts:
the `k += 32` loop of sample_pdf_warp past 32 new samples per ray, dynamic shared memory above 48 KB (composite at
S + O >= 308, up-sampling at n >= 385, inverse-CDF sampling at n >= 1025) up to the largest size each entry point accepts,
warp scans of one chunk or with a chunk boundary exactly at S or S + O, exact ties in the sorted merge, a strided udf
column, the `weights` adjoint, and rays that are opaque or far from any surface.  Each configuration below names the branch
it is there for.

Compositing runs through ops.composite (forward and backward) and is checked against the pinned oracle's composite in fp64
with autograd (the arbiter), the oracle's fp32 run being the noise yardstick (parity(): 2e-4 forward, 2e-3 backward).  The
synthetic inputs are nudged at least 1e-4 away from every hard threshold of the reference (true_cos < 0.01, the sign of the
normalised cosine, |p| < 1, |p| < 1.2, udf < 0.05), so that a mask flip cannot pass for a kernel error nor hide one; the
clamp edges at exactly 0 and 1 are produced on purpose (q = 1 exactly where raw_occ underflows, q > 1 past it).  Sampling
indices must equal the CPU fp32 oracle's except at near-ties, which are counted and reported; sample values are compared
with fp64 where the indices agree.  The whole renderer then runs sampling schedules the CLI accepts and no other test runs.
"""
import ctypes
import time

import numpy as np
import pytest
import torch

from neuraludf_b200 import _lib as L
from neuraludf_b200 import ops
from oracle import oracle_torch as O
from tests.gpu_util import build_modules, err_inf, oracle_params, parity, report, scale_inf

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64, F32 = torch.float64, torch.float32

# thresholds of the reference and how far every synthetic sample is kept from them
TC_MASK, TC_UP, UDF_NEAR, R_IN, R_RELAX = 0.01, 0.05, 0.05, 1.0, 1.2
MARGIN = 1e-4


@pytest.fixture(scope="module", autouse=True)
def _device():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    t0 = time.perf_counter()
    yield
    report("ray_shapes.module_seconds", seconds=time.perf_counter() - t0)


def _status_clear():
    ops.status_word(torch.device(DEV)).zero_()


@pytest.fixture(autouse=True)
def _status_word():
    """a failed check must not leave the device status bit set for whatever runs next in the process"""
    yield
    _status_clear()


def _assert_status_clear():
    assert int(ops.status_word(torch.device(DEV)).item()) == 0, "a kernel raised the non-finite status bit"


def _rays(N, seed):
    """rays from a radius-2.5 shell towards the origin, near / far 1.4 either side of the closest approach: every ray
    enters and leaves both the unit sphere and the 1.2 sphere"""
    o, d, near, far = O.make_rays(N, seed)
    mid = 0.5 * (near + far)
    return o, d, mid - 1.4, mid + 1.4


# ---------------------------------------------------------------------------------------------------------------
# synthetic compositing inputs
# ---------------------------------------------------------------------------------------------------------------
# (inv_s, beta, gamma) per UDF profile
HEADS = {"near": (403.4, 148.4, 20.1), "far": (403.4, 148.4, 20.1), "opaque": (2000.0, 148.4, 20.1)}


def _nudge_masks(pts, d, grads, udf):
    """Move every sample at least MARGIN away from the reference's hard thresholds (in place, fp32 values, fp64 tests);
    returns the smallest distance to a threshold found afterwards."""
    dd = d.double()[:, None, :]
    for _ in range(20):
        r = pts.double().norm(dim=-1)
        bad_r = ((r - R_IN).abs() < MARGIN) | ((r - R_RELAX).abs() < MARGIN)
        pts[bad_r] = (pts[bad_r].double() * (1.0 + 3 * MARGIN)).float()
        g = grads.double()
        tc = (dd * g).sum(-1)
        cosn = (dd * (g / (g.norm(dim=-1, keepdim=True) + 1e-5))).sum(-1)
        bad_c = ((tc - TC_MASK).abs() < MARGIN) | ((cosn - TC_MASK).abs() < MARGIN) | (cosn.abs() < MARGIN)
        grads[bad_c] = (g[bad_c] + 3 * MARGIN * dd.expand_as(g)[bad_c]).float()
        bad_u = (udf.double() - UDF_NEAR).abs() < MARGIN
        udf[bad_u] = (udf[bad_u].double() + 3 * MARGIN).float()
        if not (bool(bad_r.any()) or bool(bad_c.any()) or bool(bad_u.any())):
            break
    r = pts.double().norm(dim=-1)
    g = grads.double()
    tc = (dd * g).sum(-1)
    cosn = (dd * (g / (g.norm(dim=-1, keepdim=True) + 1e-5))).sum(-1)
    return min(float((r - R_IN).abs().min()), float((r - R_RELAX).abs().min()), float((tc - TC_MASK).abs().min()),
               float((cosn - TC_MASK).abs().min()), float(cosn.abs().min()), float((udf.double() - UDF_NEAR).abs().min()))


def make_case(seed, N, S, O_, profile):
    """tests/test_raymath_host.make_case for any N, S and O, with three UDF profiles:
    near   -- a sphere-like UDF scaled into the near-surface band, as the other compositing tests use;
    far    -- udf >= 0.8: beta * udf > 110, so raw_occ underflows to 0 in fp32 and q = 1 - alpha_occ is exactly 1;
    opaque -- a thin shell (udf 0.02 |r - 0.5|) seen at inv_s = 2000: alpha ~ 1 at the crossings and T at the 1e-7 floor."""
    g = torch.Generator().manual_seed(seed)
    o, d, near, far = _rays(N, seed)
    z = near + (far - near) * torch.linspace(0, 1, S)[None, :]
    sd = float(((far - near) / S).mean())
    dists = torch.cat([z[:, 1:] - z[:, :-1], torch.full((N, 1), sd)], -1)
    mid = z + dists * 0.5
    pts = (o[:, None, :] + d[:, None, :] * mid[..., None]).contiguous()
    rs = (pts.norm(dim=-1) - 0.5).abs()
    scale = {"near": 0.05, "far": 1.0, "opaque": 0.02}[profile]
    udf = (rs * scale + (0.8 if profile == "far" else 0.0)
           + (1e-4 if profile == "opaque" else 1e-3) * torch.rand(N, S, generator=g)).float()
    grads = (pts / pts.norm(dim=-1, keepdim=True) * torch.sign(pts.norm(dim=-1, keepdim=True) - 0.5)
             + 0.2 * torch.randn(N, S, 3, generator=g)).float()
    margin = _nudge_masks(pts, d, grads, udf)
    assert margin >= MARGIN, "input within %.1e of a threshold" % margin
    scb = torch.rand(N, S, 3, generator=g)
    sc = torch.rand(N, S, 3, generator=g)
    bga = torch.rand(N, S + O_, generator=g) * 0.3
    bgc = torch.rand(N, S + O_, 3, generator=g)
    cpix = torch.rand(N, S, 3, generator=g)
    return dict(o=o, d=d, z=z, dists=dists, mid=mid, pts=pts, udf=udf, grads=grads, scb=scb, sc=sc, bga=bga, bgc=bgc,
                cpix=cpix, sd=sd)


# (S, O, N, profile, cos_anneal_ratio, flip_saturation, use_norm_grad_for_cosine, background_rgb on, branch)
COMPOSITE_CFGS = {
    "one":     (1, 0, 1, "near", None, 0.0, 0, 0, "one sample: dist = sample_dist, a single partial chunk"),
    "s7":      (7, 0, 5, "far", 0.0, 0.0, 1, 1, "S < 32, last block partly empty; q = 1 exactly (inclusive clamp edge)"),
    "so32":    (31, 1, 4, "opaque", 0.35, 1.5, 0, 1, "S + O = 32: one transmittance chunk, the fg scans end at 31"),
    "s32":     (32, 0, 9, "near", 1.0, 0.4, 1, 0, "S = 32: fg scans end exactly at a chunk boundary"),
    "s32o32":  (32, 32, 6, "opaque", None, 0.4, 0, 1, "chunk boundaries at S and at S + O"),
    "so64":    (33, 31, 6, "far", 0.35, 1.5, 1, 0, "S + O = 64; q > 1 (gradient masked)"),
    "dtu":     (114, 32, 512, "near", 0.35, 0.4, 0, 0, "DTU control at the runner's batch"),
    "garment": (142, 0, 512, "near", 1.0, 0.0, 0, 0, "garment control at the runner's batch"),
    "smem":    (300, 8, 13, "opaque", 0.0, 0.4, 1, 1, "S + O = 308: the first size above 48 KB of shared memory"),
    "max":     (1000, 280, 3, "near", None, 1.5, 0, 1, "S + O = 1280: the largest size the kernels accept"),
    "blocks":  (64, 32, 4099, "near", 0.35, 0.4, 1, 1, "many blocks, a ragged last block"),
}
BG_RGB = torch.tensor([0.2, 0.5, 0.9])
SSF = 300.0
FWD_KEYS = ("color_base", "color", "depth", "weight_sum", "weight_sum_fg_bg")
DIAG = ("weights", "normals", "vis_prob", "alpha", "alpha_plus", "alpha_minus", "alpha_occ", "raw_occ", "true_cos",
        "gradient_mag", "gradients_flip")


def _oracle_composite(c, S, O_, profile, r, fs, use_norm, bg, dt, bars):
    """oracle composite in dtype dt with autograd: (outputs, gradients of the test loss by input name)"""
    leaves = {k: c[k].to(dt).clone().requires_grad_(True) for k in ("udf", "grads", "scb", "sc", "bga", "bgc")}
    heads = [torch.tensor(v, dtype=dt, requires_grad=True) for v in HEADS[profile]]
    ret = O.composite(c["d"].to(dt), c["pts"].to(dt), c["mid"].to(dt), c["dists"].to(dt), leaves["udf"], leaves["grads"],
                      leaves["scb"], leaves["sc"], heads[0], heads[1], heads[2], cos_anneal_ratio=r, flip_saturation=fs,
                      background_rgb=BG_RGB.to(dt) if bg else None, background_alpha=leaves["bga"] if O_ else None,
                      background_sampled_color=leaves["bgc"] if O_ else None, sparse_scale_factor=SSF,
                      use_norm_grad_for_cosine=bool(use_norm))
    loss = sum((ret[k] * bars[k].to(dt)).sum() for k in FWD_KEYS + ("weights",)) + bars["reg"][0] * ret["gradient_error"] \
        + bars["reg"][1] * ret["gradient_error_near_surface"] + bars["reg"][2] * ret["sparse_error"]
    names = ["udf", "grads", "scb", "sc"] + (["bga", "bgc"] if O_ else [])
    gr = torch.autograd.grad(loss, [leaves[k] for k in names] + heads)
    grads = dict(zip(names, gr[:len(names)]))
    grads["heads"] = torch.stack(list(gr[len(names):]))
    return {k: (v.detach() if isinstance(v, torch.Tensor) else v) for k, v in ret.items()}, grads


def _device_inputs(c, S, O_, profile, r, fs, use_norm, bg, rows=None):
    """leaves and launch arguments of ops.composite for rays `rows` (all by default)"""
    sel = slice(None) if rows is None else slice(0, rows)
    N = c["udf"][sel].shape[0]
    P = N * S
    dev = lambda t: t[sel].float().to(DEV).contiguous()
    leaves = dict(udf=dev(c["udf"]).reshape(P), grads=dev(c["grads"]).reshape(P, 3), scb=dev(c["scb"]).reshape(P, 3),
                  sc=dev(c["sc"]).reshape(P, 3), bga=dev(c["bga"]) if O_ else None, bgc=dev(c["bgc"]) if O_ else None,
                  heads=torch.tensor(HEADS[profile], device=DEV))
    cfg = ops._make_cfg(N, S, O_, c["sd"], r, fs, SSF, bool(use_norm), BG_RGB if bg else None)
    geom = (dev(c["d"]), dev(c["pts"]).reshape(P, 3), dev(c["mid"]), dev(c["dists"]))
    return leaves, cfg, geom


def _run_composite(leaves, cfg, geom, bar_dev, udf=None, udf_leaf=None):
    """forward + backward through ops.composite with explicit upstream gradients (bar_dev: per-ray tensors, ray_sums
    included); returns (outputs, {input: gradient}).  udf: another udf argument, a view of udf_leaf (the tensor whose
    gradient is returned) when given."""
    ls = {k: (v.clone().requires_grad_(True) if v is not None else None) for k, v in leaves.items()}
    u = ls["udf"] if udf is None else udf
    comp = ops.composite(u, ls["grads"], ls["scb"], ls["sc"], ls["bga"], ls["bgc"], ls["heads"], geom, cfg)
    outs = [comp[k] for k in bar_dev]
    wrt = [t for t in ([u if udf_leaf is None else udf_leaf] + [ls[k] for k in ("grads", "scb", "sc", "bga", "bgc", "heads")])
           if t is not None]
    gr = torch.autograd.grad(outs, wrt, [bar_dev[k] for k in bar_dev])
    names = ["udf", "grads", "scb", "sc"] + (["bga", "bgc"] if ls["bga"] is not None else []) + ["heads"]
    return {k: v.detach() for k, v in comp.items()}, dict(zip(names, gr))


@pytest.mark.parametrize("name", list(COMPOSITE_CFGS))
def test_composite_shapes_vs_fp64(name):
    S, O_, N, profile, r, fs, use_norm, bg, why = COMPOSITE_CFGS[name]
    c = make_case(7919 + S * 31 + O_, N, S, O_, profile)
    gen = torch.Generator().manual_seed(17 + S)
    bars = {k: torch.randn(N, w, generator=gen, dtype=F64) for k, w in (("color_base", 3), ("color", 3), ("depth", 1),
                                                                        ("weight_sum", 1), ("weight_sum_fg_bg", 1))}
    bars["weights"] = torch.randn(N, S + O_ if O_ else S, generator=gen, dtype=F64)
    bars["reg"] = torch.randn(3, generator=gen, dtype=F64)
    torch.set_num_threads(min(32, torch.get_num_threads()))
    r64, g64 = _oracle_composite(c, S, O_, profile, r, fs, use_norm, bg, F64, bars)
    r32, g32 = _oracle_composite(c, S, O_, profile, r, fs, use_norm, bg, F32, bars)
    if profile == "far":
        assert float(r32["raw_occ"].abs().max()) == 0.0 and bool((r32["alpha_occ"] == 0).all())
    if profile == "opaque":
        # some sample is opaque to fp32: 1 - alpha + 1e-7 at the floor
        assert float(r64["alpha"].max()) > 1.0 - 1e-7
    _status_clear()
    leaves, cfg, geom = _device_inputs(c, S, O_, profile, r, fs, use_norm, bg)
    P = N * S
    ls = {k: (v.clone().requires_grad_(True) if v is not None else None) for k, v in leaves.items()}
    comp = ops.composite(ls["udf"], ls["grads"], ls["scb"], ls["sc"], ls["bga"], ls["bgc"], ls["heads"], geom, cfg)
    tag = "ray_shapes.composite[%s]." % name
    worst = {}

    def check(key, new, k64, k32, tol):
        parity(tag + key, new, k64, k32, tol=tol)
        worst[key] = err_inf(new, k64) / scale_inf(k64)

    for k in FWD_KEYS + DIAG:
        check(k, comp[k].reshape(r64[k].shape), r64[k], r32[k], 2e-4)
    assert torch.equal(comp["inside_sphere"].cpu().double(), r64["inside_sphere"]), "inside_sphere mask differs"
    rs = comp["ray_sums"]
    ge = rs[:, 0].sum() / (rs[:, 1].sum().detach() + 1e-5)
    gens = rs[:, 2].sum() / (rs[:, 3].sum().detach() + 1e-5)
    sp = rs[:, 4].sum() / N
    check("gradient_error", ge, r64["gradient_error"], r32["gradient_error"], 2e-4)
    check("gradient_error_ns", gens, r64["gradient_error_near_surface"], r32["gradient_error_near_surface"], 2e-4)
    check("sparse_error", sp, r64["sparse_error"], r32["sparse_error"], 2e-4)
    dvb = lambda k: bars[k].float().to(DEV)
    loss = sum((comp[k] * dvb(k)).sum() for k in FWD_KEYS + ("weights",)) + float(bars["reg"][0]) * ge \
        + float(bars["reg"][1]) * gens + float(bars["reg"][2]) * sp
    loss.backward()
    _assert_status_clear()
    tol = 2e-3
    check("udf_bar", ls["udf"].grad.reshape(N, S), g64["udf"], g32["udf"], tol)
    check("grads_bar", ls["grads"].grad.reshape(N, S, 3), g64["grads"], g32["grads"], tol)
    check("scb_bar", ls["scb"].grad.reshape(N, S, 3), g64["scb"], g32["scb"], tol)
    check("sc_bar", ls["sc"].grad.reshape(N, S, 3), g64["sc"], g32["sc"], tol)
    check("heads_bar", ls["heads"].grad, g64["heads"], g32["heads"], tol)
    if O_:
        # behind an opaque surface these adjoints are ~1e-100: an absolute floor tied to the foreground adjoints
        floor = 1e-6 * scale_inf(g64["scb"])
        for k in ("bga", "bgc"):
            new, a64, a32 = ls[k].grad[:, S:], g64[k][:, S:], g32[k][:, S:]
            e = err_inf(new, a64)
            bound = max(tol * scale_inf(a64), 2.0 * err_inf(a32, a64)) + floor
            report(tag + k + "_bar", err=e, rel=e / scale_inf(a64), bound=bound, ok=bool(e <= bound))
            assert e <= bound, (k, e, bound)
            worst[k + "_bar"] = e / scale_inf(a64)
        # the foreground columns of bg_alpha / bg_color take no gradient
        assert float(ls["bga"].grad[:, :S].abs().max()) == 0.0 and float(ls["bgc"].grad[:, :S].abs().max()) == 0.0
    key = max(worst, key=worst.get)
    report("ray_shapes.composite_worst", config=name, S=S, O=O_, N=N, profile=profile, why=why, worst_key=key,
           worst_rel=worst[key])


def _bars_device(N, S, O_, seed):
    gen = torch.Generator().manual_seed(seed)
    w = {"color_base": 3, "color": 3, "depth": 1, "weight_sum": 1, "weight_sum_fg_bg": 1, "ray_sums": 5,
         "weights": S + O_}
    return {k: torch.randn(N, n, generator=gen).to(DEV) for k, n in w.items()}


@pytest.mark.parametrize("name", list(COMPOSITE_CFGS))
def test_composite_shapes_bitwise_invariants(name):
    """rows 0..k of an N-ray run equal a k-ray run (forward and backward); the view renderer's composite gives the
    same color / depth / weight_sum bits as ops.composite, and its normal and color_pixel match an fp64 restatement; a udf
    given as a [P, 5] column (ld_udf = 5) or as [N, S] gives the bits of the contiguous [P] run, its gradient in its
    own shape"""
    S, O_, N, profile, r, fs, use_norm, bg, why = COMPOSITE_CFGS[name]
    c = make_case(7919 + S * 31 + O_, N, S, O_, profile)
    P = N * S
    bar = _bars_device(N, S, O_, 5 + S)
    leaves, cfg, geom = _device_inputs(c, S, O_, profile, r, fs, use_norm, bg)
    _status_clear()
    full, gfull = _run_composite(leaves, cfg, geom, bar)
    # ---- prefix of the batch ----
    k = max(1, (N + 1) // 2)
    lk, cfgk, geomk = _device_inputs(c, S, O_, profile, r, fs, use_norm, bg, rows=k)
    part, gpart = _run_composite(lk, cfgk, geomk, {n: t[:k] for n, t in bar.items()})
    for key in part:
        assert torch.equal(part[key], full[key][:part[key].shape[0]]), "forward %s of rows 0..%d differs" % (key, k)
    for key in ("udf", "grads", "scb", "sc") + (("bga", "bgc") if O_ else ()):
        assert torch.equal(gpart[key], gfull[key][:gpart[key].shape[0]]), "gradient %s of rows 0..%d differs" % (key, k)
    # ---- strided and [N, S] udf ----
    u5 = torch.randn(P, 5, device=DEV)
    u5[:, 3] = leaves["udf"]
    u5.requires_grad_(True)
    col, gcol = _run_composite(leaves, cfg, geom, bar, udf=u5[:, 3], udf_leaf=u5)
    for key in full:
        assert torch.equal(col[key], full[key]), "ld_udf = 5 changes %s" % key
    assert gcol["udf"].shape == (P, 5) and torch.equal(gcol["udf"][:, 3], gfull["udf"])
    assert float(gcol["udf"][:, [0, 1, 2, 4]].abs().max()) == 0.0
    uns = leaves["udf"].reshape(N, S).clone().requires_grad_(True)
    ns, gns = _run_composite(leaves, cfg, geom, bar, udf=uns)
    for key in full:
        assert torch.equal(ns[key], full[key]), "a [N, S] udf changes %s" % key
    assert gns["udf"].shape == (N, S) and torch.equal(gns["udf"].reshape(P), gfull["udf"])
    # ---- the view renderer's composite ----
    rot = [[0.36, 0.48, -0.8], [-0.8, 0.6, 0.0], [0.48, 0.64, 0.6]]
    f = lambda w: torch.full((N, w), float("nan"), device=DEV)
    outs = {"color": f(3), "color_pixel": f(3), "depth": f(1), "normal": f(3), "weight_sum": f(1)}
    cpix = c["cpix"].float().to(DEV).reshape(P, 3).contiguous()
    rays_d, pts, mid, dists = geom
    ops.view_composite(cfg, leaves["heads"], rays_d, pts, mid, dists, leaves["udf"], leaves["grads"], leaves["sc"], cpix,
                       leaves["bga"], leaves["bgc"], rot, outs)
    for key in ("color", "depth", "weight_sum"):
        assert torch.equal(outs[key], full[key]), "view composite %s differs from ops.composite" % key
    # fp64 restatement from the oracle's weights, gradients_flip and inside_sphere
    res = {}
    for dt in (F64, F32):
        ret = O.composite(c["d"].to(dt), c["pts"].to(dt), c["mid"].to(dt), c["dists"].to(dt), c["udf"].to(dt),
                          c["grads"].to(dt), c["scb"].to(dt), c["sc"].to(dt), *[torch.tensor(v, dtype=dt) for v in HEADS[profile]],
                          cos_anneal_ratio=r, flip_saturation=fs, background_rgb=BG_RGB.to(dt) if bg else None,
                          background_alpha=c["bga"].to(dt) if O_ else None,
                          background_sampled_color=c["bgc"].to(dt) if O_ else None, sparse_scale_factor=SSF,
                          use_norm_grad_for_cosine=bool(use_norm))
        w, ins = ret["weights"], ret["inside_sphere"]
        nrm = (ret["gradients_flip"] * w[:, :S, None] * ins[..., None]).sum(dim=1)
        nrm = nrm @ torch.tensor(rot, dtype=dt).T
        cp = c["cpix"].to(dt)
        if O_:
            cp = cp * ins[..., None] + c["bgc"].to(dt)[:, :S] * (1.0 - ins[..., None])
            cp = torch.cat([cp, c["bgc"].to(dt)[:, S:]], dim=1)
        res[dt] = {"normal": nrm, "color_pixel": (cp * w[:, :, None]).sum(dim=1)}
    for key in ("normal", "color_pixel"):
        parity("ray_shapes.view[%s].%s" % (name, key), outs[key], res[F64][key], res[F32][key], tol=2e-4)
    _assert_status_clear()


def test_composite_refusals():
    """S + O = 1281 and mis-shaped tensors are refused on the host, before any launch"""
    c = make_case(3, 2, 8, 0, "near")
    leaves, cfg, geom = _device_inputs(c, 8, 0, "near", None, 0.0, 0, 0)
    big = ops._make_cfg(1, 1000, 281, c["sd"], None, 0.0, SSF, False, None)
    bga, bgc = torch.zeros(1, 1281, device=DEV), torch.zeros(1, 1281, 3, device=DEV)
    one = dict(udf=torch.zeros(1000, device=DEV), grads=torch.zeros(1000, 3, device=DEV), scb=torch.zeros(1000, 3, device=DEV),
               sc=torch.zeros(1000, 3, device=DEV))
    g1 = (torch.ones(1, 3, device=DEV), torch.zeros(1000, 3, device=DEV), torch.zeros(1, 1000, device=DEV),
          torch.zeros(1, 1000, device=DEV))
    with pytest.raises(RuntimeError, match="too many samples"):
        ops.composite(one["udf"], one["grads"], one["scb"], one["sc"], bga, bgc, leaves["heads"], g1, big)
    P = 16
    bad = [("udf", leaves["udf"][:P - 1]), ("udf", leaves["udf"].reshape(P, 1).expand(P, 2)),
           ("udf", leaves["udf"].reshape(4, 4)), ("grads", leaves["grads"][:P - 1]), ("scb", leaves["scb"].reshape(P * 3)[:-3]),
           ("sc", torch.zeros(P, 4, device=DEV))]
    for k, t in bad:
        args = dict(leaves)
        args[k] = t
        with pytest.raises(ValueError, match=k):
            ops.composite(args["udf"], args["grads"], args["scb"], args["sc"], None, None, args["heads"], geom, cfg)
    rays_d, pts, mid, dists = geom
    for i, t in enumerate((rays_d[:1], pts[:-1], mid[:, :-1], dists.reshape(-1)[:-1])):
        gm = list(geom)
        gm[i] = t
        with pytest.raises(ValueError):
            ops.composite(leaves["udf"], leaves["grads"], leaves["scb"], leaves["sc"], None, None, leaves["heads"], tuple(gm), cfg)
    cfg_o = ops._make_cfg(2, 8, 4, c["sd"], None, 0.0, SSF, False, None)
    with pytest.raises(ValueError, match="bg_alpha"):
        ops.composite(leaves["udf"], leaves["grads"], leaves["scb"], leaves["sc"], torch.zeros(2, 11, device=DEV),
                      torch.zeros(2, 12, 3, device=DEV), leaves["heads"], geom, cfg_o)
    with pytest.raises(ValueError, match="bg_color"):
        ops.composite(leaves["udf"], leaves["grads"], leaves["scb"], leaves["sc"], torch.zeros(2, 12, device=DEV),
                      torch.zeros(2, 12, 2, device=DEV), leaves["heads"], geom, cfg_o)


# ---------------------------------------------------------------------------------------------------------------
# B. sampling
# ---------------------------------------------------------------------------------------------------------------
def _near_tie_check(tag, inds, ref_inds, cdf32, cdf64, u):
    """Indices must equal the fp32 oracle's, except at near-ties: a mismatch is one only if every fp64 cdf entry the two
    indices disagree about lies within 8x the ray's own max|cdf32 - cdf64| (floor 1e-7) of u_k.  Returns the count."""
    inds, ref_inds = inds.cpu(), ref_inds.cpu()
    mism = (inds != ref_inds).nonzero().tolist()
    dev = (cdf32.double() - cdf64).abs().max(dim=1).values
    bad = []
    n = cdf64.shape[1]
    for r, k in mism:
        lo, hi = sorted((int(inds[r, k]), int(ref_inds[r, k])))
        if lo < 0 or hi > n:
            bad.append((r, k, int(inds[r, k]), int(ref_inds[r, k]), None, float(dev[r])))
            continue
        gap = float((cdf64[r, lo:hi] - float(u[k])).abs().max())
        if gap > max(8.0 * float(dev[r]), 1e-7):
            bad.append((r, k, int(inds[r, k]), int(ref_inds[r, k]), gap, float(dev[r])))
    report(tag + ".near_ties", count=len(mism), total=int(inds.numel()), not_ties=len(bad))
    assert not bad, "index mismatches that are not near-ties (ray, k, ours, oracle, |cdf - u|, cdf noise): %s" % bad[:5]
    return len(mism)


def _check_samples(tag, s, inds, ref, s64, s32):
    """sample values where all three index sets agree, to fp64 with the up-sampling bound; non-decreasing per ray"""
    s = s.cpu()
    assert bool((s[:, 1:] >= s[:, :-1]).all()), "samples of a ray decrease"
    agree = (inds.cpu() == ref[0]) & (inds.cpu() == ref[1])
    parity(tag + ".samples", s[agree], s64[agree], s32[agree], tol=1e-5, noise_mult=4.0)


def _bins(N, n, seed):
    g = torch.Generator().manual_seed(seed)
    base = 0.5 + 3.0 * torch.rand(N, 1, generator=g)
    steps = torch.rand(N, n, generator=g) * (3.0 / n) + 1e-3
    return (base + torch.cumsum(steps, dim=1)).float()


def _weights(N, n, profile, seed):
    g = torch.Generator().manual_seed(seed)
    if profile == "random":
        return torch.rand(N, n - 1, generator=g)
    if profile == "zero":                               # a flat pdf
        return torch.zeros(N, n - 1)
    if profile == "spikes":                             # one-hot spikes: cdf plateaus, the denom < 1e-5 branch
        w = torch.zeros(N, n - 1)
        k = torch.randint(0, n - 1, (N, 2), generator=g)
        w.scatter_(1, k, torch.rand(N, 2, generator=g) + 0.5)
        return w
    j = torch.arange(n - 1, dtype=torch.float64)       # steep decay
    return torch.exp(-30.0 * j / max(n - 2, 1))[None, :].expand(N, -1).float().contiguous()


# (n bins, m samples, N rays, weight profile)
PDF_CASES = [(2, 1, 4099, "random"), (2, 33, 5, "zero"), (3, 32, 4099, "spikes"), (3, 129, 1, "decay"),
             (33, 31, 4099, "decay"), (33, 50, 5, "spikes"), (65, 129, 4099, "random"), (65, 32, 5, "zero"),
             (1025, 50, 5, "spikes"), (1025, 33, 1, "random"), (4266, 129, 5, "decay"), (4266, 1, 1, "zero"),
             (4266, 31, 5, "random")]


@pytest.mark.parametrize("n,m,N,profile", PDF_CASES)
def test_sample_pdf_shapes(n, m, N, profile):
    """m > 32 reaches the `k += 32` loop; n = 1025 / 4266 the shared memory above 48 KB and the largest accepted size"""
    bins, w = _bins(N, n, n * 7 + m), _weights(N, n, profile, n + m)
    _status_clear()
    s, inds = ops.sample_pdf(bins.to(DEV), w.to(DEV), m, return_inds=True)
    tr32, tr64 = [], []
    s32, i32 = O.sample_pdf_det(bins, w, m, return_inds=True, trace=tr32)
    s64, i64 = O.sample_pdf_det(bins.double(), w.double(), m, return_inds=True, trace=tr64)
    tag = "ray_shapes.sample_pdf[n%d,m%d,N%d,%s]" % (n, m, N, profile)
    _near_tie_check(tag, inds, i32, tr32[0]["cdf"], tr64[0]["cdf"], tr64[0]["u"][0])
    _check_samples(tag, s, inds, (i32, i64), s64, s32)
    torch.cuda.synchronize()
    _assert_status_clear()


def test_sample_pdf_refuses_past_the_largest_size():
    bins, w = _bins(1, 4267, 1).to(DEV), torch.rand(1, 4266).to(DEV)
    with pytest.raises(RuntimeError, match="too many bins"):
        ops.sample_pdf(bins, w, 4)


def _sphere_udf(o, d, z):
    p = o[:, None, :] + d[:, None, :] * z[..., None]
    return (p.norm(dim=-1) - 0.5).abs()


def _up_case(N, n, seed):
    """coarse z (uniform, near / far around the unit sphere) and a sphere-like UDF of radius 0.5, every ray kept 1e-4 away
    from |p| = 1 at its samples and every section's true_cos 1e-4 away from 0.05 (the up-sampling masks)"""
    o, d, near, far = _rays(N, seed)
    g = torch.Generator().manual_seed(seed)
    t = torch.linspace(0.0, 1.0, n)[None, :]
    for _ in range(60):
        z = (near + (far - near) * t).float()
        udf = _sphere_udf(o, d, z).float()
        r = (o.double()[:, None, :] + d.double()[:, None, :] * z.double()[..., None]).norm(dim=-1)
        tc = (udf.double()[:, 1:] - udf.double()[:, :-1]) / (z.double()[:, 1:] - z.double()[:, :-1] + 1e-5)
        bad = ((r - 1.0).abs() < MARGIN).any(1) | ((tc - TC_UP).abs() < MARGIN).any(1)
        if not bool(bad.any()):
            break
        shift = torch.rand(N, 1, generator=g) * (2.8 / n) * bad[:, None]
        near, far = near + shift, far + shift
    assert not bool(bad.any()), "could not move the samples off the up-sampling thresholds"
    sd = float(((far - near) / n).mean())
    return o, d, z.contiguous(), udf.contiguous(), sd


# (mode, n, m, N, round i of the runner's schedule)
UP_CASES = [(0, 2, 1, 64, 0), (1, 2, 10, 64, 0), (0, 31, 13, 256, 1), (1, 33, 50, 256, 2), (0, 33, 64, 256, 3),
            (0, 64, 50, 512, 0), (1, 64, 13, 512, 1), (0, 104, 100, 64, 4), (0, 129, 10, 64, 2), (1, 129, 64, 16, 3),
            (0, 385, 50, 8, 1), (1, 385, 100, 8, 0), (0, 1600, 64, 3, 2), (1, 1600, 13, 3, 4)]


@pytest.mark.parametrize("mode,n,m,N,i", UP_CASES)
def test_up_sample_shapes(mode, n, m, N, i):
    """mode 0: up_sample_unbias, mode 1: up_sample_no_occ_aware; inv_s = 64 2^i, beta = 64 2^(i+1), gamma = 20 2^(5-i)
    clipped to 20..320, as the runner's rounds; n = 385 / 1600 above 48 KB of shared memory, m = 50 / 64 / 100 past 32"""
    o, d, z, udf, sd = _up_case(N, n, 31 * n + m)
    inv_s, beta, gamma = 64.0 * 2 ** i, 64.0 * 2 ** (i + 1), float(np.clip(20 * 2 ** (5 - i), 20, 320))
    _status_clear()
    s, inds = ops.up_sample(mode, o.to(DEV), d.to(DEV), z.to(DEV), udf.to(DEV), sd, m, inv_s, beta, gamma, return_inds=True)
    res = {}
    for dt in (F32, F64):
        tr = []
        a = (o.to(dt), d.to(dt), z.to(dt), udf.to(dt), sd, m)
        if mode == 0:
            smp, ri = O.up_sample_unbias(*a, inv_s, beta, gamma, return_inds=True, trace=tr)
        else:
            smp, ri = O.up_sample_no_occ_aware(*a, beta, gamma, return_inds=True, trace=tr)
        res[dt] = (smp, ri, tr[0])
    tag = "ray_shapes.up_sample[mode%d,n%d,m%d,N%d,i%d]" % (mode, n, m, N, i)
    _near_tie_check(tag, inds, res[F32][1], res[F32][2]["cdf"], res[F64][2]["cdf"], res[F64][2]["u"][0])
    _check_samples(tag, s, inds, (res[F32][1], res[F64][1]), res[F64][0], res[F32][0])
    torch.cuda.synchronize()
    _assert_status_clear()


def test_up_sample_refuses_past_the_largest_size():
    o, d, z, udf, sd = _up_case(1, 1601, 5)
    for mode in (0, 1):
        with pytest.raises(RuntimeError, match="too many samples"):
            ops.up_sample(mode, o.to(DEV), d.to(DEV), z.to(DEV), udf.to(DEV), sd, 4, 64.0, 128.0, 20.0)


def _merge_direct(z, new_z, udf, new_udf):
    """nudf_merge_z into NaN-filled outputs (ops.merge_z allocates uninitialised ones)"""
    N, n = z.shape
    m = new_z.shape[1]
    z_out = torch.full((N, n + m), float("nan"), device=DEV)
    udf_out = torch.full((N, n + m), float("nan"), device=DEV)
    L.check(L.lib().nudf_merge_z(L.ptr(z), L.ptr(new_z), L.ptr(udf), L.ptr(new_udf), N, n, m, L.ptr(z_out), L.ptr(udf_out),
                                 L.stream_ptr()), "nudf_merge_z")
    return z_out, udf_out


# (n old, m new, N rays): n + m below, at and past the 256-thread block, m = 1
MERGE_CASES = [(1, 1, 7), (2, 1, 33), (64, 50, 19), (200, 56, 5), (255, 1, 9), (256, 1, 9), (128, 129, 11), (1000, 600, 3)]


@pytest.mark.parametrize("n,m,N", MERGE_CASES)
def test_merge_z_ties(n, m, N):
    """Half of the new values repeat old ones exactly, and new values repeat among themselves.  z must equal
    torch.sort(cat) bit for bit, every slot be written once, and the gathered udf equal the oracle's gather (tied z carry
    equal udf here).  The tie order is old before new: at equal z, the old sample takes the lower slot -- merge_z_kernel
    counts new values strictly below an old one, and old values at or below a new one."""
    g = torch.Generator().manual_seed(n * 1000 + m)
    z = torch.sort(torch.rand(N, n, generator=g) * 4.0 + 0.5, dim=1).values
    fresh = torch.rand(N, m, generator=g) * 4.0 + 0.5
    pick = torch.gather(z, 1, torch.randint(0, n, (N, m), generator=g))
    new = torch.where(torch.rand(N, m, generator=g) < 0.5, pick, fresh)
    dup = torch.rand(N, m, generator=g) < 0.3                     # repeats inside new_z
    new = torch.where(dup, torch.roll(new, 1, dims=1), new)
    new = torch.sort(new, dim=1).values.contiguous()
    assert m == 1 or bool((new[:, 1:] == new[:, :-1]).any()), "no repeated new values"
    assert bool((new[:, :, None] == z[:, None, :]).any()), "no new value equals an old one"
    fz = lambda t: torch.sin(7.0 * t) + 2.0                        # equal z -> equal udf
    zd, nd = z.to(DEV), new.to(DEV)
    z_out, udf_out = _merge_direct(zd, nd, fz(z).to(DEV), fz(new).to(DEV))
    assert not bool(torch.isnan(z_out).any()) and not bool(torch.isnan(udf_out).any()), "an output slot was not written"
    zs, index = O.merge_z(z, new)
    assert torch.equal(z_out.cpu(), zs), "merged z differs from torch.sort(cat)"
    assert torch.equal(udf_out.cpu(), torch.gather(torch.cat([fz(z), fz(new)], 1), 1, index))
    # the library wrapper gives the same bits
    z2, u2 = ops.merge_z(zd, nd, fz(z).to(DEV), fz(new).to(DEV))
    assert torch.equal(z2, z_out) and torch.equal(u2, udf_out)
    # tie order: mark old samples 0, new samples 1; within a run of equal z the marks never decrease
    _, mark = _merge_direct(zd, nd, torch.zeros(N, n, device=DEV), torch.ones(N, m, device=DEV))
    same = z_out[:, 1:] == z_out[:, :-1]
    assert int(same.sum()) > 0
    assert bool((mark[:, 1:][same] >= mark[:, :-1][same]).all()), "a new sample precedes an equal old one"
    assert int(mark.sum()) == N * m


@pytest.mark.parametrize("n", [1, 9])
def test_point_kernels_edges(n):
    """ray_points and points_on_rays at S = 1 (and 9), outside_points at col0 = n - 1 (and 0): the first two bit for bit
    against a CPU multiply-then-add, outside_points within a few ulps of fp64 (its norm may be contracted)"""
    N = 37
    o, d, near, far = _rays(N, 11 + n)
    z = (near + (far - near) * torch.linspace(0.0, 1.0, n)[None, :] * 4.0).float().contiguous()
    sd = 0.0173
    dv = lambda t: t.to(DEV)
    pts, mid, dists = ops.ray_points(dv(o), dv(d), dv(z), sd)
    dist_ref = torch.cat([z[:, 1:] - z[:, :-1], torch.full((N, 1), sd)], 1)
    mid_ref = z + dist_ref * 0.5
    pts_ref = o[:, None, :] + d[:, None, :] * mid_ref[..., None]
    assert torch.equal(dists.cpu(), dist_ref) and torch.equal(mid.cpu(), mid_ref)
    assert torch.equal(pts.cpu(), pts_ref.reshape(-1, 3))
    por = ops.points_on_rays(dv(o), dv(d), dv(z))
    assert torch.equal(por.cpu(), (o[:, None, :] + d[:, None, :] * z[..., None]).reshape(-1, 3))
    for col0 in sorted({0, n - 1}):
        pts4, od = ops.outside_points(dv(o), dv(d), dv(z), col0, sd)
        p = pts_ref[:, col0:].double()
        rr = p.norm(dim=-1, keepdim=True).clamp(1.0, 1e10)
        ref = torch.cat([p / rr, 1.0 / rr], -1).reshape(-1, 4)
        assert torch.equal(od.cpu(), dist_ref[:, col0:])
        ulp = 2.0 ** -23 * ref.abs().clamp(min=2.0 ** -10)
        e = float(((pts4.cpu().double() - ref).abs() / ulp).max())
        report("ray_shapes.outside_points[n%d,col0%d]" % (n, col0), max_ulps=e)
        assert e <= 4.0, e
        if col0 == 0 and n > 1:
            assert float(rr.max()) > 1.0 and float(rr.min()) == 1.0      # both sides of the clamp


# ---------------------------------------------------------------------------------------------------------------
# C. sampling schedules end to end, golden scene networks
# ---------------------------------------------------------------------------------------------------------------
# (n_samples, n_importance, up_sample_steps, n_outside, upsampling_type, rays, branch)
SCHEDULES = {
    "dtu1": (64, 50, 1, 32, "classical", 64, "the conf's documented alternative: one round of m = 50"),
    "wide": (128, 256, 4, 32, "classical", 32, "S + O = 416: composite above 48 KB"),
    "mix60": (64, 240, 3, 0, "mix", 32, "mix schedule, m = 60 per round"),
    "dense": (512, 512, 1, 0, "classical", 16, "up-sampling n = 512 above 48 KB; S = 1024"),
}
FIXED_Z = ("wide", "dense")


def _oracle_fine(g, o, d, z, z_out, sd, n_outside, dt):
    """render_core of the oracle (after sampling) on given z, with the NeRF++ background of render()"""
    up, cp = oracle_params(g, "udf", dt), oracle_params(g, "color", dt)
    sc = {k: v.to(dt) for k, v in g.params["sc"].items()}
    o, d, z = o.to(dt), d.to(dt), z.to(dt)
    bg_alpha = bg_color = None
    if n_outside > 0:
        np_ = oracle_params(g, "nerf", dt)
        z_feed, _ = torch.sort(torch.cat([z, z_out.to(dt).expand(z.shape[0], -1)], -1), -1)
        ro = O.render_core_outside(lambda a, b: O.nerf_mlp(np_, g.nerf_c, a, b), o, d, z_feed, sd, n_outside)
        bg_alpha, bg_color = ro["alpha"], ro["sampled_color"]
    ret = O.render_core(up, g.udf_c, cp, g.col_c, sc, o, d, z, sd, cos_anneal_ratio=0.7, flip_saturation=0.2,
                        background_alpha=bg_alpha, background_sampled_color=bg_color)
    return {k: v.detach() for k, v in ret.items() if isinstance(v, torch.Tensor)}


@pytest.mark.parametrize("name", list(SCHEDULES))
def test_sampling_schedules_end_to_end(golden, name):
    from neuraludf_b200 import render as R
    from neuraludf_b200.models.udf_renderer_blending import UDFRendererBlending
    S0, n_imp, K, n_out, kind, Nr, why = SCHEDULES[name]
    g = golden
    udf, col, nerf, var, beta = build_modules(g, DEV)
    ren = UDFRendererBlending(nerf, udf, var, col, beta, n_samples=S0, n_importance=n_imp, n_outside=n_out,
                              up_sample_steps=K, perturb=0.0, upsampling_type=kind)
    o, d, near, far = g.t("rays_o")[:Nr], g.t("rays_d")[:Nr], g.t("near")[:Nr], g.t("far")[:Nr]
    tag = "ray_shapes.schedule[%s]" % name
    torch.set_num_threads(min(32, torch.get_num_threads()))
    # ---- 1. importance-sampled z against the oracle, fp64 arbiter and fp32 yardstick ----
    refs = {}
    for dt in (F64, F32):
        p = oracle_params(g, "udf", dt)
        udf_fn = lambda x: O.udf_mlp(p, g.udf_c, x)[:, 0]
        z0, _, sd = O.coarse_z(near.to(dt), far.to(dt), S0, n_out)
        with torch.no_grad():
            if kind == "classical":
                refs[dt] = O.importance_sample(udf_fn, o.to(dt), d.to(dt), z0, sd, n_imp, K)
            else:
                _, b_, g_ = O.scalar_heads({k: v.to(dt) for k, v in g.params["sc"].items()})
                refs[dt] = O.importance_sample_mix(udf_fn, o.to(dt), d.to(dt), z0, sd, n_imp, K, b_, g_)
    sd = ((far - near) / S0).mean().item()
    z0 = (near + (far - near) * torch.linspace(0.0, 1.0, S0)[None, :]).to(DEV).contiguous()
    od, dd = o.to(DEV), d.to(DEV)
    z = ren.importance_sample(od, dd, z0, sd) if kind == "classical" else ren.importance_sample_mix(od, dd, z0, sd)
    ref64, ref32 = refs[F64], refs[F32]
    assert z.shape == ref64.shape == (Nr, S0 + (n_imp // K) * K if kind == "classical" else S0 + (n_imp // (K + 1)) * (K + 1))
    assert bool((z[:, 1:] >= z[:, :-1]).all())
    diff = (z.cpu().double() - ref64).abs()
    frac_bad = float((diff > 1e-4).float().mean())
    ref_bad = float(((ref32.double() - ref64).abs() > 1e-4).float().mean())
    report(tag + ".z", frac_gt_1e4=frac_bad, ref32_frac_gt_1e4=ref_bad, max_abs=float(diff.max()))
    assert frac_bad <= max(2e-3, 3 * ref_bad)
    assert float(diff.max()) <= 3 * float((ref32.double() - ref64).abs().max()) + 1e-4
    # ---- 2. render_view gives render()'s colour and depth bits ----
    nd, fd = near.to(DEV), far.to(DEV)
    with torch.no_grad():
        full = ren.render(od, dd, nd, fd, cos_anneal_ratio=0.7, perturb_overwrite=0)
        view = R.render_view(ren, od.reshape(1, Nr, 3), dd.reshape(1, Nr, 3), nd.reshape(1, Nr, 1), fd.reshape(1, Nr, 1),
                             cos_anneal_ratio=0.7)
    assert torch.equal(view["color"].reshape(Nr, 3), full["color"]), "render_view colour differs from render()"
    assert torch.equal(view["depth"].reshape(Nr, 1), full["depth"]), "render_view depth differs from render()"
    # ---- 3. the fine pass on the oracle's own fp64 z, against the oracle's render_core ----
    if name in FIXED_Z:
        _, z_out, _ = O.coarse_z(near, far, S0, n_out)
        r64 = _oracle_fine(g, o, d, ref64, z_out, sd, n_out, F64)
        r32 = _oracle_fine(g, o, d, ref64.float(), z_out, sd, n_out, F32)
        ret = ren._render_from_z(od, dd, ref64.float().to(DEV).contiguous(), None if z_out is None else z_out.to(DEV), sd,
                                 cos_anneal_ratio=0.7, flip_saturation=0.2)
        for k in ("color", "depth", "weights", "gradient_error"):
            parity(tag + ".fixed_z." + k, ret[k].detach().cpu().reshape(r64[k].shape), r64[k], r32[k], tol=3e-4)
    report(tag, why=why)

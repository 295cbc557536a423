"""The 'theorical' alpha rule of neuraludf_b200/csrc/raymath.cuh (sdf2alpha, :321-323), compiled for the host with g++
(tests/host/theorical_host.cpp) and compared with fp64 autograd of the oracle: per sample (value and the derivatives
in sdf, true_cos and inv_s, including the edges where torch's autograd defines them) and per ray (a whole composite
forward and backward under the rule, over the parameter grid of test_raymath_host.py).  CPU only."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import oracle_theorical as OT
from tests.test_raymath_host import Cfg, fp, make_case

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def lib():
    out = os.path.join(HERE, "host", "_build")
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, "libtheorical_host.so")
    src = os.path.join(HERE, "host", "theorical_host.cpp")
    subprocess.check_call(["g++", "-O1", "-ffp-contract=off", "-shared", "-fPIC", "-o", so, src])
    L = ctypes.CDLL(so)
    L.theorical_sample.argtypes = [ctypes.c_float] * 4 + [ctypes.c_int, ctypes.c_float, ctypes.c_float,
                                                          ctypes.POINTER(ctypes.c_float)]
    return L


def host_sample(lib, sdf, tc, dist, s, r, a_bar=1.0):
    out = (ctypes.c_float * 4)()
    lib.theorical_sample(sdf, tc, dist, s, 0 if r is None else 1, 0.0 if r is None else r, a_bar, out)
    return np.array(out[:], np.float64)


def ref_sample(sdf, tc, dist, s, r, dtype=torch.float64):
    """alpha and d/d(sdf, true_cos, inv_s) of render_core's call (:414-415): sdf2alpha(sdf, -|true_cos|, ...)"""
    leaves = [torch.tensor(v, dtype=dtype, requires_grad=True) for v in (sdf, tc, s)]
    a = OT.theorical_alpha(leaves[0], -leaves[1].abs(), torch.tensor(dist, dtype=dtype), leaves[2], r)
    grads = torch.autograd.grad(a, leaves)
    return np.array([a.item()] + [g.item() for g in grads])


@pytest.mark.parametrize("r", [None, 0.0, 0.35, 1.0])
def test_sample_value_and_derivatives(lib, r):
    g = np.random.default_rng(5)
    n = 0
    for _ in range(400):
        sdf = float(np.float32(g.choice([-1, 1]) * 10 ** g.uniform(-5, 0)))
        tc = float(np.float32(g.uniform(-1.5, 1.5)))
        dist = float(np.float32(10 ** g.uniform(-3, -1)))
        s = float(np.float32(10 ** g.uniform(0.5, 3.5)))
        h = host_sample(lib, sdf, tc, dist, s, r)
        want = ref_sample(sdf, tc, dist, s, r)
        # where 1 - sigmoid(sdf s) rounds to (near) 0 in fp32 the derivatives are set by that rounding, 6e-8 absolute in
        # 1 - sigmoid: allow it, scaled by the largest factor any of the three derivatives puts on it
        floor = 1e-7 * s * dist * max(s, 1.0) * (1.0 + abs(sdf))
        # alpha = 1 - exp(-x) is formed in fp32 as written: a few ulps of 1 absolute, plus the rounding of 1 - sigmoid
        assert np.abs(h[0] - want[0]) <= 4e-7 + 2e-6 * abs(want[0]) + 1.5e-7 * s * dist, (sdf, tc, dist, s, h, want)
        for k in (1, 2, 3):
            assert abs(h[k] - want[k]) <= 5e-5 * abs(want[k]) + floor, (k, sdf, tc, dist, s, h, want)
        n += 1
    assert n == 400


@pytest.mark.parametrize("r", [None, 0.5])
def test_sample_edges(lib, r):
    # true_cos = 0: |iter_cos| is 0 without anneal, so raw == 0: alpha 0 and every derivative 0 (relu'(0) = 0,
    # sign(0) = 0); with anneal iter_cos = -(1 - r)/2 and only d/d true_cos vanishes (relu(-0) and |0|)
    h = host_sample(lib, 0.01, 0.0, 0.01, 400.0, r)
    want = ref_sample(0.01, 0.0, 0.01, 400.0, r)
    assert np.allclose(h, want, rtol=1e-5, atol=0.0), (h, want)
    if r is None:
        assert h.tolist() == [0.0, 0.0, 0.0, 0.0]
    assert h[2] == 0.0 and want[2] == 0.0
    # sdf * inv_s large enough that 1 - sigmoid is exactly 0 in fp32: alpha is exactly 0, as the reference's, and the
    # relu's derivative at raw == 0 is 0
    for sdf, s in ((0.5, 400.0), (20.0, 1.0), (0.06, 3000.0)):
        h = host_sample(lib, sdf, -0.7, 0.02, s, r)
        ref32 = ref_sample(sdf, -0.7, 0.02, s, r, dtype=torch.float32)
        assert ref32[0] == 0.0 and h[0] == 0.0, (sdf, s, h, ref32)
        assert h[1:].tolist() == [0.0, 0.0, 0.0] and ref32[1:].tolist() == [0.0, 0.0, 0.0]
    # the other sign saturates the other way: 1 - sigmoid(-large) = 1 and raw = |ic| s
    h = host_sample(lib, -0.5, -0.7, 0.02, 400.0, None)
    assert abs(h[0] - (1.0 - np.exp(-0.7 * 400.0 * 0.02))) < 1e-6


@pytest.mark.parametrize("S,Oo,has_r,use_norm,bg_rgb,near", [(40, 0, 1, 0, 0, False), (70, 9, 1, 0, 1, True),
                                                               (33, 5, 0, 1, 0, True), (64, 0, 0, 0, 0, True)])
def test_composite_forward_backward(lib, S, Oo, has_r, use_norm, bg_rgb, near):
    c = make_case(3 + S, S, Oo, near)
    N = c["udf"].shape[0]
    inv_s, beta, gamma, r, fs, ssf = 403.4, 148.4, 20.1, 0.35, 0.4, 300.0
    bgv = torch.tensor([0.2, 0.5, 0.9])
    dt = torch.float64
    leaves = {k: c[k].to(dt).clone().requires_grad_(True) for k in ("udf", "grads", "scb", "sc", "bga", "bgc")}
    heads = [torch.tensor(v, dtype=dt, requires_grad=True) for v in (inv_s, beta, gamma)]
    ret = OT.composite(c["d"].to(dt), c["pts"].to(dt), c["mid"].to(dt), c["dists"].to(dt), leaves["udf"],
                       leaves["grads"], leaves["scb"], leaves["sc"], heads[0], heads[1], heads[2],
                       cos_anneal_ratio=r if has_r else None, flip_saturation=fs,
                       background_rgb=bgv.to(dt) if bg_rgb else None,
                       background_alpha=leaves["bga"] if Oo else None,
                       background_sampled_color=leaves["bgc"] if Oo else None, sparse_scale_factor=ssf,
                       use_norm_grad_for_cosine=bool(use_norm), sdf2alpha_type="theorical")
    # the rule is live: the alphas differ from the numerical rule's
    ret_num = OT.composite(c["d"].to(dt), c["pts"].to(dt), c["mid"].to(dt), c["dists"].to(dt), c["udf"].to(dt),
                           c["grads"].to(dt), c["scb"].to(dt), c["sc"].to(dt), inv_s, beta, gamma,
                           cos_anneal_ratio=r if has_r else None, flip_saturation=fs, sparse_scale_factor=ssf,
                           use_norm_grad_for_cosine=bool(use_norm))
    assert (ret_num["alpha_plus"] - ret["alpha_plus"].detach()).abs().max() > 1e-3
    gen = torch.Generator().manual_seed(99)
    bars = {k: torch.randn(ret[k].shape, generator=gen, dtype=dt) for k in
            ("color_base", "color", "depth", "weight_sum", "weight_sum_fg_bg")}
    sb = torch.randn(3, generator=gen, dtype=dt)
    loss = sum((ret[k] * bars[k]).sum() for k in bars) + sb[0] * ret["gradient_error"] \
        + sb[1] * ret["gradient_error_near_surface"] + sb[2] * ret["sparse_error"]
    wanted = [leaves["udf"], leaves["grads"], leaves["scb"], leaves["sc"]] + heads + \
        ([leaves["bga"], leaves["bgc"]] if Oo else [])
    gr = torch.autograd.grad(loss, wanted)
    cfg = Cfg(S, Oo, inv_s, beta, gamma, r, has_r, fs, ssf, use_norm, bg_rgb, (ctypes.c_float * 3)(*bgv.tolist()))
    f32 = lambda t: np.ascontiguousarray(t.detach().float().numpy())
    outs = np.zeros((N, 14), np.float32)
    W = np.zeros((N, S + Oo), np.float32)
    arr = {k: f32(c[k]) for k in ("d", "pts", "mid", "dists", "udf", "grads", "scb", "sc", "bga", "bgc")}
    for i in range(N):
        lib.ray_forward_host(ctypes.byref(cfg), fp(arr["d"][i]), fp(arr["pts"][i]), fp(arr["mid"][i]), fp(arr["dists"][i]),
                             fp(arr["udf"][i]), fp(arr["grads"][i]), fp(arr["scb"][i]), fp(arr["sc"][i]), fp(arr["bga"][i]),
                             fp(arr["bgc"][i]), fp(outs[i]), fp(W[i]))

    def close(a, b, tol, name):
        a = np.asarray(a, np.float64)
        b = np.asarray(b.detach().numpy(), np.float64)
        err = np.abs(a - b).max() / (np.abs(b).max() + 1e-30)
        assert err < tol, (name, err)

    close(outs[:, 0:3], ret["color_base"], 2e-4, "color_base")
    close(outs[:, 3:6], ret["color"], 2e-4, "color")
    close(outs[:, 6:7], ret["depth"], 2e-4, "depth")
    close(outs[:, 7:8], ret["weight_sum"], 2e-4, "ws")
    close(outs[:, 8:9], ret["weight_sum_fg_bg"], 2e-4, "ws_all")
    close(W, ret["weights"], 2e-4, "weights")
    relax_sum, near_sum = outs[:, 10].sum(), outs[:, 12].sum()
    coef = np.array([sb[0] / (relax_sum + 1e-5), sb[1] / (near_sum + 1e-5), sb[2] / N], np.float32)
    ub = np.zeros((N, S), np.float32)
    gb = np.zeros((N, S, 3), np.float32)
    scbb = np.zeros((N, S, 3), np.float32)
    scb_ = np.zeros((N, S, 3), np.float32)
    bab = np.zeros((N, S + Oo), np.float32)
    bcb = np.zeros((N, S + Oo, 3), np.float32)
    scal = np.zeros((N, 3), np.float32)
    for i in range(N):
        bar = np.concatenate([f32(bars["color_base"][i]), f32(bars["color"][i]), f32(bars["depth"][i]),
                              f32(bars["weight_sum"][i]), f32(bars["weight_sum_fg_bg"][i])]).astype(np.float32)
        lib.ray_backward_host(ctypes.byref(cfg), fp(arr["d"][i]), fp(arr["pts"][i]), fp(arr["mid"][i]), fp(arr["dists"][i]),
                              fp(arr["udf"][i]), fp(arr["grads"][i]), fp(arr["scb"][i]), fp(arr["sc"][i]),
                              fp(arr["bga"][i]), fp(arr["bgc"][i]), fp(bar), fp(coef), fp(ub[i]), fp(gb[i]), fp(scbb[i]),
                              fp(scb_[i]), fp(bab[i]), fp(bcb[i]), fp(scal[i]))
    tol = 2e-3
    close(ub, gr[0], tol, "udf_bar")
    close(gb, gr[1], tol, "grads_bar")
    close(scbb, gr[2], tol, "scb_bar")
    close(scb_, gr[3], tol, "sc_bar")
    close(scal[:, 0].sum(), gr[4], tol, "inv_s_bar")
    close(scal[:, 1].sum(), gr[5], tol, "beta_bar")
    close(scal[:, 2].sum(), gr[6], tol, "gamma_bar")
    if Oo:
        close(bab[:, S:], gr[7][:, S:], tol, "bg_alpha_bar")
        close(bcb[:, S:], gr[8][:, S:], tol, "bg_color_bar")

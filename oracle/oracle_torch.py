"""CPU oracle for the NeuralUDF volume-rendering hot path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

A functional (stateless) PyTorch restatement of the reference algorithm, written from the maths in
SURVEY.md App. A.  It is the checker for the CUDA path: only `tests/`, `__graft_entry__.smoke()` and
`bench.py`'s `cpu_baseline` / `--impl reference` legs may import it.  The product path
(`neuraludf_b200/`) never does, and fails loudly when its CUDA library is missing.

Pinning: the reference has no tests and no golden vectors (SURVEY.md 8(c)), so this restatement is
pinned against outputs of the UNMODIFIED reference code run in the dev container -- see
`oracle/make_golden.py` (generator) and `tests/test_oracle_pinned.py` (fixtures under
`tests/golden/`, plus a live comparison whenever /root/reference is present).

Every function cites the reference lines it follows (paths relative to the reference root).
All functions are dtype-generic: feed float64 tensors to obtain the fp64 arbiter of SURVEY 8(c).
Parameters are plain dicts keyed by the reference's `state_dict()` names.
"""
import math

import torch
import torch.nn.functional as F

# scene / shape generators live in the (kernel-free) product utility module so that bench.py's CUDA arm does not
# import the oracle; re-exported here for the tests.
from neuraludf_b200.synthetic import (color_cfg, make_blend_views, make_color_params,  # noqa: E402,F401
                                      make_nerf_params, make_rays, make_scalars, make_udf_params, nerf_cfg, udf_cfg)


def to_dtype(params, dtype):
    return {k: v.to(dtype) for k, v in params.items()}


# ----------------------------------------------------------------------------------------------
# a1: positional encoding, models/embedder.py:11-36 ----------------------------------------------
# ----------------------------------------------------------------------------------------------

def positional_encoding(x, n_freqs):
    """[x | sin(2^0 x) | cos(2^0 x) | sin(2^1 x) | ...], each block as wide as x."""
    if n_freqs <= 0:
        return x
    out = [x]
    for k in range(n_freqs):
        f = 2.0 ** k
        out.append(torch.sin(x * f))
        out.append(torch.cos(x * f))
    return torch.cat(out, dim=-1)


def fold_weight_norm(g, v):
    """legacy nn.utils.weight_norm, dim=0: W = g * v / ||v||_2 (per output row); the same ATen primitive the
    reference's modules call, so fp32 results agree bit-for-bit."""
    return torch._weight_norm(v, g, 0)


def softplus100(z):
    """nn.Softplus(beta=100), threshold 20 (models/fields.py:180)."""
    return F.softplus(z, beta=100.0)


# ----------------------------------------------------------------------------------------------
# a2/a3: UDF network, models/fields.py:192-231 ---------------------------------------------------
# ----------------------------------------------------------------------------------------------

def udf_mlp_raw(p, cfg, x):
    """Returns the raw last-layer output y [P, d_out] BEFORE abs (y[:,0] is the signed value)."""
    inp = x * cfg["scale"]
    e = positional_encoding(inp, cfg["multires"])
    h = e
    n_lin = len(cfg["layers"])
    for l in range(n_lin):
        if l in cfg["skip_in"]:
            h = torch.cat([h, e], dim=1) / math.sqrt(2)
        w = fold_weight_norm(p["lin%d.weight_g" % l], p["lin%d.weight_v" % l])
        h = F.linear(h, w, p["lin%d.bias" % l])
        if l < n_lin - 1:
            h = softplus100(h)
    return h


def udf_out(y0, cfg):
    t = cfg["udf_type"]
    if t == "abs":
        return y0.abs()
    if t == "square":
        return y0 ** 2
    return y0


def udf_mlp(p, cfg, x):
    """UDFNetwork.forward: cat(udf_out(y0)/scale, y[1:]) (models/fields.py:210)."""
    y = udf_mlp_raw(p, cfg, x)
    return torch.cat([udf_out(y[:, :1], cfg) / cfg["scale"], y[:, 1:]], dim=-1)


def udf_gradient_autograd(p, cfg, x, create_graph=True):
    """UDFNetwork.gradient (models/fields.py:219-231): exact d udf / d x by autograd."""
    x = x.detach().requires_grad_(True)
    with torch.enable_grad():
        y = udf_mlp(p, cfg, x)[:, :1]
        g = torch.autograd.grad(y, x, torch.ones_like(y), create_graph=create_graph,
                                retain_graph=True)[0]
    return g


def udf_value_and_gradient_analytic(p, cfg, x):
    """Same quantities by the hand-written reverse sweep of SURVEY App. A (what the CUDA path does).
    Returns (out [P,d_out], grad [P,3]).  Not differentiable; used to validate the derivation."""
    assert cfg["udf_type"] == "abs"
    scale = cfg["scale"]
    inp = x * scale
    L = cfg["multires"]
    e = positional_encoding(inp, L)
    n_lin = len(cfg["layers"])
    ws, acts = [], []
    h = e
    for l in range(n_lin):
        if l in cfg["skip_in"]:
            h = torch.cat([h, e], dim=1) / math.sqrt(2)
        w = fold_weight_norm(p["lin%d.weight_g" % l], p["lin%d.weight_v" % l])
        ws.append(w)
        z = F.linear(h, w, p["lin%d.bias" % l])
        if l < n_lin - 1:
            h = softplus100(z)
            acts.append(torch.sigmoid(100.0 * z))
        else:
            h = z
    y = h
    out = torch.cat([y[:, :1].abs() / scale, y[:, 1:]], dim=-1)
    sgn = torch.sign(y[:, :1])
    g = (sgn / scale) * ws[n_lin - 1][0:1, :]            # d udf / d a_last  [P, d_hidden]
    g_pe = torch.zeros_like(e)
    for l in range(n_lin - 2, -1, -1):
        if (l + 1) in cfg["skip_in"]:                    # g is the grad of the concatenated input of layer l+1
            g = g / math.sqrt(2)
            g_pe = g_pe + g[:, -cfg["d_pe"]:]
            g = g[:, :-cfg["d_pe"]]
        d = g * acts[l]
        g = d @ ws[l]
    g_pe = g_pe + g
    d_in = cfg["d_in"]
    grad = g_pe[:, :d_in].clone()
    for k in range(L):
        f = 2.0 ** k
        s_blk = g_pe[:, d_in * (1 + 2 * k): d_in * (2 + 2 * k)]
        c_blk = g_pe[:, d_in * (2 + 2 * k): d_in * (3 + 2 * k)]
        grad = grad + f * (torch.cos(inp * f) * s_blk - torch.sin(inp * f) * c_blk)
    return out, grad * scale


# ----------------------------------------------------------------------------------------------
# a4: ResidualRenderingNetwork (mode no_normal), models/fields.py:452-495 ------------------------
# ----------------------------------------------------------------------------------------------

def color_mlp(p, cfg, pts, view_dirs, feat):
    n_lin = len(cfg["dims"]) - 1
    v = positional_encoding(view_dirs, cfg["multires_view"])
    h = torch.cat([pts, feat], dim=-1)
    x_hidden = None
    for l in range(n_lin):
        w = fold_weight_norm(p["lin_base%d.weight_g" % l], p["lin_base%d.weight_v" % l])
        h = F.linear(h, w, p["lin_base%d.bias" % l])
        if l < n_lin - 1:
            h = F.relu(h)
        if l == n_lin - 2:
            x_hidden = h
    color_base = torch.sigmoid(h[:, :cfg["d_out"]])
    h = torch.cat([v, color_base, x_hidden], dim=-1)
    for l in range(n_lin):
        w = fold_weight_norm(p["lin%d.weight_g" % l], p["lin%d.weight_v" % l])
        h = F.linear(h, w, p["lin%d.bias" % l])
        if l < n_lin - 1:
            h = F.relu(h)
    color = torch.sigmoid(h[:, :cfg["d_out"]])
    return color_base, color, h[:, cfg["d_out"]:]


# ----------------------------------------------------------------------------------------------
# a5: NeRF++ background network, models/fields.py:599-628 ----------------------------------------
# ----------------------------------------------------------------------------------------------

def nerf_mlp(p, cfg, pts, views):
    e = positional_encoding(pts, cfg["multires"])
    ev = positional_encoding(views, cfg["multires_view"])
    h = e
    for i in range(cfg["D"]):
        h = F.relu(F.linear(h, p["pts_linears.%d.weight" % i], p["pts_linears.%d.bias" % i]))
        if i in cfg["skips"]:
            h = torch.cat([e, h], dim=-1)
    alpha = F.linear(h, p["alpha_linear.weight"], p["alpha_linear.bias"])
    feat = F.linear(h, p["feature_linear.weight"], p["feature_linear.bias"])
    h = torch.cat([feat, ev], dim=-1)
    h = F.relu(F.linear(h, p["views_linears.0.weight"], p["views_linears.0.bias"]))
    rgb = F.linear(h, p["rgb_linear.weight"], p["rgb_linear.bias"])
    return alpha, rgb


# ----------------------------------------------------------------------------------------------
# a6: scalar heads -------------------------------------------------------------------------------
# ----------------------------------------------------------------------------------------------

def scalar_heads(sc, beta_min=5e-5):
    """inv_s = exp(10 variance) (fields.py:655); beta = clip(exp(10 b), 0, 1/beta_min) (:675);
    gamma = exp(10 g) (:678); then render_core clips all to [1e-6, 1e6] (udf_renderer_blending.py:373-377)."""
    inv_s = torch.exp(sc["variance"] * 10.0).clip(1e-6, 1e6)
    beta = torch.exp(sc["beta"] * 10.0).clip(0, 1.0 / beta_min).clip(1e-6, 1e6)
    gamma = torch.exp(sc["gamma"] * 10.0).clip(1e-6, 1e6)
    return inv_s, beta, gamma


# ----------------------------------------------------------------------------------------------
# a12: UDF -> density / alpha, models/udf_renderer_blending.py:151-159, 292-325 ------------------
# ----------------------------------------------------------------------------------------------

def logistic_density(udf, inv_s, gamma=1.0, abs_cos=1.0):
    e = torch.exp(-inv_s * udf)
    return abs_cos * inv_s * e / (1 + e) ** 2 * gamma


def neus_alpha(sdf, true_cos, dists, inv_s, cos_anneal_ratio=None):
    """'numerical' branch of sdf2alpha (:308-320)."""
    if cos_anneal_ratio is not None:
        iter_cos = -(F.relu(-true_cos * 0.5 + 0.5) * (1.0 - cos_anneal_ratio)
                     + F.relu(-true_cos) * cos_anneal_ratio)
    else:
        iter_cos = true_cos
    nxt = sdf + iter_cos * dists * 0.5
    prv = sdf - iter_cos * dists * 0.5
    c_prev = torch.sigmoid(prv * inv_s)
    c_next = torch.sigmoid(nxt * inv_s)
    return ((c_prev - c_next + 1e-5) / (c_prev + 1e-5)).clip(0.0, 1.0)


def exclusive_cumprod(t):
    """cumprod(cat([1, t]))[:, :-1] -- the transmittance pattern used at :249-251, :261-262, :407-410, :508."""
    ones = torch.ones_like(t[:, :1])
    return torch.cumprod(torch.cat([ones, t], dim=-1), dim=-1)[:, :-1]


# ----------------------------------------------------------------------------------------------
# a9: inverse-CDF sampling, models/udf_renderer_blending.py:66-104 (det=True only) ---------------
# ----------------------------------------------------------------------------------------------

def sample_pdf_det(bins, weights, n_samples, return_inds=False, trace=None):
    """trace: a list that receives dict(weights, cdf, u, inds) of the call (the cdf the indices were searched in)."""
    raw_weights = weights
    weights = weights + 1e-5
    pdf = weights / torch.sum(weights, -1, keepdim=True)
    cdf = torch.cumsum(pdf, -1)
    cdf = torch.cat([torch.zeros_like(cdf[..., :1]), cdf], -1)
    u = torch.linspace(0.0 + 0.5 / n_samples, 1.0 - 0.5 / n_samples, steps=n_samples,
                       dtype=cdf.dtype, device=cdf.device)
    u = u.expand(list(cdf.shape[:-1]) + [n_samples]).contiguous()
    inds = torch.searchsorted(cdf, u, right=True)
    below = (inds - 1).clamp(min=0)
    above = inds.clamp(max=cdf.shape[-1] - 1)
    c0, c1 = torch.gather(cdf, 1, below), torch.gather(cdf, 1, above)
    b0, b1 = torch.gather(bins, 1, below), torch.gather(bins, 1, above)
    denom = c1 - c0
    denom = torch.where(denom < 1e-5, torch.ones_like(denom), denom)
    t = (u - c0) / denom
    samples = b0 + t * (b1 - b0)
    if trace is not None:
        trace.append(dict(weights=raw_weights.detach().clone(), cdf=cdf.detach().clone(), u=u[:1].clone(),
                          inds=inds.clone()))
    if return_inds:
        return samples, inds
    return samples


# ----------------------------------------------------------------------------------------------
# a8/a11/a10: up-sampling rounds, models/udf_renderer_blending.py:197-290, 834-866 ---------------
# ----------------------------------------------------------------------------------------------

def _append_last(t, value):
    return torch.cat([t, torch.full_like(t[..., :1], value)], dim=-1)


def up_sample_unbias(o, d, z, udf, sample_dist, n_importance, inv_s, beta, gamma, return_inds=False, trace=None):
    """trace: as sample_pdf_det."""
    n_rays, n = z.shape
    pts = o[:, None, :] + d[:, None, :] * z[..., :, None]
    radius = torch.linalg.norm(pts, ord=2, dim=-1)
    inside = (radius[:, :-1] < 1.0) | (radius[:, 1:] < 1.0)
    dists_raw = _append_last(z[..., 1:] - z[..., :-1], sample_dist)
    mid_udf = (udf[:, :-1] + udf[:, 1:]) * 0.5
    dists = z[:, 1:] - z[:, :-1]
    true_cos = (udf[:, 1:] - udf[:, :-1]) / (z[:, 1:] - z[:, :-1] + 1e-5)
    cos_val = -1 * true_cos.abs()
    prev_cos = torch.cat([torch.zeros_like(cos_val[:, :1]), cos_val[:, :-1]], dim=-1)
    cos_val = torch.minimum(prev_cos, cos_val)
    cos_val = cos_val.clip(-1e3, 0.0) * inside
    vis_mask = (true_cos < 0.05).to(z.dtype)
    vis_mask = torch.cat([torch.ones_like(vis_mask[:, :1]), vis_mask], dim=-1)
    raw_occ = logistic_density(udf, beta, 1.0, 1.0)
    alpha_occ = 1.0 - torch.exp(-F.relu(raw_occ) * gamma * dists_raw)
    vis_prob = exclusive_cumprod((1.0 - alpha_occ + vis_mask).clip(0, 1) + 1e-7)
    signs = vis_prob[:, :-1]
    a_plus = neus_alpha(mid_udf, cos_val, dists, inv_s)
    a_minus = neus_alpha(-mid_udf, cos_val, dists, inv_s)
    alpha = a_plus * signs + a_minus * (1 - signs)
    weights = alpha * exclusive_cumprod(1.0 - alpha + 1e-7)
    return sample_pdf_det(z, weights, n_importance, return_inds=return_inds, trace=trace)


def up_sample_no_occ_aware(o, d, z, udf, sample_dist, n_importance, beta, gamma, return_inds=False, trace=None):
    """:834-866 -- note the reference passes (inv_s, beta, gamma) but only beta/gamma are used.  trace: as sample_pdf_det."""
    dists = _append_last(z[..., 1:] - z[..., :-1], sample_dist)
    raw_occ = logistic_density(udf, beta, gamma, 1.0)
    alpha_occ = 1.0 - torch.exp(-F.relu(raw_occ) * dists)
    return sample_pdf_det(z, alpha_occ[:, :-1], n_importance, return_inds=return_inds, trace=trace)


def merge_z(z, new_z):
    """cat + sort of cat_z_vals (:278-279); returns sorted z and the permutation."""
    return torch.sort(torch.cat([z, new_z], dim=-1), dim=-1)


def importance_sample(udf_fn, o, d, z, sample_dist, n_importance, up_sample_steps, trace=None):
    """'classical' schedule, :723-755.  udf_fn maps [P,3] points to [P] udf values."""
    n_rays = o.shape[0]
    pts = o[:, None, :] + d[:, None, :] * z[..., :, None]
    udf = udf_fn(pts.reshape(-1, 3)).reshape(n_rays, -1)
    m = n_importance // up_sample_steps
    for i in range(up_sample_steps):
        gamma = float(min(max(20 * 2 ** (up_sample_steps - i), 20), 320))
        new_z, inds = up_sample_unbias(o, d, z, udf, sample_dist, m, 64 * 2 ** i, 64 * 2 ** (i + 1),
                                       gamma, return_inds=True)
        if trace is not None:
            trace.append(dict(z=z.clone(), udf=udf.clone(), new_z=new_z.clone(), inds=inds.clone()))
        last = (i + 1 == up_sample_steps)
        zs, index = merge_z(z, new_z)
        if not last:
            npts = o[:, None, :] + d[:, None, :] * new_z[..., :, None]
            new_udf = udf_fn(npts.reshape(-1, 3)).reshape(n_rays, -1)
            udf = torch.gather(torch.cat([udf, new_udf], dim=-1), 1, index)
        z = zs
    return z


def importance_sample_mix(udf_fn, o, d, z, sample_dist, n_importance, up_sample_steps, beta, gamma):
    """'mix' schedule, :762-832: K no-occlusion rounds then one unbiased round."""
    n_rays = o.shape[0]
    pts = o[:, None, :] + d[:, None, :] * z[..., :, None]
    udf = udf_fn(pts.reshape(-1, 3)).reshape(n_rays, -1)
    m = n_importance // (up_sample_steps + 1)

    def add(z, udf, new_z, last):
        zs, index = merge_z(z, new_z)
        if not last:
            npts = o[:, None, :] + d[:, None, :] * new_z[..., :, None]
            new_udf = udf_fn(npts.reshape(-1, 3)).reshape(n_rays, -1)
            udf = torch.gather(torch.cat([udf, new_udf], dim=-1), 1, index)
        return zs, udf

    for i in range(up_sample_steps):
        new_z = up_sample_no_occ_aware(o, d, z, udf, sample_dist, m, 64 * 2 ** (i + 1), gamma)
        z, udf = add(z, udf, new_z, False)
    i = up_sample_steps - 1
    new_z = up_sample_unbias(o, d, z, udf, sample_dist, m, 64 * 2 ** i, 64 * 2 ** (i + 1),
                             20.0 if i < 4 else 10.0)
    z, udf = add(z, udf, new_z, True)
    return z


# ----------------------------------------------------------------------------------------------
# a14: NeRF++ outside pass, models/udf_renderer_blending.py:161-195 -------------------------------
# ----------------------------------------------------------------------------------------------

def render_core_outside(nerf_fn, o, d, z, sample_dist, n_outside):
    n_rays, n = z.shape
    dists = _append_last(z[..., 1:] - z[..., :-1], sample_dist)
    mid = z + dists * 0.5
    pts = o[:, None, :] + d[:, None, :] * mid[..., :, None]
    if n_outside > 0:
        r = torch.linalg.norm(pts, ord=2, dim=-1, keepdim=True).clip(1.0, 1e10)
        pts = torch.cat([pts / r, 1.0 / r], dim=-1)
    dirs = d[:, None, :].expand(n_rays, n, 3)
    raw, rgb = nerf_fn(pts.reshape(-1, pts.shape[-1]), dirs.reshape(-1, 3))
    alpha = 1.0 - torch.exp(-F.relu(raw.reshape(n_rays, n)) * dists)
    return dict(sampled_color=rgb.reshape(n_rays, n, 3), alpha=alpha)


# ----------------------------------------------------------------------------------------------
# a13: render_core, models/udf_renderer_blending.py:327-584 (blending branch: a16 below) ----------
# ----------------------------------------------------------------------------------------------

def composite(d, pts, mid, dists, udf, grads, scb, sc_, inv_s, beta, gamma, cos_anneal_ratio=None,
              flip_saturation=0.0, background_rgb=None, background_alpha=None, background_sampled_color=None,
              sparse_scale_factor=25000.0, use_norm_grad_for_cosine=False):
    """Everything of render_core after the networks (:370-553): udf [N,S], grads [N,S,3], sampled colours
    [N,S,3] x2, scalar heads already clipped.  Differentiable w.r.t. all floating inputs."""
    n_rays, n = udf.shape
    dirs = d[:, None, :].expand(n_rays, n, 3)
    g_mag = torch.linalg.norm(grads, ord=2, dim=-1, keepdim=True)
    g_norm = grads / (g_mag + 1e-5)
    true_cos = (dirs * (g_norm if use_norm_grad_for_cosine else grads)).sum(-1)
    with torch.no_grad():
        flip = -torch.sign((dirs * g_norm).sum(-1, keepdim=True))
        flip[flip == 0] = 1
    raw_occ = logistic_density(udf, beta, 1.0, 1.0)
    alpha_occ = 1.0 - torch.exp(-F.relu(raw_occ) * gamma * dists)
    vm = (true_cos < 0.01).to(udf.dtype)
    vm = torch.cat([vm[:, 1:], torch.ones_like(vm[:, :1])], dim=-1)
    vis_prob = exclusive_cumprod((1.0 - alpha_occ + flip_saturation * vm).clip(0, 1) + 1e-7).clip(0, 1)
    a_plus = neus_alpha(udf, -true_cos.abs(), dists, inv_s, cos_anneal_ratio)
    a_minus = neus_alpha(-udf, -true_cos.abs(), dists, inv_s, cos_anneal_ratio)
    alpha = a_plus * vis_prob + a_minus * (1 - vis_prob)
    pn = torch.linalg.norm(pts.reshape(n_rays, n, 3), ord=2, dim=-1)
    inside = (pn < 1.0).to(udf.dtype)
    relax = (pn < 1.2).to(udf.dtype)
    near_surface = (udf < 0.05).to(udf.dtype).detach()
    alpha_fg = alpha
    cb, c = scb, sc_
    if background_alpha is not None:
        alpha = torch.cat([alpha, background_alpha[:, n:]], dim=-1)
        cb = torch.cat([cb, background_sampled_color[:, n:]], dim=1)
        c = torch.cat([c, background_sampled_color[:, n:]], dim=1)
    weights = alpha * exclusive_cumprod(1.0 - alpha + 1e-7)
    wsum = weights.sum(dim=-1, keepdim=True)
    color_base = (cb * weights[:, :, None]).sum(dim=1)
    color = (c * weights[:, :, None]).sum(dim=1)
    depth = (mid * weights[:, :n]).sum(dim=1, keepdim=True)
    if background_rgb is not None:
        color = color + background_rgb * (1.0 - wsum)
    ge = (torch.linalg.norm(grads, ord=2, dim=-1) - 1.0) ** 2
    gradient_error = (relax * ge).sum() / (relax.sum() + 1e-5)
    gradient_error_ns = (near_surface * ge).sum() / (near_surface.sum() + 1e-5)
    g_flip = flip * grads
    sparse_error = torch.exp(-sparse_scale_factor * udf).sum(dim=1).mean()
    return {
        "color_base": color_base, "color": color, "weights": weights, "depth": depth,
        "gradient_error": gradient_error, "gradient_error_near_surface": gradient_error_ns,
        "normals": (g_flip * weights[:, :n, None]).sum(dim=1), "gradients": grads,
        "gradients_flip": g_flip, "inside_sphere": inside, "udf": udf,
        "gradient_mag": g_mag.reshape(n_rays, n), "true_cos": true_cos,
        "vis_prob": vis_prob, "alpha": alpha_fg, "alpha_plus": a_plus, "alpha_minus": a_minus,
        "mid_z_vals": mid, "dists": dists, "sparse_error": sparse_error, "alpha_occ": alpha_occ,
        "raw_occ": raw_occ, "sampled_color_base": scb, "sampled_color": sc_,
        "weight_sum": weights[:, :n].sum(dim=-1, keepdim=True), "weight_sum_fg_bg": wsum,
    }


def render_core(udf_p, udf_c, col_p, col_c, sc, o, d, z, sample_dist, cos_anneal_ratio=None,
                background_rgb=None, background_alpha=None, background_sampled_color=None,
                flip_saturation=0.0, sparse_scale_factor=25000.0, use_norm_grad_for_cosine=False,
                beta_min=5e-5, blending=None):
    """blending: None or dict(color_maps, w2cs, intrinsics, query_c2w, rays_uv) (rays_uv may be None)."""
    n_rays, n = z.shape
    dists = _append_last(z[..., 1:] - z[..., :-1], sample_dist)
    mid = z + dists * 0.5
    pts = (o[:, None, :] + d[:, None, :] * mid[..., :, None]).reshape(-1, 3)
    dirs = d[:, None, :].expand(n_rays, n, 3).reshape(-1, 3)

    pts_g = pts.detach().requires_grad_(True)
    with torch.enable_grad():
        out = udf_mlp(udf_p, udf_c, pts_g)
        udf = out[:, :1]
        feat = out[:, 1:]
        # the reference re-runs the forward inside gradient(); the values are identical
        grads = torch.autograd.grad(udf, pts_g, torch.ones_like(udf), create_graph=True,
                                    retain_graph=True)[0]
    inv_s, beta, gamma = scalar_heads(sc, beta_min)
    cb, c, blend = color_mlp(col_p, col_c, pts_g, dirs, feat)
    ret = composite(d, pts, mid, dists, udf.reshape(n_rays, n), grads.reshape(n_rays, n, 3),
                    cb.reshape(n_rays, n, 3), c.reshape(n_rays, n, 3), inv_s, beta, gamma,
                    cos_anneal_ratio=cos_anneal_ratio, flip_saturation=flip_saturation,
                    background_rgb=background_rgb, background_alpha=background_alpha,
                    background_sampled_color=background_sampled_color,
                    sparse_scale_factor=sparse_scale_factor,
                    use_norm_grad_for_cosine=use_norm_grad_for_cosine)
    ret["s_val"] = 1.0 / inv_s.reshape(1, 1).expand(n_rays * n, 1)
    ret["beta"] = 1.0 / beta
    ret["gamma"] = gamma
    ret["blending_weights"] = blend.reshape(n_rays, n, -1)
    if blending is not None:
        ret.update(blend_outputs(ret, pts, d, blending["color_maps"], blending["w2cs"], blending["intrinsics"],
                                 blending["query_c2w"], blending.get("rays_uv"), background_sampled_color))
    return ret


# ----------------------------------------------------------------------------------------------
# a16: pixel / patch blending of the fine-tuning stage ------------------------------------------
#   models/udf_renderer_blending.py:431-480, 503-524; models/patch_projector.py:21-166;
#   models/projector_utils.py:8-85; models/fields.py:498-537.  Written per source view (V is small).
# ----------------------------------------------------------------------------------------------

def pixel_warp(pts, imgs, intrinsics, w2cs):
    """pts [N,S,3], imgs [V,3,H,W] -> colours [N,S,V,3], in-image mask [N,S,V]  (patch_projector.py:21-43)."""
    n_views, _, h, w = imgs.shape
    cols, masks = [], []
    for v in range(n_views):
        pm = intrinsics[v, :3, :3] @ w2cs[v, :3, :]                       # projector_utils.py:69-70
        cam = pts @ pm[:, :3].T + pm[:, 3]
        zc = cam[..., 2].clamp(min=1e-3)
        gx = 2 * (cam[..., 0] / zc) / (w - 1) - 1
        gy = 2 * (cam[..., 1] / zc) / (h - 1) - 1
        gx = torch.where((gx > 1) | (gx < -1), torch.full_like(gx, 2.0), gx)      # :36-40, padding 'zeros'
        gy = torch.where((gy > 1) | (gy < -1), torch.full_like(gy, 2.0), gy)
        grid = torch.stack([gx, gy], dim=-1)[None]
        masks.append((gx.abs() < 1.0) & (gy.abs() < 1.0))
        cols.append(F.grid_sample(imgs[v:v + 1], grid, padding_mode="zeros", align_corners=True)[0].permute(1, 2, 0))
    return torch.stack(cols, dim=2), torch.stack(masks, dim=2)


def patch_warp(pts, uv, normals, imgs, ref_intrinsic, src_intrinsics, ref_c2w, src_c2ws, h_patch_size=3,
               plane_dist_thresh=0.001):
    """Plane-induced homographies of the reference patch into every source view (patch_projector.py:45-150).
    pts, normals [N,S,3]; uv [N,2] in (-1,1) -> colours [N,S,V,Npx,3], mask [N,S,V,Npx]."""
    normals = normals.detach()                                            # detach_normal=True at the call site (:455)
    n_rays, n_samples, _ = pts.shape
    n_views, _, h, w = imgs.shape
    px = torch.stack([(uv[:, 0] + 1) / 2.0 * (w - 1), (uv[:, 1] + 1) / 2.0 * (h - 1)], dim=-1)
    r = torch.arange(-h_patch_size, h_patch_size + 1, dtype=pts.dtype)
    oy, ox = torch.meshgrid(r, r, indexing="ij")
    offs = torch.stack([ox.reshape(-1), oy.reshape(-1)], dim=-1)          # (dx, dy), dx fastest (:212-214)
    pix = px[:, None, :] + offs[None]                                     # [N,Npx,2]
    hom_pix = torch.cat([pix, torch.ones_like(pix[..., :1])], dim=-1)     # [N,Npx,3]
    k_ref_inv = torch.inverse(ref_intrinsic[:3, :3])
    w2c_ref = torch.inverse(ref_c2w)
    dist_to_cam = torch.linalg.norm(pts - ref_c2w[:3, 3], dim=-1)         # [N,S]
    cols, masks = [], []
    with torch.no_grad():
        n_cam = normals @ w2c_ref[:3, :3].T                               # plane normal in the reference camera frame
        p_cam = pts @ w2c_ref[:3, :3].T + w2c_ref[:3, 3]
        d1 = (n_cam * p_cam).sum(-1)                                      # plane distance to the reference camera
        sgn = torch.sign(d1)
        sgn[sgn == 0] = 1
        d_safe = torch.clamp(d1.abs(), 1e-8) * sgn
    for v in range(n_views):
        with torch.no_grad():
            rel = torch.inverse(src_c2ws[v]) @ ref_c2w
            r_rel, t_rel = rel[:3, :3], rel[:3, 3]
            c_src = -(r_rel.T @ t_rel)                                    # source camera centre in the reference frame
            d2 = (n_cam * c_src).sum(-1)
            ok = (d1.abs() > plane_dist_thresh) & ((d1 - d2).abs() > plane_dist_thresh) & ((d2 / d1) < 1)
            k_src = src_intrinsics[v, :3, :3]
            hom = k_src @ (r_rel + t_rel[:, None] * n_cam[..., None, :] / d_safe[..., None, None]) @ k_ref_inv
            zax = torch.tensor([0.0, 0.0, 1.0], dtype=pts.dtype)
            hom_fp = k_src @ (r_rel + t_rel[:, None] * zax[None, :] / dist_to_cam[..., None, None]) @ k_ref_inv
            hom = torch.where(ok[..., None, None], hom, hom_fp)           # fronto-parallel fallback (:120-129)
        wp = torch.einsum("nsik,npk->nspi", hom, hom_pix)                 # [N,S,Npx,3]
        g = wp[..., :2] / torch.clamp(wp[..., 2:], 1e-8)
        m = (wp[..., 2] > 0) & (g[..., 0] < (w - h_patch_size)) & (g[..., 1] < (h - h_patch_size)) & \
            (g >= h_patch_size).all(dim=-1)
        gn = torch.stack([2 * g[..., 0] / (w - 1) - 1, 2 * g[..., 1] / (h - 1) - 1], dim=-1).clamp(-10, 10)
        c = F.grid_sample(imgs[v:v + 1], gn.reshape(1, -1, 1, 2), align_corners=True)[0, :, :, 0].T
        cols.append(c.reshape(n_rays, n_samples, -1, 3))
        masks.append(m)
    return torch.stack(cols, dim=2), torch.stack(masks, dim=2)


def color_blend(blend_logits, pix_col, pix_mask, pat_col=None, pat_mask=None):
    """Masked-softmax fusion over the source views (fields.py:498-537, img_index=None)."""
    n_views = pix_col.shape[-2]
    sm = torch.softmax(blend_logits[..., :n_views], dim=-1)
    wp = sm * pix_mask
    wp = wp / (wp.sum(dim=-1, keepdim=True) + 1e-8)
    c_pix = (pix_col * wp[..., None]).sum(dim=-2)
    c_pat, m_pat = None, None
    if pat_col is not None:
        full = pat_mask.sum(dim=-1) > pat_col.shape[3] - 1                # every pixel of the patch lands inside
        wq = sm * full
        wq = wq / (wq.sum(dim=-1, keepdim=True) + 1e-8)
        c_pat = (pat_col * wq[..., None, None]).sum(dim=-3)
        m_pat = full.sum(dim=-1) > 0
    return c_pix, c_pat, m_pat


def blend_outputs(ret, pts, d, color_maps, w2cs, intrinsics, query_c2w, rays_uv, background_sampled_color=None,
                  h_patch_size=3):
    """color_pixel / patch_colors / patch_mask of render_core (:431-480, 503-524) from a composite() result."""
    n_rays, n = ret["udf"].shape
    p3 = pts.reshape(n_rays, n, 3)
    pix_col, pix_mask = pixel_warp(p3, color_maps, intrinsics, w2cs)
    pat_col, pat_mask = None, None
    if rays_uv is not None:
        g = ret["gradients"].reshape(n_rays, n, 3).detach()
        gn = g / (torch.linalg.norm(g, ord=2, dim=-1, keepdim=True) + 1e-5)
        flip = -torch.sign((d[:, None, :] * gn).sum(-1, keepdim=True))
        flip[flip == 0] = 1
        pat_col, pat_mask = patch_warp(p3, rays_uv, flip * gn, color_maps, intrinsics[0], intrinsics, query_c2w,
                                       torch.inverse(w2cs), h_patch_size)
    c_pix, c_pat, m_pat = color_blend(ret["blending_weights"], pix_col, pix_mask, pat_col, pat_mask)
    w = ret["weights"]
    if background_sampled_color is not None:
        inside = ret["inside_sphere"][:, :, None]
        c_pix = c_pix * inside + background_sampled_color[:, :n] * (1.0 - inside)
        c_pix = torch.cat([c_pix, background_sampled_color[:, n:]], dim=1)
    out = {"color_pixel": (c_pix * w[:, :c_pix.shape[1], None]).sum(dim=1), "patch_colors": None, "patch_mask": None}
    if c_pat is not None:
        out["patch_colors"] = (c_pat * w[:, :n, None, None]).sum(dim=1)
        out["patch_mask"] = (m_pat.to(w.dtype) * w[:, :n]).sum(dim=1)
    return out


# ----------------------------------------------------------------------------------------------
# a7 + whole render(), models/udf_renderer_blending.py:586-721 (perturb = 0 path) -----------------
# ----------------------------------------------------------------------------------------------

def coarse_z(near, far, n_samples, n_outside):
    """:605-630 with perturb == 0 (RNG-free); returns (z [N,S0], z_outside [N,O] or None, sample_dist)."""
    sample_dist = ((far - near) / n_samples).mean().item()
    t = torch.linspace(0.0, 1.0, n_samples, dtype=near.dtype)
    z = near + (far - near) * t[None, :]
    z_out = None
    if n_outside > 0:
        zo = torch.linspace(1e-3, 1.0 - 1.0 / (n_outside + 1.0), n_outside, dtype=near.dtype)
        z_out = far / torch.flip(zo, dims=[-1]) + 1.0 / n_samples
    return z, z_out, sample_dist


def render(udf_p, udf_c, col_p, col_c, nerf_p, nerf_c, sc, o, d, near, far, n_samples, n_importance,
           n_outside, up_sample_steps, cos_anneal_ratio=None, flip_saturation=0.0,
           upsampling_type="classical", background_rgb=None, **kw):
    z, z_out, sample_dist = coarse_z(near, far, n_samples, n_outside)
    with torch.no_grad():
        udf_fn = lambda x: udf_mlp(udf_p, udf_c, x)[:, 0]
        if n_importance > 0:
            if upsampling_type == "classical":
                z = importance_sample(udf_fn, o, d, z, sample_dist, n_importance, up_sample_steps)
            else:
                _, beta, gamma = scalar_heads(sc)
                z = importance_sample_mix(udf_fn, o, d, z, sample_dist, n_importance, up_sample_steps,
                                          beta, gamma)
    bg_alpha = bg_color = None
    if n_outside > 0:
        z_feed, _ = torch.sort(torch.cat([z, z_out], dim=-1), dim=-1)
        ro = render_core_outside(lambda a, b: nerf_mlp(nerf_p, nerf_c, a, b), o, d, z_feed, sample_dist,
                                 n_outside)
        bg_alpha, bg_color = ro["alpha"], ro["sampled_color"]
    ret = render_core(udf_p, udf_c, col_p, col_c, sc, o, d, z, sample_dist,
                      cos_anneal_ratio=cos_anneal_ratio, background_rgb=background_rgb,
                      background_alpha=bg_alpha, background_sampled_color=bg_color,
                      flip_saturation=flip_saturation, **kw)
    n = z.shape[1]
    ret["z_vals"] = z
    ret["variance"] = ret["s_val"]
    return ret


def training_loss(ret, target_rgb, igr_weight=0.1, color_base_weight=0.01):
    """The fixed scalar used to seed backward in parity tests and in the benchmark:
    L1 colour (loss/loss.py:21-56, mask=None) + igr_weight * eikonal (exp_runner_blending.py:365-371)."""
    l_color = (ret["color"] - target_rgb).abs().mean()
    l_base = (ret["color_base"] - target_rgb).abs().mean()
    return l_color + color_base_weight * l_base + igr_weight * ret["gradient_error"]

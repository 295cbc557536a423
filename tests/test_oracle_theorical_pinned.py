"""Pins the 'theorical' sdf2alpha rule of the oracle (oracle/oracle_theorical.py) against outputs of the UNMODIFIED
reference run with sdf2alpha_type='theorical' (tests/golden/theorical_outputs.*.npz, oracle/make_golden_theorical.py),
with the tolerances of test_oracle_pinned.py; and the renderer mirror's sdf2alpha() helper and constructor.  CPU only."""
import pytest
import torch

from oracle import oracle_theorical as OT
from oracle import oracle_torch as O
from tests.golden_util import Fixtures, rel_err

TOL = {torch.float64: 1e-8, torch.float32: 2e-5}
TAGS = [(torch.float32, "f32"), (torch.float64, "f64")]


@pytest.fixture(scope="module")
def th():
    return Fixtures("theorical_outputs")


def T(fx, key, dtype=None):
    a = torch.from_numpy(fx[key])
    return a if dtype is None else a.to(dtype)


def _rays(g, dtype, n=64):
    return (g.t("rays_o", dtype)[:n], g.t("rays_d", dtype)[:n], g.t("near", dtype)[:n], g.t("far", dtype)[:n])


@pytest.mark.parametrize("dtype,tag", TAGS)
def test_up_sampling_rounds(golden, th, dtype, tag):
    o, d, near, far = _rays(golden, dtype)
    z, udf = golden.t("up_z_" + tag), golden.t("up_udf_" + tag)
    sd = ((far - near) / 64).mean().item()
    for i in range(5):
        gamma = float(min(max(20 * 2 ** (5 - i), 20), 320))
        nz, inds = OT.up_sample_unbias(o, d, z, udf, sd, 10, 64 * 2 ** i, 64 * 2 ** (i + 1), gamma, return_inds=True,
                                       sdf2alpha_type="theorical")
        assert torch.equal(nz, T(th, "up_newz_r%d_%s" % (i, tag))), i
        assert torch.equal(inds, T(th, "up_inds_r%d_%s" % (i, tag))), i
        # the default is the numerical rule, unchanged
        assert torch.equal(OT.up_sample_unbias(o, d, z, udf, sd, 10, 64 * 2 ** i, 64 * 2 ** (i + 1), gamma),
                           O.up_sample_unbias(o, d, z, udf, sd, 10, 64 * 2 ** i, 64 * 2 ** (i + 1), gamma))


@pytest.mark.parametrize("dtype,tag", TAGS)
def test_importance_sampling(golden, th, dtype, tag):
    p = O.to_dtype(golden.params["udf"], dtype)
    o, d, near, far = _rays(golden, dtype)
    z0, _, sd = O.coarse_z(near, far, 64, 0)
    udf_fn = lambda x: O.udf_mlp(p, golden.udf_c, x)[:, 0]
    with torch.no_grad():
        z = OT.importance_sample(udf_fn, o, d, z0, sd, 50, 5, sdf2alpha_type="theorical")
        assert rel_err(z, T(th, "imp_z_" + tag)) < 10 * TOL[dtype]
        _, beta, gamma = O.scalar_heads(O.to_dtype(golden.params["sc"], dtype))
        zm = OT.importance_sample_mix(udf_fn, o, d, z0, sd, 78, 5, beta, gamma, sdf2alpha_type="theorical")
        assert rel_err(zm, T(th, "impmix_z_" + tag)) < 10 * TOL[dtype]


def rc_case(golden, case, dtype):
    """keyword arguments of render_core for a fixture case; the NeRF++ background of rc_bg is recomputed by the oracle"""
    kw = dict(cos_anneal_ratio=None, flip_saturation=0.0) if case == "rc_na" else dict(cos_anneal_ratio=0.5,
                                                                                       flip_saturation=0.3)
    if case == "rc_bg":
        o, d, near, far = _rays(golden, dtype)
        S = 128
        z = near + (far - near) * torch.linspace(0.0, 1.0, S, dtype=dtype)[None, :]
        sd = ((far - near) / S).mean().item()
        zo = torch.linspace(1e-3, 1.0 - 1.0 / 33.0, 32, dtype=dtype)
        z_feed, _ = torch.sort(torch.cat([z, far / torch.flip(zo, dims=[-1]) + 1.0 / S], dim=-1), dim=-1)
        npar = O.to_dtype(golden.params["nerf"], dtype)
        with torch.no_grad():
            bg = O.render_core_outside(lambda a, b: O.nerf_mlp(npar, golden.nerf_c, a, b), o, d, z_feed, sd, 32)
        kw.update(background_alpha=bg["alpha"], background_sampled_color=bg["sampled_color"])
    return kw


RC_KEYS = ["color_base", "color", "weights", "depth", "gradient_error", "gradient_error_near_surface", "normals",
           "alpha", "alpha_plus", "alpha_minus", "sparse_error"]


@pytest.mark.parametrize("dtype,tag", TAGS)
@pytest.mark.parametrize("case", ["rc", "rc_na", "rc_bg"])
def test_render_core_and_grads(golden, th, dtype, tag, case):
    up = {k: v.clone().requires_grad_(True) for k, v in O.to_dtype(golden.params["udf"], dtype).items()}
    cp = {k: v.clone().requires_grad_(True) for k, v in O.to_dtype(golden.params["color"], dtype).items()}
    sc = {k: v.clone().requires_grad_(True) for k, v in O.to_dtype(golden.params["sc"], dtype).items()}
    o, d, near, far = _rays(golden, dtype)
    S = 128
    z = near + (far - near) * torch.linspace(0.0, 1.0, S, dtype=dtype)[None, :]
    sd = ((far - near) / S).mean().item()
    if case == "rc_bg" and dtype == torch.float32:
        # the fixture's own fp32 background (the oracle's NeRF differs from it in the last bits)
        kw = dict(cos_anneal_ratio=0.5, flip_saturation=0.3, background_alpha=T(th, "rc_bg_alpha_in_f32"),
                  background_sampled_color=T(th, "rc_bg_color_in_f32"))
    else:
        kw = rc_case(golden, case, dtype)
    ret = OT.render_core(up, golden.udf_c, cp, golden.col_c, sc, o, d, z, sd, sdf2alpha_type="theorical", **kw)
    tol = TOL[dtype] if dtype == torch.float64 else 2e-3      # as test_oracle_pinned.py's render_core
    for k in RC_KEYS:
        assert rel_err(ret[k], T(th, "%s_%s_%s" % (case, k, tag))) < tol, k
    from oracle.make_golden_theorical import rc_loss
    loss = rc_loss(ret, S, dtype)
    assert rel_err(loss, T(th, "%s_loss_%s" % (case, tag))) < tol
    if dtype != torch.float64:
        return
    loss.backward()
    from oracle.make_golden import GRAD_STRIDE
    n_checked = 0
    for mn, pd in (("udf", up), ("color", cp)):
        for pn, p in pd.items():
            key = "%s_grad.%s.%s_f64" % (case, mn, pn)
            if key in th:
                assert rel_err(p.grad, T(th, key)) < 1e-7, key
                n_checked += 1
            elif key + "_sub" in th:
                assert rel_err(p.grad.reshape(-1)[::GRAD_STRIDE], T(th, key + "_sub")) < 1e-7, key
                assert rel_err(p.grad.norm(), T(th, key + "_norm")) < 1e-7, key
                n_checked += 1
    assert n_checked >= 50
    assert rel_err(sc["variance"].grad, T(th, "%s_grad.var.variance_f64" % case)) < 1e-7
    assert rel_err(sc["beta"].grad, T(th, "%s_grad.beta.beta_f64" % case)) < 1e-7


def test_whole_render(golden, th):
    dtype = torch.float64
    up = {k: v.clone().requires_grad_(True) for k, v in O.to_dtype(golden.params["udf"], dtype).items()}
    cp = {k: v.clone().requires_grad_(True) for k, v in O.to_dtype(golden.params["color"], dtype).items()}
    npar = {k: v.clone().requires_grad_(True) for k, v in O.to_dtype(golden.params["nerf"], dtype).items()}
    sc = {k: v.clone().requires_grad_(True) for k, v in O.to_dtype(golden.params["sc"], dtype).items()}
    o, d, near, far = _rays(golden, dtype, 32)
    ret = OT.render(up, golden.udf_c, cp, golden.col_c, npar, golden.nerf_c, sc, o, d, near, far, 64, 50, 32, 5,
                    cos_anneal_ratio=0.7, flip_saturation=0.2, sdf2alpha_type="theorical")
    for k in ["z_vals", "color", "color_base", "weights", "depth", "weight_sum", "weight_sum_fg_bg", "udf",
              "gradients", "gradient_error", "sparse_error", "normals", "alpha"]:
        assert rel_err(ret[k], T(th, "render_%s_f64" % k)) < 1e-8, k
    tgt = torch.full((32, 3), 0.4, dtype=dtype)
    loss = ((ret["color"] - tgt).abs().mean() + 0.01 * (ret["color_base"] - tgt).abs().mean()
            + 0.1 * ret["gradient_error"])
    assert rel_err(loss, T(th, "render_loss_f64")) < 1e-8
    loss.backward()
    from oracle.make_golden import GRAD_STRIDE
    key = "render_grad.udf.lin4.weight_v_f64"
    assert rel_err(up["lin4.weight_v"].grad.reshape(-1)[::GRAD_STRIDE], T(th, key + "_sub")) < 1e-7
    assert rel_err(sc["variance"].grad, T(th, "render_grad.var.variance_f64")) < 1e-7


def _mirror(sdf2alpha_type):
    from neuraludf_b200.models.udf_renderer_blending import UDFRendererBlending
    return UDFRendererBlending(None, None, None, None, None, 64, 64, 0, 4, 0.0, sdf2alpha_type=sdf2alpha_type)


def test_renderer_constructor_accepts_theorical_only():
    assert _mirror("theorical").sdf2alpha_type == "theorical"
    assert _mirror("numerical").alpha_rule == 0 and _mirror("theorical").alpha_rule == 1
    for bad in ("theoretical", "Numerical", ""):
        with pytest.raises(NotImplementedError):
            _mirror(bad)


@pytest.mark.parametrize("sdf2alpha_type", ["theorical", "numerical"])
@pytest.mark.parametrize("r", [None, 0.3])
def test_mirror_sdf2alpha_helper_matches_reference(sdf2alpha_type, r):
    from oracle import refshim
    if not refshim.available():
        pytest.skip("reference checkout not present")
    _, R = refshim.load()
    ref = R.UDFRendererBlending(None, None, None, None, None, 64, 64, 0, 4, 0.0, sdf2alpha_type=sdf2alpha_type)
    mine = _mirror(sdf2alpha_type)
    g = torch.Generator().manual_seed(3)
    for dtype in (torch.float32, torch.float64):
        sdf = (torch.randn(64, 16, generator=g, dtype=torch.float64) * 0.05).to(dtype)
        sdf[0, :4] = torch.tensor([0.0, 1.0, -1.0, 50.0])
        tc = -(torch.rand(64, 16, generator=g, dtype=torch.float64) * 1.5).to(dtype)
        tc[1, :2] = 0.0
        dists = (torch.rand(64, 16, generator=g, dtype=torch.float64) * 0.02).to(dtype)
        inv_s = torch.tensor(300.0, dtype=dtype)
        want = ref.sdf2alpha(sdf, tc, dists, inv_s, r)
        got = mine.sdf2alpha(sdf, tc, dists, inv_s, r)
        assert torch.equal(got, want)
        assert torch.equal(OT.sdf2alpha(sdf, tc, dists, inv_s, r, sdf2alpha_type=sdf2alpha_type), want)

"""Golden fixtures of the 'theorical' sdf2alpha rule, from the UNMODIFIED reference (dev container only).

    python oracle/make_golden_theorical.py      # writes tests/golden/theorical_outputs.NN.npz

The seeded scene, rays and coarse samples are those of oracle/make_golden.py (reference_outputs.*.npz holds the inputs
`rays_*`, `near`, `far`, `up_z_*`, `up_udf_*`); the reference renderer is built with sdf2alpha_type='theorical' and run
in fp32 and fp64:
  * the five up_sample_unbias rounds of the classical schedule on the coarse samples, with the searchsorted indices of
    each round (recorded around the reference's own sample_pdf);
  * importance_sample (classical) and importance_sample_mix;
  * render_core on 64 rays x 128 samples with parameter gradients, with and without cos_anneal_ratio, and with the
    NeRF++ background composited behind (rc_bg; its background alpha / colour are stored as inputs);
  * one whole render() of 32 rays with parameter gradients.
Pins oracle/oracle_theorical.py (tests/test_oracle_theorical_pinned.py) and the CUDA path (tests/test_gpu_theorical.py).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import oracle_torch as O  # noqa: E402
from oracle import refshim  # noqa: E402
from oracle.make_golden import GRAD_STRIDE, build_ref_nets, np_  # noqa: E402
from tests.golden_util import save_fixtures, scene_digest  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")
RC_CASES = (("rc", dict(cos_anneal_ratio=0.5, flip_saturation=0.3), False),
            ("rc_na", dict(cos_anneal_ratio=None, flip_saturation=0.0), False),
            ("rc_bg", dict(cos_anneal_ratio=0.5, flip_saturation=0.3), True))


RULE_FREE = ("sampled_color_base", "sampled_color", "blending_weights", "gradients_flip", "gradients", "s_val", "udf",
             "gradient_mag", "true_cos", "inside_sphere", "mid_z_vals", "dists", "alpha_occ", "raw_occ", "vis_prob")


def rc_loss(ret, S, dtype):
    tgt = torch.full((ret["color"].shape[0], 3), 0.4, dtype=dtype, device=ret["color"].device)
    return ((ret["color"] - tgt).abs().mean() + 0.01 * (ret["color_base"] - tgt).abs().mean()
            + 0.1 * ret["gradient_error"] + 1e-3 * ret["sparse_error"]
            + 0.05 * ret["gradient_error_near_surface"]
            + 0.1 * ((ret["weights"][:, :S].sum(-1) - 0.5) ** 2).mean())


def main():
    F, R = refshim.load()
    params = {"udf": O.make_udf_params(O.udf_cfg(), seed=0),
              "udf_small": O.make_udf_params(O.udf_cfg(d_hidden=128, n_layers=4), seed=3),
              "color": O.make_color_params(O.color_cfg(), seed=1), "nerf": O.make_nerf_params(O.nerf_cfg(), seed=2),
              "sc": O.make_scalars()}
    with open(os.path.join(OUT, "scene_params.sha256")) as f:
        assert scene_digest(params) == f.read().strip(), "the seeded scene differs from reference_outputs'"
    udf_c, col_c, nerf_c = O.udf_cfg(), O.color_cfg(), O.nerf_cfg()
    fx = {}
    ref_sample_pdf = R.sample_pdf
    for dtype, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
        udf, col, nerf, var, beta = build_ref_nets(F, udf_c, col_c, nerf_c, params["udf"], params["color"],
                                                   params["nerf"], params["sc"], dtype)
        ren = R.UDFRendererBlending(nerf, udf, var, col, beta, n_samples=64, n_importance=50, n_outside=32,
                                    up_sample_steps=5, perturb=0.0, sdf2alpha_type="theorical")
        o, d, near, far = O.make_rays(64, seed=0)
        o, d, near, far = o.to(dtype), d.to(dtype), near.to(dtype), far.to(dtype)

        # ---- up-sampling rounds (with indices), both importance schedules ----
        sample_dist = ((far - near) / 64).mean().item()
        z0 = near + (far - near) * torch.linspace(0.0, 1.0, 64)[None, :]
        rounds = []

        def recording_sample_pdf(bins, weights, n_samples, det=False):
            _, inds = O.sample_pdf_det(bins, weights, n_samples, return_inds=True)
            rounds.append(inds)
            return ref_sample_pdf(bins, weights, n_samples, det=det)

        with torch.no_grad():
            pts = o[:, None, :] + d[:, None, :] * z0[..., :, None]
            u0 = udf(pts.reshape(-1, 3))[:, 0].reshape(64, 64)
            R.sample_pdf = recording_sample_pdf
            try:
                for i in range(5):
                    nz = ren.up_sample_unbias(o, d, z0, u0, sample_dist, 10, 64 * 2 ** i, 64 * 2 ** (i + 1),
                                              gamma=float(np.clip(20 * 2 ** (5 - i), 20, 320)))
                    fx["up_newz_r%d_%s" % (i, tag)] = np_(nz)
                    fx["up_inds_r%d_%s" % (i, tag)] = rounds[-1].numpy()
            finally:
                R.sample_pdf = ref_sample_pdf
            fx["imp_z_" + tag] = np_(ren.importance_sample(o, d, z0, sample_dist))
            ren.upsampling_type = "mix"
            ren.n_importance, ren.up_sample_steps = 78, 5
            fx["impmix_z_" + tag] = np_(ren.importance_sample_mix(o, d, z0, sample_dist))
            ren.upsampling_type = "classical"
            ren.n_importance, ren.up_sample_steps = 50, 5

        # ---- render_core, 64 rays x 128 samples, + parameter gradients ----
        S = 128
        z = near + (far - near) * torch.linspace(0.0, 1.0, S)[None, :]
        sd = ((far - near) / S).mean().item()
        with torch.no_grad():
            zo = torch.linspace(1e-3, 1.0 - 1.0 / 33.0, 32, dtype=dtype)
            z_out = far / torch.flip(zo, dims=[-1]) + 1.0 / S
            z_feed, _ = torch.sort(torch.cat([z, z_out], dim=-1), dim=-1)
            bg = ren.render_core_outside(o, d, z_feed, sd, nerf)
        fx["rc_bg_alpha_in_" + tag], fx["rc_bg_color_in_" + tag] = np_(bg["alpha"]), np_(bg["sampled_color"])
        for name, kw, with_bg in RC_CASES:
            for m in (udf, col, var, beta):
                m.zero_grad(set_to_none=True)
            if with_bg:
                kw = dict(kw, background_alpha=bg["alpha"], background_sampled_color=bg["sampled_color"])
            ret = ren.render_core(o, d, z, sd, udf, var, col, beta_network=beta, **kw)
            loss = rc_loss(ret, S, dtype)
            loss.backward()
            for k, v in ret.items():
                if isinstance(v, torch.Tensor):
                    fx["%s_%s_%s" % (name, k, tag)] = np_(v)
            fx["%s_loss_%s" % (name, tag)] = np_(loss)
            for mn, m in (("udf", udf), ("color", col), ("var", var), ("beta", beta)):
                for pn, p in m.named_parameters():
                    if p.grad is not None:
                        fx["%s_grad.%s.%s_%s" % (name, mn, pn, tag)] = np_(p.grad)

        # ---- whole render(), DTU conf, perturb 0, 32 rays ----
        for m in (udf, col, var, beta, nerf):
            m.zero_grad(set_to_none=True)
        o2, d2, n2, f2 = o[:32], d[:32], near[:32], far[:32]
        # render() draws `torch.rand([1024,3]).float()` for sparse_random_error (:683), which breaks an fp64 run; cast
        # inside .udf() only (that output is not part of any comparison)
        udf.udf = (lambda x, _m=udf, _dt=dtype: F.UDFNetwork.udf(_m, x.to(_dt)))
        ret = ren.render(o2, d2, n2, f2, cos_anneal_ratio=0.7, perturb_overwrite=0, flip_saturation=0.2)
        tgt = torch.full((32, 3), 0.4, dtype=dtype)
        loss = ((ret["color"] - tgt).abs().mean() + 0.01 * (ret["color_base"] - tgt).abs().mean()
                + 0.1 * ret["gradient_error"])
        loss.backward()
        for k in ("z_vals", "color", "color_base", "weights", "depth", "weight_sum", "weight_sum_fg_bg", "udf",
                  "gradients", "gradient_error", "sparse_error", "normals", "alpha"):
            fx["render_%s_%s" % (k, tag)] = np_(ret[k])
        fx["render_loss_" + tag] = np_(loss)
        for mn, m in (("udf", udf), ("color", col), ("var", var), ("beta", beta), ("nerf", nerf)):
            for pn, p in m.named_parameters():
                if p.grad is not None:
                    fx["render_grad.%s.%s_%s" % (mn, pn, tag)] = np_(p.grad)

    torch.set_default_dtype(torch.float32)
    # as make_golden.py: large gradients keep the fp64 arbiter only, as a strided subsample plus its L2 norm
    for k in list(fx):
        if "_grad." in k and fx[k].size > 4096:
            if k.endswith("_f32"):
                del fx[k]
                continue
            full = fx.pop(k).astype(np.float64).reshape(-1)
            fx[k + "_sub"] = full[::GRAD_STRIDE].copy()
            fx[k + "_norm"] = np.array(np.sqrt((full ** 2).sum()))
    # per-sample outputs that do not depend on the alpha rule (reference_outputs holds them) or that no test reads
    for k in list(fx):
        if any(k.startswith("%s_%s_" % (c, n)) for c, _, _ in RC_CASES for n in RULE_FREE):
            del fx[k]
    del fx["rc_bg_color_in_f64"], fx["rc_bg_alpha_in_f64"]      # inputs: the fp32 run's suffice
    save_fixtures("theorical_outputs", fx)
    print("wrote", len(fx), "arrays;", sum(v.nbytes for v in fx.values()) / 1e6, "MB raw")


if __name__ == "__main__":
    main()

"""The 'theorical' sdf2alpha rule in the PyTorch restatement of the renderer (test infrastructure only).

Reference: models/udf_renderer_blending.py:292-325.  The 'theorical' branch (:321-323) is

    raw   = |iter_cos| * inv_s * (1 - sigmoid(sdf * inv_s))
    alpha = 1 - exp(-relu(raw) * dists)            (no clip)

with iter_cos as in the 'numerical' branch.  `udf_eps` is never passed by any caller and is left out.

oracle_torch.py restates the 'numerical' rule; every function of it that reaches sdf2alpha (up_sample_unbias,
importance_sample, importance_sample_mix, composite, render_core, render) looks `neus_alpha` up in its module at call
time.  The functions here take an `sdf2alpha_type` keyword ('numerical' by default) and run oracle_torch's function with
that rule in place of `neus_alpha` for the duration of the call, so the two rules share every other line of the
restatement.  Pinned against the unmodified reference by tests/test_oracle_theorical_pinned.py.
"""
import contextlib

import torch
import torch.nn.functional as F

from oracle import oracle_torch as O


def iter_cos(true_cos, cos_anneal_ratio=None):
    """:295-299"""
    if cos_anneal_ratio is None:
        return true_cos
    return -(F.relu(-true_cos * 0.5 + 0.5) * (1.0 - cos_anneal_ratio) + F.relu(-true_cos) * cos_anneal_ratio)


def theorical_alpha(sdf, true_cos, dists, inv_s, cos_anneal_ratio=None):
    """'theorical' branch of sdf2alpha (:321-323): 1 - sigmoid is formed as written, the sigmoid first."""
    abs_cos_val = iter_cos(true_cos, cos_anneal_ratio).abs()
    raw = abs_cos_val * inv_s * (1 - torch.sigmoid(sdf * inv_s))
    return 1.0 - torch.exp(-F.relu(raw) * dists)


SDF2ALPHA = {"numerical": O.neus_alpha, "theorical": theorical_alpha}


def sdf2alpha(sdf, true_cos, dists, inv_s, cos_anneal_ratio=None, sdf2alpha_type="numerical"):
    return SDF2ALPHA[sdf2alpha_type](sdf, true_cos, dists, inv_s, cos_anneal_ratio)


@contextlib.contextmanager
def _rule(sdf2alpha_type):
    fn = SDF2ALPHA[sdf2alpha_type]
    saved = O.neus_alpha
    O.neus_alpha = fn
    try:
        yield
    finally:
        O.neus_alpha = saved


def _with_rule(name):
    base = getattr(O, name)

    def f(*args, sdf2alpha_type="numerical", **kw):
        with _rule(sdf2alpha_type):
            return base(*args, **kw)

    f.__name__ = name
    f.__doc__ = "oracle_torch.%s under the sdf2alpha rule `sdf2alpha_type`.\n\n%s" % (name, base.__doc__ or "")
    return f


up_sample_unbias = _with_rule("up_sample_unbias")
importance_sample = _with_rule("importance_sample")
importance_sample_mix = _with_rule("importance_sample_mix")
composite = _with_rule("composite")
render_core = _with_rule("render_core")
render = _with_rule("render")

// Per-sample formulas of the UDF -> visibility-weighted density -> alpha pipeline, with hand-derived derivatives.
// Reference: models/udf_renderer_blending.py:151-159 (udf2logistic), :292-325 (sdf2alpha 'numerical'),
// :394-419 (render_core), :228-262 (up_sample_unbias).  Every function is NUDF_HD: the CUDA kernels in
// ray_kernels.cu / sampling.cu call them per lane, and tests/host/raymath_host.cpp compiles the same code with g++
// to check values and derivatives against the oracle's autograd on the CPU-only dev box.
#pragma once
#include "common.cuh"

namespace nudf {

// ---- logistic occlusion density and its alpha (:157-158, :394-397) ----------------------------------------------
// raw = beta e^{-beta u} / (1 + e^{-beta u})^2 ;  alpha_occ = 1 - exp(-relu(raw) * gamma * dist)
NUDF_HD void occ_forward(float u, float dist, float beta, float gamma, float* raw, float* aocc) {
  float e = expf(-beta * u);
  float den = (1.0f + e);
  float r = beta * e / (den * den);
  *raw = r;
  *aocc = 1.0f - expf(-fmaxf(r, 0.0f) * gamma * dist);
}
NUDF_HD void occ_backward(float u, float dist, float beta, float gamma, float aocc_bar, float* u_bar, float* beta_bar,
                          float* gamma_bar) {
  float e = expf(-beta * u);
  float den = 1.0f + e;
  float h = e / (den * den);            // sigma (1 - sigma), sigma = 1/(1+e)
  float hp = h * (e - 1.0f) / den;      // dh/dy at y = beta u :  sigma(1-sigma)(1-2 sigma)
  float raw = beta * h;
  float rr = fmaxf(raw, 0.0f);
  float m_bar = aocc_bar * expf(-rr * gamma * dist);
  float raw_bar = raw > 0.0f ? m_bar * gamma * dist : 0.0f;
  *gamma_bar = m_bar * rr * dist;
  *beta_bar = raw_bar * (h + beta * u * hp);
  *u_bar = raw_bar * beta * beta * hp;
}

// ---- cosine annealing (:295-299); input is the signed true_cos, the pipeline uses -|true_cos| -------------------
NUDF_HD float iter_cos_forward(float true_cos, int has_r, float r) {
  float tcn = -fabsf(true_cos);
  if (!has_r) return tcn;
  return -(fmaxf(-tcn * 0.5f + 0.5f, 0.0f) * (1.0f - r) + fmaxf(-tcn, 0.0f) * r);
}
// d iter_cos / d true_cos
NUDF_HD float iter_cos_dtc(float true_cos, int has_r, float r) {
  float sg = true_cos > 0.0f ? 1.0f : (true_cos < 0.0f ? -1.0f : 0.0f);
  float dtcn = -sg;                                   // d(-|tc|)/d tc
  if (!has_r) return dtcn;
  float a = fabsf(true_cos);
  float d_ic_dtcn = 0.5f * (1.0f - r) + (a > 0.0f ? r : 0.0f);
  return d_ic_dtcn * dtcn;
}

// ---- NeuS discrete alpha, 'numerical' branch (:308-320) ----------------------------------------------------------
NUDF_HD float neus_alpha_forward(float sdf, float ic, float dist, float s) {
  float half = ic * dist * 0.5f;
  float nxt = sdf + half;
  float prv = sdf - half;
  float cp = sigmoidf_(prv * s);
  float cn = sigmoidf_(nxt * s);
  float x = (cp - cn + 1e-5f) / (cp + 1e-5f);
  return clampf_(x, 0.0f, 1.0f);
}
NUDF_HD void neus_alpha_backward(float sdf, float ic, float dist, float s, float a_bar, float* sdf_bar, float* ic_bar,
                                 float* s_bar) {
  float half = ic * dist * 0.5f;
  float nxt = sdf + half;
  float prv = sdf - half;
  float cp = sigmoidf_(prv * s);
  float cn = sigmoidf_(nxt * s);
  float den = cp + 1e-5f;
  float x = (cp - cn + 1e-5f) / den;
  float x_bar = (x >= 0.0f && x <= 1.0f) ? a_bar : 0.0f;
  float cp_bar = x_bar * (1.0f - x) / den;
  float cn_bar = -x_bar / den;
  float parg = cp_bar * cp * (1.0f - cp);
  float narg = cn_bar * cn * (1.0f - cn);
  *s_bar = parg * prv + narg * nxt;
  float prv_bar = parg * s, nxt_bar = narg * s;
  *sdf_bar = prv_bar + nxt_bar;
  *ic_bar = (nxt_bar - prv_bar) * dist * 0.5f;
}

// ---- NeuS density alpha, 'theorical' branch (:321-323) -----------------------------------------------------------
// raw = |ic| * s * (1 - sigmoid(sdf * s)) ;  alpha = 1 - exp(-relu(raw) * dist).  No clip.  1 - sigmoid is formed as
// written (sigmoid, then the subtraction), so that it is exactly 0 where the reference's is.
NUDF_HD float theorical_alpha_forward(float sdf, float ic, float dist, float s) {
  float m = 1.0f - sigmoidf_(sdf * s);
  float raw = fabsf(ic) * s * m;
  return 1.0f - expf(-fmaxf(raw, 0.0f) * dist);
}
// d/d(sdf, ic, s) with torch's conventions at the edges: d|ic|/d ic = sign(ic) (0 at 0), relu'(0) = 0
NUDF_HD void theorical_alpha_backward(float sdf, float ic, float dist, float s, float a_bar, float* sdf_bar, float* ic_bar,
                                      float* s_bar) {
  float sg = sigmoidf_(sdf * s);
  float m = 1.0f - sg;
  float A = fabsf(ic);
  float As = A * s;
  float raw = As * m;
  float rr = fmaxf(raw, 0.0f);
  float raw_bar = raw > 0.0f ? a_bar * expf(-rr * dist) * dist : 0.0f;
  float x_bar = -(raw_bar * As) * (sg * (1.0f - sg));   // through m = 1 - sigmoid(x), x = sdf * s
  float As_bar = raw_bar * m;
  float A_bar = As_bar * s;
  *sdf_bar = x_bar * s;
  *s_bar = As_bar * A + x_bar * sdf;
  *ic_bar = ic > 0.0f ? A_bar : (ic < 0.0f ? -A_bar : 0.0f);
}

// The alpha rule as a compile-time choice (sdf2alpha_type): the kernels are instantiated once per rule, so neither
// pays a per-sample branch.  Rule 0 is 'numerical', rule 1 'theorical'.
enum AlphaRule : int { ALPHA_NUMERICAL = 0, ALPHA_THEORICAL = 1 };
template <int RULE>
NUDF_HD float alpha_forward(float sdf, float ic, float dist, float s) {
  if constexpr (RULE == ALPHA_THEORICAL) return theorical_alpha_forward(sdf, ic, dist, s);
  else return neus_alpha_forward(sdf, ic, dist, s);
}
template <int RULE>
NUDF_HD void alpha_backward(float sdf, float ic, float dist, float s, float a_bar, float* sdf_bar, float* ic_bar,
                            float* s_bar) {
  if constexpr (RULE == ALPHA_THEORICAL) theorical_alpha_backward(sdf, ic, dist, s, a_bar, sdf_bar, ic_bar, s_bar);
  else neus_alpha_backward(sdf, ic, dist, s, a_bar, sdf_bar, ic_bar, s_bar);
}

// ---- gradient-derived quantities (:370-388) ----------------------------------------------------------------------
struct GradQ { float gmag, tc, cosn, flip; };
NUDF_HD GradQ grad_quantities(const float g[3], const float d[3], int use_norm) {
  GradQ q;
  q.gmag = sqrtf(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
  float inv = 1.0f / (q.gmag + 1e-5f);
  float dg = d[0] * g[0] + d[1] * g[1] + d[2] * g[2];
  q.cosn = d[0] * (g[0] * inv) + d[1] * (g[1] * inv) + d[2] * (g[2] * inv);
  q.tc = use_norm ? q.cosn : dg;
  q.flip = q.cosn > 0.0f ? -1.0f : 1.0f;   // -sign(cos), with sign(0) -> +1 (:387-388)
  return q;
}
// adjoint: g_bar += tc_bar * d tc/d g + eik_coef * (|g|-1) 2 g/|g|   (eik_coef already holds mask/denominator/upstream)
NUDF_HD void grad_quantities_backward(const float g[3], const float d[3], int use_norm, float tc_bar, float eik_coef,
                                      float g_bar[3]) {
  float gmag = sqrtf(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
  float dg = d[0] * g[0] + d[1] * g[1] + d[2] * g[2];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v;
    if (use_norm) {
      float den = gmag + 1e-5f;
      // tc = (d.g)/den ; d den / d g_c = g_c / gmag
      v = tc_bar * (d[c] / den - (gmag > 0.0f ? dg * g[c] / (gmag * den * den) : 0.0f));
    } else {
      v = tc_bar * d[c];
    }
    if (gmag > 0.0f) v += eik_coef * 2.0f * (gmag - 1.0f) * g[c] / gmag;
    g_bar[c] = v;
  }
}

}  // namespace nudf

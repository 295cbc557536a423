// Host (g++) harness of the 'theorical' alpha rule of neuraludf_b200/csrc/raymath.cuh (sdf2alpha, :321-323).
//  * theorical_sample: one sample's alpha and its derivatives d/d(sdf, true_cos, inv_s), with the kernels' iter_cos;
//  * ray_forward_host / ray_backward_host: the sequential per-ray composite of raymath_host.cpp, compiled here with the
//    'theorical' rule in place of the 'numerical' one (the same substitution the kernels' template argument makes).
#include "../../neuraludf_b200/csrc/raymath.cuh"

using namespace nudf;

extern "C" {

// out = (alpha, sdf_bar, true_cos_bar, inv_s_bar) for upstream a_bar; true_cos is the signed cosine the kernels read
void theorical_sample(float sdf, float true_cos, float dist, float s, int has_r, float r, float a_bar, float* out) {
  const float ic = iter_cos_forward(true_cos, has_r, r);
  out[0] = alpha_forward<ALPHA_THEORICAL>(sdf, ic, dist, s);
  float sdf_bar, ic_bar, s_bar;
  alpha_backward<ALPHA_THEORICAL>(sdf, ic, dist, s, a_bar, &sdf_bar, &ic_bar, &s_bar);
  out[1] = sdf_bar;
  out[2] = ic_bar * iter_cos_dtc(true_cos, has_r, r);
  out[3] = s_bar;
}

}  // extern "C"

// raymath.cuh is included above (#pragma once), so these names change only in the per-ray harness below
#define neus_alpha_forward theorical_alpha_forward
#define neus_alpha_backward theorical_alpha_backward
#include "raymath_host.cpp"

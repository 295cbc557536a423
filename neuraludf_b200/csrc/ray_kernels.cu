// render_core ray kernels: sample-point generation, UDF -> alpha conversion, visibility and transmittance scans,
// alpha compositing, regulariser partial sums -- forward and hand-written backward.
// One warp per ray; lanes stride over the samples of the ray (coalesced loads), the two exclusive product scans
// (vis_prob, transmittance) and the two reverse affine scans of the backward pass are warp-shuffle scans with a
// carry across 32-sample chunks.  Reference: models/udf_renderer_blending.py:352-362, 370-419, 484-553.
#include "../../include/nudf.h"
#include "common.cuh"
#include "raymath.cuh"

namespace nudf {

constexpr int RK_WARPS = 4;
constexpr unsigned FULL = 0xffffffffu;

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
  return v;
}
// inclusive product scan over the warp
__device__ __forceinline__ float warp_scan_mul(float v, int lane) {
  for (int o = 1; o < 32; o <<= 1) {
    float t = __shfl_up_sync(FULL, v, o);
    if (lane >= o) v *= t;
  }
  return v;
}
// reverse inclusive scan of affine maps x -> a + f x : afterwards (a, f) of lane i is the composition of lanes i..31
__device__ __forceinline__ void warp_rscan_affine(float& a, float& f, int lane) {
  for (int o = 1; o < 32; o <<= 1) {
    float a2 = __shfl_down_sync(FULL, a, o);
    float f2 = __shfl_down_sync(FULL, f, o);
    if (lane + o < 32) { a = a + f * a2; f = f * f2; }
  }
}

// pts = o + d * mid ; written without fma contraction so that thresholds on |pts| agree with a mul-then-add evaluation
__global__ void ray_points_kernel(const float* __restrict__ o, const float* __restrict__ d, const float* __restrict__ z,
                                  int n_rays, int S, float sample_dist, float* __restrict__ pts, float* __restrict__ mid_z,
                                  float* __restrict__ dists) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n_rays * S) return;
  int r = (int)(idx / S), i = (int)(idx - (int64_t)r * S);
  float z0 = z[idx];
  float dist = (i + 1 < S) ? __fsub_rn(z[idx + 1], z0) : sample_dist;
  float mid = __fadd_rn(z0, __fmul_rn(dist, 0.5f));
  if (mid_z) mid_z[idx] = mid;
  if (dists) dists[idx] = dist;
  if (pts) {
#pragma unroll
    for (int c = 0; c < 3; ++c) pts[idx * 3 + c] = __fadd_rn(o[r * 3 + c], __fmul_rn(d[r * 3 + c], mid));
  }
}

// generic points on rays: pts[r, i] = o + d * z   (importance sampling inputs, :205, :277, :729)
__global__ void points_on_rays_kernel(const float* __restrict__ o, const float* __restrict__ d, const float* __restrict__ z,
                                      int n_rays, int n, float* __restrict__ pts) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n_rays * n) return;
  int r = (int)(idx / n);
  float zz = z[idx];
#pragma unroll
  for (int c = 0; c < 3; ++c) pts[idx * 3 + c] = __fadd_rn(o[r * 3 + c], __fmul_rn(d[r * 3 + c], zz));
}

// NeRF++ inverted-sphere inputs for columns [col0, n) of z (:164-173): pts4 = (p / r, 1 / r), r = max(|p|, 1)
__global__ void outside_points_kernel(const float* __restrict__ o, const float* __restrict__ d, const float* __restrict__ z,
                                      int n_rays, int n, int col0, float sample_dist, float* __restrict__ pts4,
                                      float* __restrict__ dists) {
  int m = n - col0;
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)n_rays * m) return;
  int r = (int)(idx / m), j = (int)(idx - (int64_t)r * m), i = col0 + j;
  float z0 = z[(int64_t)r * n + i];
  float dist = (i + 1 < n) ? __fsub_rn(z[(int64_t)r * n + i + 1], z0) : sample_dist;
  float mid = __fadd_rn(z0, __fmul_rn(dist, 0.5f));
  float p[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) p[c] = __fadd_rn(o[r * 3 + c], __fmul_rn(d[r * 3 + c], mid));
  float rr = sqrtf(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
  rr = fminf(fmaxf(rr, 1.0f), 1e10f);
  pts4[idx * 4 + 0] = p[0] / rr; pts4[idx * 4 + 1] = p[1] / rr; pts4[idx * 4 + 2] = p[2] / rr; pts4[idx * 4 + 3] = 1.0f / rr;
  dists[idx] = dist;
}

// ---------------------------------------------------------------------------------------------------------------
// Shared per-ray forward state (one slot per sample, in shared memory, private to the warp).
// ---------------------------------------------------------------------------------------------------------------
struct RaySmem {
  float* tc;      // true_cos (fg)
  float* t;       // clip(1 - alpha_occ + fs * vis_mask, 0, 1) + 1e-7 (fg), pre-clip q kept in `q`
  float* q;
  float* P;       // exclusive cumprod of t (un-clipped vis_prob)
  float* ap;      // alpha_plus
  float* am;      // alpha_minus
  float* alpha;   // all S+O
  float* T;       // exclusive transmittance, all S+O
  float* wbar;    // backward only
  float* abar;    // backward only
};

struct RayIn {
  const float* heads;   // device (inv_s, beta, gamma)
  const float* rays_d; const float* pts; const float* mid_z; const float* dists; const float* udf; int64_t ld_udf;
  const float* grads; const float* scb; const float* sc; const float* bg_alpha; const float* bg_color;
};

// Steps shared by forward and backward: fills tc, q, t, P, ap, am, alpha, T for ray r.  RULE is the alpha rule
// (AlphaRule, raymath.cuh) of pass 3.
template <int RULE>
__device__ __forceinline__ void ray_forward_state(const nudf_render_cfg& cfg, const RayIn& in, int r, int lane, RaySmem sm) {
  const int S = cfg.n_samples, O = cfg.n_outside, SO = S + O;
  const int64_t base = (int64_t)r * S;
  const float d[3] = {in.rays_d[r * 3 + 0], in.rays_d[r * 3 + 1], in.rays_d[r * 3 + 2]};
  const float inv_s = in.heads[0], beta = in.heads[1], gamma = in.heads[2];
  // pass 1: true_cos for every fg sample
  for (int i = lane; i < S; i += 32) {
    const float g[3] = {in.grads[(base + i) * 3 + 0], in.grads[(base + i) * 3 + 1], in.grads[(base + i) * 3 + 2]};
    GradQ gq = grad_quantities(g, d, cfg.use_norm_grad_for_cosine);
    sm.tc[i] = gq.tc;
  }
  __syncwarp();
  // pass 2: occlusion alpha, visibility factor, exclusive product scan -> P
  float carry = 1.0f;
  for (int i0 = 0; i0 < S; i0 += 32) {
    int i = i0 + lane;
    float t = 1.0f;
    if (i < S) {
      float u = in.udf[(base + i) * in.ld_udf];
      float dist = in.dists[base + i];
      float raw, aocc;
      occ_forward(u, dist, beta, gamma, &raw, &aocc);
      float vm = (i + 1 < S) ? (sm.tc[i + 1] < 0.01f ? 1.0f : 0.0f) : 1.0f;
      float q = 1.0f - aocc + cfg.flip_saturation * vm;
      t = clampf_(q, 0.0f, 1.0f) + 1e-7f;
      sm.q[i] = q;
      sm.t[i] = t;
    }
    float inc = warp_scan_mul(t, lane);
    float exc = __shfl_up_sync(FULL, inc, 1);
    if (lane == 0) exc = 1.0f;
    if (i < S) sm.P[i] = carry * exc;
    carry *= __shfl_sync(FULL, inc, 31);
  }
  __syncwarp();
  // pass 3: alpha (+/-), blended alpha; background alphas appended
  for (int i = lane; i < SO; i += 32) {
    float a;
    if (i < S) {
      float u = in.udf[(base + i) * in.ld_udf];
      float dist = in.dists[base + i];
      float ic = iter_cos_forward(sm.tc[i], cfg.has_cos_anneal, cfg.cos_anneal_ratio);
      float ap = alpha_forward<RULE>(u, ic, dist, inv_s);
      float am = alpha_forward<RULE>(-u, ic, dist, inv_s);
      float vis = clampf_(sm.P[i], 0.0f, 1.0f);
      sm.ap[i] = ap; sm.am[i] = am;
      a = ap * vis + am * (1.0f - vis);
    } else {
      a = in.bg_alpha[(int64_t)r * SO + i];
    }
    sm.alpha[i] = a;
  }
  __syncwarp();
  // pass 4: transmittance
  carry = 1.0f;
  for (int i0 = 0; i0 < SO; i0 += 32) {
    int i = i0 + lane;
    float f = (i < SO) ? (1.0f - sm.alpha[i] + 1e-7f) : 1.0f;
    float inc = warp_scan_mul(f, lane);
    float exc = __shfl_up_sync(FULL, inc, 1);
    if (lane == 0) exc = 1.0f;
    if (i < SO) sm.T[i] = carry * exc;
    carry *= __shfl_sync(FULL, inc, 31);
  }
  __syncwarp();
}

__device__ __forceinline__ RaySmem carve(float* base, int SO) {
  RaySmem sm;
  sm.tc = base; sm.t = base + SO; sm.q = base + 2 * SO; sm.P = base + 3 * SO; sm.ap = base + 4 * SO;
  sm.am = base + 5 * SO; sm.alpha = base + 6 * SO; sm.T = base + 7 * SO; sm.wbar = base + 8 * SO; sm.abar = base + 9 * SO;
  return sm;
}
constexpr int RK_ARRAYS = 10;

// Compositing sums every forward entry point shares: colour, depth and the weight sums, accumulated in one fixed order
// per accumulator and with explicitly rounded products / fused multiply-adds (the compiler's contraction choices depend
// on the surrounding kernel), so that every entry point returns the same bits for them.  `ex` adds the caller's own per-sample terms:
// ex.fg(i, p, w, u, g, gq) for a foreground sample (p = flat sample index), ex.bg(i, q, w, col) for a background column
// (q = flat [N, S+O] index, col its colour).
struct RaySums { float cc[3]; float depth, ws_fg, ws_all; };

template <class Extra>
__device__ __forceinline__ RaySums ray_composite(const nudf_render_cfg& cfg, const RayIn& in, int r, int lane, RaySmem sm,
                                                 Extra& ex) {
  const int S = cfg.n_samples, O = cfg.n_outside, SO = S + O;
  const int64_t base = (int64_t)r * S;
  const float d[3] = {in.rays_d[r * 3 + 0], in.rays_d[r * 3 + 1], in.rays_d[r * 3 + 2]};
  RaySums s = {{0.f, 0.f, 0.f}, 0.f, 0.f, 0.f};
  for (int i = lane; i < SO; i += 32) {
    const float w = __fmul_rn(sm.alpha[i], sm.T[i]);
    s.ws_all = __fadd_rn(s.ws_all, w);
    if (i < S) {
      const int64_t p = base + i;
      s.ws_fg = __fadd_rn(s.ws_fg, w);
      float u = in.udf[p * in.ld_udf];
      const float g[3] = {in.grads[p * 3 + 0], in.grads[p * 3 + 1], in.grads[p * 3 + 2]};
      GradQ gq = grad_quantities(g, d, cfg.use_norm_grad_for_cosine);
#pragma unroll
      for (int c = 0; c < 3; ++c) s.cc[c] = __fmaf_rn(w, in.sc[p * 3 + c], s.cc[c]);
      s.depth = __fmaf_rn(w, in.mid_z[p], s.depth);
      ex.fg(i, p, w, u, g, gq);
    } else {
      const int64_t q = (int64_t)r * SO + i;
      float col[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        col[c] = in.bg_color[q * 3 + c];
        s.cc[c] = __fmaf_rn(w, col[c], s.cc[c]);
      }
      ex.bg(i, q, w, col);
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) s.cc[c] = warp_sum(s.cc[c]);
  s.depth = warp_sum(s.depth); s.ws_fg = warp_sum(s.ws_fg); s.ws_all = warp_sum(s.ws_all);
  return s;
}

// colour of the ray: composite plus the constant background colour behind it (:527-528)
__device__ __forceinline__ float ray_color(const nudf_render_cfg& cfg, const RaySums& s, int c) {
  float col = s.cc[c];
  if (cfg.has_background_rgb) col = __fmaf_rn(cfg.background_rgb[c], __fsub_rn(1.0f, s.ws_all), col);
  return col;
}

// sphere test of the regularisers and of the normal map (:512, :527): |pts| < 1
__device__ __forceinline__ float sample_norm(const RayIn& in, int64_t p) {
  float px = in.pts[p * 3 + 0], py = in.pts[p * 3 + 1], pz = in.pts[p * 3 + 2];
  return sqrtf(px * px + py * py + pz * pz);
}

// render_core's own per-sample terms: colour_base, normals, regulariser sums, per-sample diagnostics
struct CoreExtra {
  const nudf_render_cfg& cfg; const RayIn& in; const nudf_render_out& out; const RaySmem& sm; int r;
  float cb[3] = {0, 0, 0}, nrm[3] = {0, 0, 0};
  float s_relax_ge = 0.f, s_relax = 0.f, s_near_ge = 0.f, s_near = 0.f, s_sparse = 0.f;
  __device__ CoreExtra(const nudf_render_cfg& cfg_, const RayIn& in_, const nudf_render_out& out_, const RaySmem& sm_, int r_)
      : cfg(cfg_), in(in_), out(out_), sm(sm_), r(r_) {}
  __device__ __forceinline__ void weight(int i, float w) {
    if (out.weights) out.weights[(int64_t)r * (cfg.n_samples + cfg.n_outside) + i] = w;
  }
  __device__ __forceinline__ void fg(int i, int64_t p, float w, float u, const float g[3], const GradQ& gq) {
    weight(i, w);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      cb[c] += w * in.scb[p * 3 + c];
      nrm[c] += w * gq.flip * g[c];
    }
    float pn = sample_norm(in, p);
    float inside = pn < 1.0f ? 1.f : 0.f, relax = pn < 1.2f ? 1.f : 0.f, near = u < 0.05f ? 1.f : 0.f;
    float ge = (gq.gmag - 1.0f) * (gq.gmag - 1.0f);
    s_relax_ge += relax * ge; s_relax += relax; s_near_ge += near * ge; s_near += near;
    s_sparse += expf(-cfg.sparse_scale_factor * u);
    // per-sample diagnostics
    float raw, aocc;
    occ_forward(u, in.dists[p], in.heads[1], in.heads[2], &raw, &aocc);
    if (out.gradient_mag) out.gradient_mag[p] = gq.gmag;
    if (out.true_cos) out.true_cos[p] = gq.tc;
    if (out.vis_prob) out.vis_prob[p] = clampf_(sm.P[i], 0.f, 1.f);
    if (out.alpha) out.alpha[p] = sm.alpha[i];
    if (out.alpha_plus) out.alpha_plus[p] = sm.ap[i];
    if (out.alpha_minus) out.alpha_minus[p] = sm.am[i];
    if (out.alpha_occ) out.alpha_occ[p] = aocc;
    if (out.raw_occ) out.raw_occ[p] = raw;
    if (out.inside_sphere) out.inside_sphere[p] = inside;
    if (out.gradients_flip) {
#pragma unroll
      for (int c = 0; c < 3; ++c) out.gradients_flip[p * 3 + c] = gq.flip * g[c];
    }
  }
  __device__ __forceinline__ void bg(int i, int64_t q, float w, const float col[3]) {
    weight(i, w);
#pragma unroll
    for (int c = 0; c < 3; ++c) cb[c] = __fmaf_rn(w, col[c], cb[c]);
  }
};

template <int RULE>
__global__ void __launch_bounds__(RK_WARPS * 32)
composite_forward_kernel(nudf_render_cfg cfg, RayIn in, nudf_render_out out) {
  extern __shared__ float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * RK_WARPS + warp;
  if (r >= cfg.n_rays) return;
  const int S = cfg.n_samples, O = cfg.n_outside, SO = S + O;
  RaySmem sm = carve(smem + (size_t)warp * RK_ARRAYS * SO, SO);
  ray_forward_state<RULE>(cfg, in, r, lane, sm);

  CoreExtra ex(cfg, in, out, sm, r);
  const RaySums s = ray_composite(cfg, in, r, lane, sm, ex);
  float* cb = ex.cb; float* nrm = ex.nrm;
  const float* cc = s.cc;
  const float depth = s.depth, ws_fg = s.ws_fg, ws_all = s.ws_all;
#pragma unroll
  for (int c = 0; c < 3; ++c) { cb[c] = warp_sum(cb[c]); nrm[c] = warp_sum(nrm[c]); }
  const float s_relax_ge = warp_sum(ex.s_relax_ge), s_relax = warp_sum(ex.s_relax), s_near_ge = warp_sum(ex.s_near_ge);
  const float s_near = warp_sum(ex.s_near), s_sparse = warp_sum(ex.s_sparse);
  if (lane == 0) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      if (out.color_base) out.color_base[r * 3 + c] = cb[c];
      if (out.color) out.color[r * 3 + c] = ray_color(cfg, s, c);
      if (out.normals) out.normals[r * 3 + c] = nrm[c];
    }
    if (out.depth) out.depth[r] = depth;
    if (out.weight_sum) out.weight_sum[r] = ws_fg;
    if (out.weight_sum_fg_bg) out.weight_sum_fg_bg[r] = ws_all;
    if (out.ray_sums) {
      float* rs = out.ray_sums + (int64_t)r * 5;
      rs[0] = s_relax_ge; rs[1] = s_relax; rs[2] = s_near_ge; rs[3] = s_near; rs[4] = s_sparse;
    }
    // the reference drops into pdb on a NaN eikonal term (udf_renderer_blending.py:543-544); here a device flag is raised
    // and the Python wrapper turns it into a RuntimeError at its next host read
    if (out.status != nullptr) {
      const float chk = cc[0] + cc[1] + cc[2] + cb[0] + cb[1] + cb[2] + depth + ws_all + s_relax_ge + s_near_ge + s_sparse;
      if (!isfinite(chk)) atomicOr(out.status, NUDF_STATUS_NONFINITE_RENDER);
    }
  }
}

// The view renderer's per-sample terms: the pixel-blend composite and validate()'s normal map
// (exp_runner_blending.py:641-668: sum of gradients_flip * weights * inside_sphere over the foreground samples).
struct ViewExtra {
  const RayIn& in; const float* c_pix; int64_t row;   // row = r * (S + O): first background column of the ray
  int has_bg;
  float cp[3] = {0, 0, 0}, nrm[3] = {0, 0, 0};
  __device__ ViewExtra(const RayIn& in_, const float* c_pix_, int64_t row_, int has_bg_)
      : in(in_), c_pix(c_pix_), row(row_), has_bg(has_bg_) {}
  __device__ __forceinline__ void fg(int i, int64_t p, float w, float u, const float g[3], const GradQ& gq) {
    const bool inside = sample_norm(in, p) < 1.0f;
    if (inside) {
#pragma unroll
      for (int c = 0; c < 3; ++c) nrm[c] += gq.flip * g[c] * w;
    }
    if (c_pix) {
      // outside the unit sphere the blended colour is replaced by the NeRF++ colour of the same column (:503-507)
      const int64_t q = row + i;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float col = (has_bg && !inside) ? in.bg_color[q * 3 + c] : c_pix[p * 3 + c];
        cp[c] += col * w;
      }
    }
  }
  __device__ __forceinline__ void bg(int i, int64_t q, float w, const float col[3]) {
#pragma unroll
    for (int c = 0; c < 3; ++c) cp[c] += col[c] * w;
  }
};

struct ViewArgs {
  const float* c_pix;   // [N*S,3] or null
  float rot[9];         // row-major camera-from-world rotation of the normal map
  nudf_view_out out;
};

template <int RULE>
__global__ void __launch_bounds__(RK_WARPS * 32)
view_forward_kernel(nudf_render_cfg cfg, RayIn in, ViewArgs va) {
  extern __shared__ float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * RK_WARPS + warp;
  if (r >= cfg.n_rays) return;
  const int S = cfg.n_samples, O = cfg.n_outside, SO = S + O;
  RaySmem sm = carve(smem + (size_t)warp * RK_ARRAYS * SO, SO);
  ray_forward_state<RULE>(cfg, in, r, lane, sm);

  ViewExtra ex(in, va.c_pix, (int64_t)r * SO, O > 0);
  const RaySums s = ray_composite(cfg, in, r, lane, sm, ex);
  float cp[3], nw[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) { cp[c] = warp_sum(ex.cp[c]); nw[c] = warp_sum(ex.nrm[c]); }
  if (lane == 0) {
    const nudf_view_out& o = va.out;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      if (o.color) o.color[r * 3 + c] = ray_color(cfg, s, c);
      if (o.color_pixel) o.color_pixel[r * 3 + c] = cp[c];
      if (o.normal) o.normal[r * 3 + c] = va.rot[c * 3 + 0] * nw[0] + va.rot[c * 3 + 1] * nw[1] + va.rot[c * 3 + 2] * nw[2];
    }
    if (o.depth) o.depth[r] = s.depth;
    if (o.weight_sum) o.weight_sum[r] = s.ws_fg;
  }
}

struct RayBwdOut {
  float* udf_bar; float* grads_bar; float* scb_bar; float* sc_bar; float* bg_alpha_bar; float* bg_color_bar;
  float* scalar_bar;
};
struct RayBar {
  const float* color_base; const float* color; const float* depth; const float* weight_sum; const float* weight_sum_fg_bg;
  const float* weights;   // [N, S+O] or null
  const float* ray_sums;  // [N,5] upstream gradient of the per-ray regulariser sums
};

template <int RULE>
__global__ void __launch_bounds__(RK_WARPS * 32)
composite_backward_kernel(nudf_render_cfg cfg, RayIn in, RayBar bar, RayBwdOut out) {
  extern __shared__ float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * RK_WARPS + warp;
  if (r >= cfg.n_rays) return;
  const int S = cfg.n_samples, O = cfg.n_outside, SO = S + O;
  RaySmem sm = carve(smem + (size_t)warp * RK_ARRAYS * SO, SO);
  ray_forward_state<RULE>(cfg, in, r, lane, sm);

  const int64_t base = (int64_t)r * S;
  const float d[3] = {in.rays_d[r * 3 + 0], in.rays_d[r * 3 + 1], in.rays_d[r * 3 + 2]};
  float cbb[3], ccb[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    cbb[c] = bar.color_base ? bar.color_base[r * 3 + c] : 0.f;
    ccb[c] = bar.color ? bar.color[r * 3 + c] : 0.f;
  }
  const float depth_b = bar.depth ? bar.depth[r] : 0.f;
  const float wsfg_b = bar.weight_sum ? bar.weight_sum[r] : 0.f;
  float wsall_b = bar.weight_sum_fg_bg ? bar.weight_sum_fg_bg[r] : 0.f;
  if (cfg.has_background_rgb)
    wsall_b -= ccb[0] * cfg.background_rgb[0] + ccb[1] * cfg.background_rgb[1] + ccb[2] * cfg.background_rgb[2];

  const float inv_s = in.heads[0], beta = in.heads[1], gamma = in.heads[2];
  // the caller forms gradient_error = sum(rs0)/(sum(rs1)+1e-5) etc. from ray_sums (:533-536, :553); its autograd hands
  // back d loss / d ray_sums, whose columns 0, 2, 4 are the per-sample coefficients needed here.
  float ge_coef = 0.f, ge_ns_coef = 0.f, sparse_coef = 0.f;
  if (bar.ray_sums) {
    ge_coef = bar.ray_sums[(int64_t)r * 5 + 0];
    ge_ns_coef = bar.ray_sums[(int64_t)r * 5 + 2];
    sparse_coef = bar.ray_sums[(int64_t)r * 5 + 4];
  }
  // ---- wbar per sample; colour adjoints ----
  for (int i = lane; i < SO; i += 32) {
    float w = sm.alpha[i] * sm.T[i];
    float wb = wsall_b;
    if (bar.weights) wb += bar.weights[(int64_t)r * SO + i];
    if (i < S) {
      const int64_t p = base + i;
      float dcb = 0.f, dcc = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        dcb += cbb[c] * in.scb[p * 3 + c];
        dcc += ccb[c] * in.sc[p * 3 + c];
        out.scb_bar[p * 3 + c] = w * cbb[c];
        out.sc_bar[p * 3 + c] = w * ccb[c];
      }
      wb += dcb + dcc + depth_b * in.mid_z[p] + wsfg_b;
    } else {
      const int64_t q = (int64_t)r * SO + i;
      float dc = 0.f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        dc += (cbb[c] + ccb[c]) * in.bg_color[q * 3 + c];
        if (out.bg_color_bar) out.bg_color_bar[q * 3 + c] = w * (cbb[c] + ccb[c]);
      }
      wb += dc;
    }
    sm.wbar[i] = wb;
  }
  __syncwarp();
  // ---- reverse scan:  B_i = wbar_i alpha_i + f_i B_{i+1} ;  alpha_bar_i = T_i (wbar_i - B_{i+1}) ----
  {
    float carry = 0.f;  // B at the first sample of the chunk to the right
    int nchunk = (SO + 31) / 32;
    for (int ch = nchunk - 1; ch >= 0; --ch) {
      int i = ch * 32 + lane;
      float a = 0.f, f = 1.f;
      if (i < SO) { a = sm.wbar[i] * sm.alpha[i]; f = 1.0f - sm.alpha[i] + 1e-7f; }
      warp_rscan_affine(a, f, lane);
      float Bi = a + f * carry;                       // B_i
      float Bn = __shfl_down_sync(FULL, Bi, 1);       // B_{i+1}
      if (lane == 31) Bn = carry;
      if (i < SO) sm.abar[i] = sm.T[i] * (sm.wbar[i] - Bn);
      carry = __shfl_sync(FULL, Bi, 0);
    }
  }
  __syncwarp();
  if (out.bg_alpha_bar)
    for (int i = lane; i < SO; i += 32) out.bg_alpha_bar[(int64_t)r * SO + i] = (i < S) ? 0.f : sm.abar[i];
  // ---- vis_prob adjoint and its reverse scan: R_i = Pbar_i + t_i R_{i+1} ; t_bar_i = P_i R_{i+1} ----
  // (re-use wbar[] for Pbar, then for t_bar)
  for (int i = lane; i < S; i += 32) {
    float P = sm.P[i];
    float vb = sm.abar[i] * (sm.ap[i] - sm.am[i]);
    sm.wbar[i] = (P >= 0.0f && P <= 1.0f) ? vb : 0.0f;
  }
  __syncwarp();
  {
    float carry = 0.f;
    int nchunk = (S + 31) / 32;
    for (int ch = nchunk - 1; ch >= 0; --ch) {
      int i = ch * 32 + lane;
      float a = 0.f, f = 1.f;
      if (i < S) { a = sm.wbar[i]; f = sm.t[i]; }
      warp_rscan_affine(a, f, lane);
      float Ri = a + f * carry;
      float Rn = __shfl_down_sync(FULL, Ri, 1);
      if (lane == 31) Rn = carry;
      __syncwarp();
      if (i < S) sm.wbar[i] = sm.P[i] * Rn;            // t_bar_i  (each lane overwrites only its own slot)
      carry = __shfl_sync(FULL, Ri, 0);
    }
  }
  __syncwarp();
  // ---- per-sample chain rule ----
  float s_bar = 0.f, beta_bar = 0.f, gamma_bar = 0.f;
  for (int i = lane; i < S; i += 32) {
    const int64_t p = base + i;
    float u = in.udf[p * in.ld_udf];
    float dist = in.dists[p];
    const float g[3] = {in.grads[p * 3 + 0], in.grads[p * 3 + 1], in.grads[p * 3 + 2]};
    float tc = sm.tc[i];
    float vis = clampf_(sm.P[i], 0.0f, 1.0f);
    float ab = sm.abar[i];
    float ap_bar = ab * vis, am_bar = ab * (1.0f - vis);
    float ic = iter_cos_forward(tc, cfg.has_cos_anneal, cfg.cos_anneal_ratio);
    float sdf_b1, ic_b1, s_b1, sdf_b2, ic_b2, s_b2;
    alpha_backward<RULE>(u, ic, dist, inv_s, ap_bar, &sdf_b1, &ic_b1, &s_b1);
    alpha_backward<RULE>(-u, ic, dist, inv_s, am_bar, &sdf_b2, &ic_b2, &s_b2);
    float u_bar = sdf_b1 - sdf_b2;
    s_bar += s_b1 + s_b2;
    float tc_bar = (ic_b1 + ic_b2) * iter_cos_dtc(tc, cfg.has_cos_anneal, cfg.cos_anneal_ratio);
    // visibility factor: t = clip(q,0,1)+1e-7, q = 1 - aocc + fs*vm
    float q = sm.q[i];
    float q_bar = (q >= 0.0f && q <= 1.0f) ? sm.wbar[i] : 0.0f;
    float ub2, bb, gb;
    occ_backward(u, dist, beta, gamma, -q_bar, &ub2, &bb, &gb);
    u_bar += ub2; beta_bar += bb; gamma_bar += gb;
    // regularisers
    float px = in.pts[p * 3 + 0], py = in.pts[p * 3 + 1], pz = in.pts[p * 3 + 2];
    float pn = sqrtf(px * px + py * py + pz * pz);
    float eik = (pn < 1.2f ? ge_coef : 0.f) + (u < 0.05f ? ge_ns_coef : 0.f);
    u_bar += sparse_coef * (-cfg.sparse_scale_factor) * expf(-cfg.sparse_scale_factor * u);
    float gb3[3];
    grad_quantities_backward(g, d, cfg.use_norm_grad_for_cosine, tc_bar, eik, gb3);
    out.udf_bar[p] = u_bar;
#pragma unroll
    for (int c = 0; c < 3; ++c) out.grads_bar[p * 3 + c] = gb3[c];
  }
  s_bar = warp_sum(s_bar); beta_bar = warp_sum(beta_bar); gamma_bar = warp_sum(gamma_bar);
  if (lane == 0 && out.scalar_bar) {
    out.scalar_bar[r * 3 + 0] = s_bar; out.scalar_bar[r * 3 + 1] = beta_bar; out.scalar_bar[r * 3 + 2] = gamma_bar;
  }
}

}  // namespace nudf

using namespace nudf;

extern "C" {

int nudf_ray_points(const float* rays_o, const float* rays_d, const float* z_vals, int32_t n_rays, int32_t n_samples,
                    float sample_dist, float* pts, float* mid_z, float* dists, void* stream) {
  NUDF_REQUIRE(rays_o && rays_d && z_vals, "null pointer");
  if (n_rays <= 0 || n_samples <= 0) return 0;
  int64_t n = (int64_t)n_rays * n_samples;
  ray_points_kernel<<<(unsigned)cdiv(n, 256), 256, 0, (cudaStream_t)stream>>>(rays_o, rays_d, z_vals, n_rays, n_samples,
                                                                             sample_dist, pts, mid_z, dists);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_points_on_rays(const float* rays_o, const float* rays_d, const float* z, int32_t n_rays, int32_t n, float* pts,
                        void* stream) {
  NUDF_REQUIRE(rays_o && rays_d && z && pts, "null pointer");
  if (n_rays <= 0 || n <= 0) return 0;
  int64_t tot = (int64_t)n_rays * n;
  points_on_rays_kernel<<<(unsigned)cdiv(tot, 256), 256, 0, (cudaStream_t)stream>>>(rays_o, rays_d, z, n_rays, n, pts);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_outside_points(const float* rays_o, const float* rays_d, const float* z, int32_t n_rays, int32_t n, int32_t col0,
                        float sample_dist, float* pts4, float* dists, void* stream) {
  NUDF_REQUIRE(rays_o && rays_d && z && pts4 && dists, "null pointer");
  NUDF_REQUIRE(col0 >= 0 && col0 < n, "col0 out of range");
  if (n_rays <= 0) return 0;
  int64_t tot = (int64_t)n_rays * (n - col0);
  outside_points_kernel<<<(unsigned)cdiv(tot, 256), 256, 0, (cudaStream_t)stream>>>(rays_o, rays_d, z, n_rays, n, col0,
                                                                                   sample_dist, pts4, dists);
  NUDF_LAUNCH_OK();
  return 0;
}

}  // extern "C"

namespace {

// dynamic shared memory of a ray kernel: RK_ARRAYS per-sample arrays per warp
size_t ray_smem(const nudf_render_cfg& cfg) {
  return (size_t)RK_WARPS * RK_ARRAYS * (cfg.n_samples + cfg.n_outside) * sizeof(float);
}

// The alpha rule is checked first, so that a bad rule is refused before any pointer is looked at.
int check_cfg(const nudf_render_cfg* cfg, const float* bg_alpha, const float* bg_color) {
  NUDF_REQUIRE(cfg != nullptr, "null cfg");
  NUDF_REQUIRE(cfg->alpha_rule == ALPHA_NUMERICAL || cfg->alpha_rule == ALPHA_THEORICAL,
               "alpha_rule must be 0 (numerical) or 1 (theorical)");
  NUDF_REQUIRE(cfg->n_samples > 0 && cfg->n_outside >= 0, "bad sample counts");
  NUDF_REQUIRE(cfg->n_outside == 0 || (bg_alpha && bg_color), "n_outside > 0 needs bg_alpha / bg_color");
  NUDF_REQUIRE(ray_smem(*cfg) <= 200 * 1024, "too many samples per ray for the compositing kernel (max ~1280)");
  return 0;
}

// Launches the instantiation of a ray kernel for the cfg's alpha rule, one warp per ray.
template <class... A>
int launch_rays(void (*numerical)(nudf_render_cfg, RayIn, A...), void (*theorical)(nudf_render_cfg, RayIn, A...),
                const nudf_render_cfg* cfg, const RayIn& in, cudaStream_t st, const A&... args) {
  const auto kernel = cfg->alpha_rule == ALPHA_THEORICAL ? theorical : numerical;
  const size_t smem = ray_smem(*cfg);
  if (smem > 48 * 1024)
    NUDF_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  LaunchTimer lt_(FAM_RAY, st);
  kernel<<<(unsigned)cdiv(cfg->n_rays, RK_WARPS), RK_WARPS * 32, smem, st>>>(*cfg, in, args...);
  NUDF_LAUNCH_OK();
  return 0;
}

}  // namespace

extern "C" {

int nudf_render_composite_forward(const nudf_render_cfg* cfg, const float* heads, const float* rays_d, const float* pts,
                                  const float* mid_z, const float* dists, const float* udf, int64_t ld_udf,
                                  const float* grads, const float* sampled_color_base, const float* sampled_color,
                                  const float* bg_alpha, const float* bg_color, const nudf_render_out* out, void* stream) {
  if (int rc = check_cfg(cfg, bg_alpha, bg_color)) return rc;
  NUDF_REQUIRE(heads && rays_d && pts && mid_z && dists && udf && grads && sampled_color_base && sampled_color && out, "null pointer");
  if (cfg->n_rays <= 0) return 0;
  RayIn in{heads, rays_d, pts, mid_z, dists, udf, ld_udf, grads, sampled_color_base, sampled_color, bg_alpha, bg_color};
  return launch_rays(composite_forward_kernel<ALPHA_NUMERICAL>, composite_forward_kernel<ALPHA_THEORICAL>, cfg, in,
                     (cudaStream_t)stream, *out);
}

int nudf_render_view_forward(const nudf_render_cfg* cfg, const float* heads, const float* rays_d, const float* pts,
                             const float* mid_z, const float* dists, const float* udf, int64_t ld_udf, const float* grads,
                             const float* sampled_color, const float* c_pix, const float* bg_alpha, const float* bg_color,
                             const float* rot, const nudf_view_out* out, void* stream) {
  if (int rc = check_cfg(cfg, bg_alpha, bg_color)) return rc;
  NUDF_REQUIRE(heads && rays_d && pts && mid_z && dists && udf && grads && sampled_color && rot && out, "null pointer");
  if (cfg->n_rays <= 0) return 0;
  RayIn in{heads, rays_d, pts, mid_z, dists, udf, ld_udf, grads, nullptr, sampled_color, bg_alpha, bg_color};
  ViewArgs va;
  va.c_pix = c_pix;
  for (int k = 0; k < 9; ++k) va.rot[k] = rot[k];
  va.out = *out;
  return launch_rays(view_forward_kernel<ALPHA_NUMERICAL>, view_forward_kernel<ALPHA_THEORICAL>, cfg, in,
                     (cudaStream_t)stream, va);
}

int nudf_render_composite_backward(const nudf_render_cfg* cfg, const float* heads, const float* rays_d, const float* pts,
                                   const float* mid_z, const float* dists, const float* udf, int64_t ld_udf,
                                   const float* grads, const float* sampled_color_base, const float* sampled_color,
                                   const float* bg_alpha, const float* bg_color, const nudf_render_bar* bar,
                                   float* udf_bar, float* grads_bar, float* scb_bar, float* sc_bar, float* bg_alpha_bar,
                                   float* bg_color_bar, float* scalar_bar, void* stream) {
  if (int rc = check_cfg(cfg, bg_alpha, bg_color)) return rc;
  NUDF_REQUIRE(heads && rays_d && pts && mid_z && dists && udf && grads && sampled_color_base && sampled_color && bar, "null pointer");
  NUDF_REQUIRE(udf_bar && grads_bar && scb_bar && sc_bar, "null output pointer");
  if (cfg->n_rays <= 0) return 0;
  RayIn in{heads, rays_d, pts, mid_z, dists, udf, ld_udf, grads, sampled_color_base, sampled_color, bg_alpha, bg_color};
  RayBar rb;
  rb.color_base = bar->color_base; rb.color = bar->color; rb.depth = bar->depth; rb.weight_sum = bar->weight_sum;
  rb.weight_sum_fg_bg = bar->weight_sum_fg_bg;
  rb.weights = bar->weights;
  rb.ray_sums = bar->ray_sums;
  RayBwdOut ob{udf_bar, grads_bar, scb_bar, sc_bar, bg_alpha_bar, bg_color_bar, scalar_bar};
  return launch_rays(composite_backward_kernel<ALPHA_NUMERICAL>, composite_backward_kernel<ALPHA_THEORICAL>, cfg, in,
                     (cudaStream_t)stream, rb, ob);
}

}  // extern "C"

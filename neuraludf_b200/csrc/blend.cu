// Fused pixel / patch blending of the fine-tuning stage (SURVEY 8(f) rank 1): per sample point, project into every source
// view, gather the pixel colour and the homography-warped (2h+1)^2 patch (h <= 5: up to 11x11, the fine-tuning conf's
// h_patch_size = 5) with bilinear taps, and fuse the views with the masked, renormalised softmax of the colour network's
// blending logits -- without materialising the [N,S,V,Npx,3] colour tensor (616 MB at 1024 rays x 128 samples x 8 views
// x 49 pixels) that the op-by-op formulation reads and writes many times.
// One warp per point: lanes = views for the pixel part, lanes = patch pixels for the patch part (PPL pixels per lane,
// q = lane + 32 k for k < PPL: PPL = 2 up to 64 pixels, h <= 3; PPL = 4 up to 128 pixels, h = 4, 5).
// Reference semantics: see blendmath.cuh.  The backward pass re-gathers instead of storing per-view colours; gradients flow
// to the blending logits only (sample positions, normals and homographies are constants of the graph, like in the
// reference: z_vals are detached, the normals are detached, the homographies are built under no_grad).
#include "../../include/nudf.h"
#include "blendmath.cuh"
#include "common.cuh"

namespace nudf {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

struct BlendPtrs {
  const float* pts; const float* proj; const float* hom; const float* px; const float* imgs; const float* logits; int64_t ld_logits;
};

// softmax over the first V logits of point p: lane v holds sm_v (0 for lanes >= V)
__device__ __forceinline__ float lane_softmax(const BlendPtrs& b, int64_t p, int V, int lane) {
  const float lg = lane < V ? b.logits[p * b.ld_logits + lane] : -INFINITY;
  const float mx = warp_max(lg);
  const float e = lane < V ? expf(lg - mx) : 0.f;
  return e / warp_sum(e);
}

// patch pixel q of a (2h+1)^2 patch around (u0, v0): dx fastest
__device__ __forceinline__ void patch_pixel(int q, int side, int h, float u0, float v0, float* u, float* v) {
  *u = u0 + (float)(q % side - h);
  *v = v0 + (float)(q / side - h);
}

// sum over a lane's PPL patch pixels of <g_k, c_k>, added left to right with the three products of each pixel in turn
template <int PPL>
__device__ __forceinline__ float lane_dot(const float (&g)[PPL][3], const float (&c)[PPL][3]) {
  float s = g[0][0] * c[0][0] + g[0][1] * c[0][1] + g[0][2] * c[0][2];
#pragma unroll
  for (int k = 1; k < PPL; ++k) s = s + g[k][0] * c[k][0] + g[k][1] * c[k][1] + g[k][2] * c[k][2];
  return s;
}

// PPL patch pixels per lane: the patch has at most 32 * PPL pixels
template <bool BWD, int PPL>
__global__ void __launch_bounds__(256)
blend_kernel(nudf_blend_cfg c, BlendPtrs b, float* __restrict__ c_pix, float* __restrict__ c_pat, float* __restrict__ m_pat,
             const float* __restrict__ g_pix, const float* __restrict__ g_pat, float* __restrict__ g_logits) {
  const int64_t P = (int64_t)c.n_rays * c.n_samples;
  const int64_t p = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (p >= P) return;
  const int V = c.n_views, H = c.height, W = c.width;
  const int64_t img_stride = (int64_t)3 * H * W;
  const float sm = lane_softmax(b, p, V, lane);
  const float pt[3] = {b.pts[p * 3 + 0], b.pts[p * 3 + 1], b.pts[p * 3 + 2]};
  float dsm = 0.f;                                  // BWD: d loss / d sm_lane

  // ---- pixel colours: lane v = view v ----
  {
    float a = 0.f, col[3] = {0.f, 0.f, 0.f};
    if (lane < V) {
      float ix, iy;
      if (pixel_project(b.proj + lane * 12, pt, H, W, &ix, &iy)) {
        bilinear3(b.imgs + lane * img_stride, H, W, ix, iy, col);
        a = sm;
      }
    }
    const float A = warp_sum(a);
    const float w = a / (A + 1e-8f);
    float cp[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) cp[k] = warp_sum(w * col[k]);
    if (!BWD) {
      if (lane < 3) c_pix[p * 3 + lane] = lane == 0 ? cp[0] : (lane == 1 ? cp[1] : cp[2]);
    } else if (g_pix != nullptr) {
      const float g[3] = {g_pix[p * 3 + 0], g_pix[p * 3 + 1], g_pix[p * 3 + 2]};
      const float t = g[0] * col[0] + g[1] * col[1] + g[2] * col[2];
      const float gc = g[0] * cp[0] + g[1] * cp[1] + g[2] * cp[2];
      if (a != 0.f) dsm += (t - gc) / (A + 1e-8f);          // valid view (a = sm_v > 0); invalid views get no gradient
    }
  }

  // ---- patch colours: lanes = patch pixels q = lane + 32 k (k < PPL); views in sequence ----
  if (b.hom != nullptr) {
    const int h = c.h_patch, side = 2 * h + 1, npx = side * side;
    const int64_t n = p / c.n_samples;
    const float u0 = b.px[n * 2 + 0], v0 = b.px[n * 2 + 1];
    int q[PPL];
    float u[PPL], v[PPL], acc[PPL][3], g[PPL][3];
#pragma unroll
    for (int k = 0; k < PPL; ++k) {
      q[k] = lane + 32 * k;
      patch_pixel(q[k], side, h, u0, v0, &u[k], &v[k]);
    }
#pragma unroll
    for (int k = 0; k < PPL; ++k) acc[k][0] = acc[k][1] = acc[k][2] = g[k][0] = g[k][1] = g[k][2] = 0.f;
    if (BWD && g_pat != nullptr) {
#pragma unroll
      for (int k = 0; k < PPL; ++k) {
        if (q[k] < npx) { g[k][0] = g_pat[(p * npx + q[k]) * 3 + 0]; g[k][1] = g_pat[(p * npx + q[k]) * 3 + 1]; g[k][2] = g_pat[(p * npx + q[k]) * 3 + 2]; }
      }
    }
    float Apat = 0.f;
    float tv = 0.f;                                   // BWD: lane v keeps t_v = <g_pat, col_v> if view v is valid
    bool valid_me = false;                            // lane v: is view v valid
    for (int vw = 0; vw < V; ++vw) {
      const float* hp = b.hom + ((int64_t)vw * P + p) * 9;
      float hm[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) hm[k] = hp[k];
      float ix[PPL], iy[PPL];
      bool m_all = true;                              // every pixel of this lane inside view vw
#pragma unroll
      for (int k = 0; k < PPL; ++k) {
        ix[k] = iy[k] = 0.f;
        const bool m = q[k] < npx ? patch_warp_pixel(hm, u[k], v[k], H, W, h, &ix[k], &iy[k]) : true;
        m_all = m_all && m;
      }
      const bool all_in = __all_sync(0xffffffffu, m_all);
      if (!all_in) continue;                          // warp-uniform
      const float smv = __shfl_sync(0xffffffffu, sm, vw);
      Apat += smv;
      float col[PPL][3];
#pragma unroll
      for (int k = 0; k < PPL; ++k) {
        col[k][0] = col[k][1] = col[k][2] = 0.f;
        if (q[k] < npx) bilinear3(b.imgs + vw * img_stride, H, W, ix[k], iy[k], col[k]);
      }
#pragma unroll
      for (int k = 0; k < PPL; ++k) {
#pragma unroll
        for (int j = 0; j < 3; ++j) acc[k][j] += smv * col[k][j];
      }
      if (BWD) {
        const float t = warp_sum(lane_dot<PPL>(g, col));
        if (lane == vw) { tv = t; valid_me = true; }
      }
    }
    const float inv = 1.0f / (Apat + 1e-8f);
    if (!BWD) {
#pragma unroll
      for (int k = 0; k < PPL; ++k) {
        if (q[k] < npx) { float* o = c_pat + (p * npx + q[k]) * 3; o[0] = acc[k][0] * inv; o[1] = acc[k][1] * inv; o[2] = acc[k][2] * inv; }
      }
      if (lane == 0) m_pat[p] = Apat > 0.f ? 1.0f : 0.0f;
    } else if (g_pat != nullptr) {
      const float gc = warp_sum(lane_dot<PPL>(g, acc) * inv);
      if (valid_me) dsm += (tv - gc) * inv;
    }
  }

  if (BWD) {
    // softmax backward: d loss / d logit_v = sm_v (dsm_v - sum_u sm_u dsm_u)
    const float s = warp_sum(sm * dsm);
    if (lane < V) g_logits[p * V + lane] = sm * (dsm - s);
  }
}

// patch pixels per lane for a (2h+1)^2 patch (check_cfg admits at most 128 pixels)
static int pixels_per_lane(int h_patch) { return (2 * h_patch + 1) * (2 * h_patch + 1) <= 64 ? 2 : 4; }

static int check_cfg(const nudf_blend_cfg* c) {
  NUDF_REQUIRE(c != nullptr, "null cfg");
  NUDF_REQUIRE(c->n_rays >= 0 && c->n_samples >= 0, "negative sizes");
  NUDF_REQUIRE(c->n_views >= 1 && c->n_views <= 32, "n_views must be in 1..32");
  NUDF_REQUIRE(c->height >= 2 && c->width >= 2, "images must be at least 2 x 2");
  NUDF_REQUIRE(c->h_patch >= 0 && c->h_patch <= 5, "h_patch must be in 0..5 (patches of at most 11 x 11 = 121 pixels)");
  return 0;
}

}  // namespace nudf

using namespace nudf;

extern "C" {

int nudf_blend_forward(const nudf_blend_cfg* cfg, const float* pts, const float* proj, const float* hom, const float* px,
                       const float* imgs, const float* logits, int64_t ld_logits, float* c_pix, float* c_pat, float* m_pat,
                       void* stream) {
  if (int rc = check_cfg(cfg)) return rc;
  const int64_t P = (int64_t)cfg->n_rays * cfg->n_samples;
  if (P == 0) return 0;
  NUDF_REQUIRE(pts && proj && imgs && logits && c_pix, "null pointer");
  NUDF_REQUIRE(ld_logits >= cfg->n_views, "ld_logits < n_views");
  NUDF_REQUIRE(hom == nullptr || (px && c_pat && m_pat), "patch blending needs px, c_pat and m_pat");
  BlendPtrs b{pts, proj, hom, px, imgs, logits, ld_logits};
  const int64_t threads = P * 32;
  const unsigned grid = (unsigned)cdiv(threads, 256);
  if (pixels_per_lane(cfg->h_patch) == 2)
    blend_kernel<false, 2><<<grid, 256, 0, (cudaStream_t)stream>>>(*cfg, b, c_pix, c_pat, m_pat, nullptr, nullptr, nullptr);
  else
    blend_kernel<false, 4><<<grid, 256, 0, (cudaStream_t)stream>>>(*cfg, b, c_pix, c_pat, m_pat, nullptr, nullptr, nullptr);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_blend_backward(const nudf_blend_cfg* cfg, const float* pts, const float* proj, const float* hom, const float* px,
                        const float* imgs, const float* logits, int64_t ld_logits, const float* g_pix, const float* g_pat,
                        float* g_logits, void* stream) {
  if (int rc = check_cfg(cfg)) return rc;
  const int64_t P = (int64_t)cfg->n_rays * cfg->n_samples;
  if (P == 0) return 0;
  NUDF_REQUIRE(pts && proj && imgs && logits && g_logits, "null pointer");
  NUDF_REQUIRE(ld_logits >= cfg->n_views, "ld_logits < n_views");
  NUDF_REQUIRE(hom == nullptr || px, "patch blending needs px");
  BlendPtrs b{pts, proj, hom, px, imgs, logits, ld_logits};
  const int64_t threads = P * 32;
  const unsigned grid = (unsigned)cdiv(threads, 256);
  const float* gp = hom ? g_pat : nullptr;
  if (pixels_per_lane(cfg->h_patch) == 2)
    blend_kernel<true, 2><<<grid, 256, 0, (cudaStream_t)stream>>>(*cfg, b, nullptr, nullptr, nullptr, g_pix, gp, g_logits);
  else
    blend_kernel<true, 4><<<grid, 256, 0, (cudaStream_t)stream>>>(*cfg, b, nullptr, nullptr, nullptr, g_pix, gp, g_logits);
  NUDF_LAUNCH_OK();
  return 0;
}

}  // extern "C"

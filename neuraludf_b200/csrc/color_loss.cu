// The runner's colour loss on the device (loss/loss.py ColorLoss + loss/patch_metric.py SSIM / NCC), driven by
// neuraludf_b200/loss.py.  tests/proto/color_loss.py restates the forward and the hand-derived backward in NumPy fp64.
//   ray pass     one warp per ray, lanes stride over the patch pixels: the three pixel L1 sums of the ray and its patch
//                error (l1, ssd, ssim or ncc; every Gaussian-window moment is one weighted sum per channel, the convolution
//                having padding 0 over the whole patch).  Moments and the per-ray formulas are evaluated in fp64, rounded
//                to fp32 once per ray.
//   rejection    one CTA: k = int(0.3f * count(mask)); the first k rays of the descending order of error * mask are
//                excluded (NaN ranks largest, -0 equals +0, equal keys in ray order); the kept masked rays are
//                averaged (an empty kept set gives NaN).  Writes the five scalars and what the backward needs.
//   backward     one warp per ray: d/d pred of the three pixel terms and of the patch term, from the upstream gradients of
//                the five scalars.
// Every reduction has one fixed order (per-lane strided sums, xor butterflies, warp partials summed by warp 0), so the
// same inputs give the same bits on every run.
#include "../../include/nudf.h"
#include "common.cuh"

namespace nudf {
namespace cl {

constexpr int kRejectThreads = 1024;
constexpr int kMaxRays = 16384;             // keys of the rejection CTA live in shared memory (64 KB)
constexpr double C1 = 0.01 * 0.01, C2 = 0.03 * 0.03;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Gaussian-window moments of one ray's patch, per channel: mu1 = sum w x, mu2 = sum w y, xx = sum w x^2, yy = sum w y^2,
// xy = sum w x y (identical on every lane)
struct Moments {
  double mu1[3], mu2[3], xx[3], yy[3], xy[3];
};

__device__ __forceinline__ void moments(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ w,
                                        int npx, int lane, Moments& m) {
#pragma unroll
  for (int c = 0; c < 3; ++c) m.mu1[c] = m.mu2[c] = m.xx[c] = m.yy[c] = m.xy[c] = 0.0;
  for (int p = lane; p < npx; p += 32) {
    const double wp = (double)w[p];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double xv = (double)x[3 * p + c], yv = (double)y[3 * p + c];
      m.mu1[c] += wp * xv;
      m.mu2[c] += wp * yv;
      m.xx[c] += wp * (xv * xv);
      m.yy[c] += wp * (yv * yv);
      m.xy[c] += wp * (xv * yv);
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    m.mu1[c] = warp_sum(m.mu1[c]);
    m.mu2[c] = warp_sum(m.mu2[c]);
    m.xx[c] = warp_sum(m.xx[c]);
    m.yy[c] = warp_sum(m.yy[c]);
    m.xy[c] = warp_sum(m.xy[c]);
  }
}

// NCC's second pass: T = sum w (x - mu1)(y - mu2) and U = sum w (y - mu2), per channel
__device__ __forceinline__ void ncc_sums(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ w,
                                         int npx, int lane, const Moments& m, double* T, double* U) {
#pragma unroll
  for (int c = 0; c < 3; ++c) T[c] = U[c] = 0.0;
  for (int p = lane; p < npx; p += 32) {
    const double wp = (double)w[p];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double dy = (double)y[3 * p + c] - m.mu2[c];
      T[c] += wp * (((double)x[3 * p + c] - m.mu1[c]) * dy);
      U[c] += wp * dy;
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    T[c] = warp_sum(T[c]);
    U[c] = warp_sum(U[c]);
  }
}

__device__ __forceinline__ double ncc_sigma(double xx, double mu) { return sqrt((xx - mu * mu) + 1e-4); }

// patch error of one ray (patch_metric.py _ssim / _ncc, loss.py:69-76); the same value on every lane
__device__ double patch_error(int type, const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ w,
                              int npx, int lane) {
  if (type == NUDF_PATCH_L1 || type == NUDF_PATCH_SSD) {
    double s = 0.0;
    for (int p = lane; p < npx; p += 32) {
      double r = 0.0;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double d = (double)x[3 * p + c] - (double)y[3 * p + c];
        r += type == NUDF_PATCH_L1 ? fabs(d) : d * d;
      }
      s += r / 3.0;
    }
    return warp_sum(s);
  }
  Moments m;
  moments(x, y, w, npx, lane, m);
  double e = 0.0;
  if (type == NUDF_PATCH_SSIM) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double m12 = m.mu1[c] * m.mu2[c], m11 = m.mu1[c] * m.mu1[c], m22 = m.mu2[c] * m.mu2[c];
      const double s1 = m.xx[c] - m11, s2 = m.yy[c] - m22, s12 = m.xy[c] - m12;
      e += 1.0 - ((2.0 * m12 + C1) * (2.0 * s12 + C2)) / ((m11 + m22 + C1) * (s1 + s2 + C2));
    }
    return e / 2.0;
  }
  double T[3], U[3];
  ncc_sums(x, y, w, npx, lane, m, T, U);
#pragma unroll
  for (int c = 0; c < 3; ++c)
    e += T[c] / ((ncc_sigma(m.xx[c], m.mu1[c]) + 1e-8) * (ncc_sigma(m.yy[c], m.mu2[c]) + 1e-8));
  return 1.0 - e / 3.0;
}

__global__ void ray_kernel(nudf_color_loss_args a, float* __restrict__ ws) {
  const int64_t ray = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int N = a.n_rays;
  if (ray >= N) return;
  const int side = 2 * a.h_patch + 1, npx = side * side;
  if (a.patch_colors) {
    const double e = patch_error(a.patch_type, a.patch_colors + ray * npx * 3, a.gt_patch_colors + ray * npx * 3, a.window,
                                 npx, lane);
    if (lane == 0) ws[ray] = (float)e;
  }
  if (lane < 3) {
    const float* p = lane == 0 ? a.color_base : (lane == 1 ? a.color : a.color_pixel);
    float s = 0.0f;
    if (p) s = (fabsf(p[3 * ray] - a.gt_color[3 * ray]) + fabsf(p[3 * ray + 1] - a.gt_color[3 * ray + 1])) +
               fabsf(p[3 * ray + 2] - a.gt_color[3 * ray + 2]);
    ws[(int64_t)(1 + lane) * N + ray] = s;
  }
}

// order-preserving unsigned key of error * mask: NaN above everything, -0 equal to +0
__device__ __forceinline__ uint32_t order_key(float v) {
  if (isnan(v)) return 0xffffffffu;
  const uint32_t b = __float_as_uint(v + 0.0f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// fixed-order block sum (every thread gets the result); `red` holds kRejectThreads / 32 doubles
__device__ __forceinline__ double block_sum(double v, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double t = lane < (int)(blockDim.x >> 5) ? red[lane] : 0.0;
  return warp_sum(t);
}

__global__ void __launch_bounds__(kRejectThreads) reject_kernel(nudf_color_loss_args a, float* __restrict__ losses,
                                                                 uint8_t* __restrict__ kept, float* __restrict__ ws) {
  extern __shared__ uint32_t keys[];
  __shared__ double red[kRejectThreads / 32];
  const int N = a.n_rays, tid = threadIdx.x;
  const float* err = ws;
  const bool patch = a.patch_colors != nullptr;
  double cnt = 0.0, pm_sum = 0.0, l1[3] = {0.0, 0.0, 0.0};
  for (int i = tid; i < N; i += blockDim.x) {
    const float m = a.patch_mask && a.patch_mask[i] ? 1.0f : 0.0f;
    cnt += m;
    if (a.pixel_mask) pm_sum += (double)a.pixel_mask[i];
#pragma unroll
    for (int t = 0; t < 3; ++t) l1[t] += (double)ws[(int64_t)(1 + t) * N + i];
    if (patch) keys[i] = order_key(err[i] * m);
  }
  cnt = block_sum(cnt, red);
  pm_sum = block_sum(pm_sum, red);
#pragma unroll
  for (int t = 0; t < 3; ++t) l1[t] = block_sum(l1[t], red);
  __syncthreads();
  // torch: 0.3 * (int64 count) is a float32 tensor, int() truncates it
  const int k = patch ? (int)__fmul_rn(0.3f, (float)cnt) : 0;
  double kept_sum = 0.0, n_kept = 0.0;
  if (patch) {
    for (int i = tid; i < N; i += blockDim.x) {
      uint8_t keep = 0;
      if (a.patch_mask[i]) {
        const uint32_t ki = keys[i];
        int rank = 0;                                    // rays ahead of i in the descending order
        for (int j = 0; j < N; ++j) {
          const uint32_t kj = keys[j];
          rank += (kj > ki) || (kj == ki && j < i);
        }
        keep = rank >= k;
      }
      kept[i] = keep;
      if (keep) {
        kept_sum += (double)err[i];
        n_kept += 1.0;
      }
    }
  }
  kept_sum = block_sum(kept_sum, red);
  n_kept = block_sum(n_kept, red);
  if (tid != 0) return;
  // the pixel terms' denominators: mask.sum() + 1e-4, or N * 3 (mean).  A bool mask's sum is an integer, so the reference
  // forms count + 1e-4 in fp32 whatever the precision of the predictions
  double* st = reinterpret_cast<double*>(ws + (int64_t)4 * N);
  st[0] = st[1] = a.pixel_mask ? pm_sum + 1e-4 : 3.0 * N;
  st[2] = a.patch_mask ? (double)__fadd_rn((float)cnt, 1e-4f) : 3.0 * N;
  st[3] = n_kept;
  const float* preds[3] = {a.color_base, a.color, a.color_pixel};
  double term[4];
  for (int t = 0; t < 3; ++t) term[t] = preds[t] ? (double)(float)(l1[t] / st[t]) : 0.0;
  term[3] = patch ? (double)(float)(kept_sum / n_kept) : 0.0;
  const double wsum = (double)a.weights[0] + (double)a.weights[1] + (double)a.weights[2];
  const double total = (term[0] * a.weights[0] + term[1] * a.weights[1] + term[2] * a.weights[2]) / wsum +
                       term[3] * a.weights[3];
  losses[0] = (float)total;
  for (int t = 0; t < 4; ++t) losses[1 + t] = (float)term[t];
}

struct Bars {
  const float* p[5];
};

__device__ __forceinline__ float bar(const Bars& b, int i) { return b.p[i] ? *b.p[i] : 0.0f; }

__global__ void backward_kernel(nudf_color_loss_args a, Bars bars, const uint8_t* __restrict__ kept,
                                const float* __restrict__ ws, float* __restrict__ d_base, float* __restrict__ d_color,
                                float* __restrict__ d_pixel, float* __restrict__ d_patch) {
  const int64_t ray = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int N = a.n_rays;
  if (ray >= N) return;
  const double* st = reinterpret_cast<const double*>(ws + (int64_t)4 * N);
  const double g_loss = (double)bar(bars, 0);
  const double wsum = (double)a.weights[0] + (double)a.weights[1] + (double)a.weights[2];
  if (lane < 3) {
    const float* p = lane == 0 ? a.color_base : (lane == 1 ? a.color : a.color_pixel);
    float* out = lane == 0 ? d_base : (lane == 1 ? d_color : d_pixel);
    if (p && out) {
      // d term / d pred = sign(pred - gt) / den (the mask enters the denominator only)
      const float coef = (float)(((double)bar(bars, 1 + lane) + g_loss * a.weights[lane] / wsum) / st[lane]);
      for (int c = 0; c < 3; ++c) {
        const float d = p[3 * ray + c] - a.gt_color[3 * ray + c];
        const float s = d > 0.0f ? 1.0f : (d < 0.0f ? -1.0f : (d == 0.0f ? 0.0f : d));   // torch.sign: sign(0) = 0
        out[3 * ray + c] = s * coef;
      }
    }
  }
  if (!a.patch_colors || !d_patch) return;
  const int side = 2 * a.h_patch + 1, npx = side * side;
  const float* x = a.patch_colors + ray * npx * 3;
  const float* y = a.gt_patch_colors + ray * npx * 3;
  const float* w = a.window;
  float* dx = d_patch + ray * npx * 3;
  if (!kept[ray]) {                                   // excluded and unmasked rays get no gradient
    for (int q = lane; q < npx * 3; q += 32) dx[q] = 0.0f;
    return;
  }
  // d loss / d error of a kept ray = (upstream of color_patch_loss) / n_kept
  const double g = ((double)bar(bars, 4) + g_loss * a.weights[3]) / st[3];
  const int type = a.patch_type;
  if (type == NUDF_PATCH_L1 || type == NUDF_PATCH_SSD) {
    for (int p = lane; p < npx; p += 32)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double d = (double)x[3 * p + c] - (double)y[3 * p + c];
        const double s = type == NUDF_PATCH_L1 ? (d > 0.0 ? 1.0 : (d < 0.0 ? -1.0 : (d == 0.0 ? 0.0 : d))) : 2.0 * d;
        dx[3 * p + c] = (float)(s * g / 3.0);
      }
    return;
  }
  Moments m;
  moments(x, y, w, npx, lane, m);
  // per channel: d error / d x_p = w_p (k_mu + 2 x_p k_xx + y_p k_xy)  (ssim), or
  //              w_p (k_x (x_p - mu1) + k_y (y_p - mu2) + k_0)       (ncc)
  double k0[3], k1[3], k2[3];
  if (type == NUDF_PATCH_SSIM) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double mu1 = m.mu1[c], mu2 = m.mu2[c];
      const double m12 = mu1 * mu2, m11 = mu1 * mu1, m22 = mu2 * mu2;
      const double A = 2.0 * m12 + C1, B = 2.0 * (m.xy[c] - m12) + C2;
      const double C = m11 + m22 + C1, D = (m.xx[c] - m11) + (m.yy[c] - m22) + C2;
      const double CD = C * D, S = A * B / CD;
      const double sA = B / CD, sB = A / CD, sC = -S / C, sD = -S / D;
      const double h = -0.5 * g;                      // error = sum_c (1 - S_c) / 2
      k0[c] = h * (2.0 * mu2 * (sA - sB) + 2.0 * mu1 * (sC - sD));
      k1[c] = h * sD;                                 // d D / d xx = 1
      k2[c] = h * 2.0 * sB;                           // d B / d xy = 2
    }
    for (int p = lane; p < npx; p += 32) {
      const double wp = (double)w[p];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const double xv = (double)x[3 * p + c], yv = (double)y[3 * p + c];
        dx[3 * p + c] = (float)(wp * (k0[c] + 2.0 * xv * k1[c] + yv * k2[c]));
      }
    }
    return;
  }
  double T[3], U[3];
  ncc_sums(x, y, w, npx, lane, m, T, U);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    // ncc = a b T, a = 1 / (sigma1 + 1e-8), sigma1 = sqrt(xx - mu1^2 + 1e-4), T = sum w (x - mu1)(y - mu2):
    // d ncc / d x_p = b w_p (-T a^2 (x_p - mu1) / sigma1 + a ((y_p - mu2) - U)); error = 1 - sum_c ncc_c / 3
    const double s1 = ncc_sigma(m.xx[c], m.mu1[c]), s2 = ncc_sigma(m.yy[c], m.mu2[c]);
    const double ia = 1.0 / (s1 + 1e-8), ib = 1.0 / (s2 + 1e-8);
    const double h = -g / 3.0;
    k0[c] = h * ib * ia;                              // times ((y_p - mu2) - U)
    k1[c] = -h * ib * T[c] * ia * ia / s1;            // times (x_p - mu1)
    k2[c] = U[c];
  }
  for (int p = lane; p < npx; p += 32) {
    const double wp = (double)w[p];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double xv = (double)x[3 * p + c], yv = (double)y[3 * p + c];
      dx[3 * p + c] = (float)(wp * (k1[c] * (xv - m.mu1[c]) + k0[c] * ((yv - m.mu2[c]) - k2[c])));
    }
  }
}

static int check_args(const nudf_color_loss_args* a) {
  NUDF_REQUIRE(a != nullptr, "null args");
  NUDF_REQUIRE(a->n_rays >= 1 && a->n_rays <= kMaxRays, "n_rays must be in 1..16384");
  NUDF_REQUIRE(a->gt_color != nullptr || !(a->color_base || a->color || a->color_pixel), "pixel terms need gt_color");
  if (a->patch_colors) {
    NUDF_REQUIRE(a->gt_patch_colors && a->patch_mask, "the patch term needs gt_patch_colors and patch_mask");
    NUDF_REQUIRE(a->patch_type >= NUDF_PATCH_L1 && a->patch_type <= NUDF_PATCH_NCC, "unknown patch_type");
    NUDF_REQUIRE(a->h_patch >= 1 && a->h_patch <= 15, "h_patch must be in 1..15");
    NUDF_REQUIRE(a->window != nullptr || a->patch_type == NUDF_PATCH_L1 || a->patch_type == NUDF_PATCH_SSD,
                 "ssim / ncc need the window");
  }
  return 0;
}

// the forward keeps four doubles at ws + 4 N
static inline bool ws_aligned(const float* ws) { return (reinterpret_cast<uintptr_t>(ws) & 7u) == 0; }

static inline unsigned warp_blocks(int n) { return (unsigned)cdiv((int64_t)n * 32, 256); }

}  // namespace cl
}  // namespace nudf

using namespace nudf;
using namespace nudf::cl;

extern "C" {

int nudf_color_loss_forward(const nudf_color_loss_args* args, float* losses, uint8_t* kept, float* ws, void* stream) {
  if (int rc = check_args(args)) return rc;
  NUDF_REQUIRE(losses && ws && (kept || !args->patch_colors), "null pointer");
  NUDF_REQUIRE(ws_aligned(ws), "ws must be 8-byte aligned");
  const size_t smem = args->patch_colors ? (size_t)args->n_rays * 4 : 0;
  // the opt-in above 48 KB is a per-device attribute of the kernel: set it on the current device whenever it is needed
  if (smem > 48 * 1024)
    NUDF_CUDA_OK(cudaFuncSetAttribute(reject_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  LaunchTimer lt_(FAM_RAY, (cudaStream_t)stream);
  ray_kernel<<<warp_blocks(args->n_rays), 256, 0, (cudaStream_t)stream>>>(*args, ws);
  NUDF_LAUNCH_OK();
  reject_kernel<<<1, kRejectThreads, smem, (cudaStream_t)stream>>>(*args, losses, kept, ws);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_color_loss_backward(const nudf_color_loss_args* args, const float* const* losses_bar, const uint8_t* kept,
                             const float* ws, float* d_color_base, float* d_color, float* d_color_pixel, float* d_patch_colors,
                             void* stream) {
  if (int rc = check_args(args)) return rc;
  NUDF_REQUIRE(losses_bar && ws && (kept || !args->patch_colors), "null pointer");
  NUDF_REQUIRE(ws_aligned(ws), "ws must be 8-byte aligned");
  Bars b;
  for (int i = 0; i < 5; ++i) b.p[i] = losses_bar[i];
  LaunchTimer lt_(FAM_RAY, (cudaStream_t)stream);
  backward_kernel<<<warp_blocks(args->n_rays), 256, 0, (cudaStream_t)stream>>>(*args, b, kept, ws, d_color_base, d_color,
                                                                               d_color_pixel, d_patch_colors);
  NUDF_LAUNCH_OK();
  return 0;
}

}  // extern "C"

// Hierarchical importance sampling on the device: one warp per ray, no host synchronisation.
// Reference: models/udf_renderer_blending.py:66-104 (sample_pdf), :197-272 (up_sample_unbias),
// :834-866 (up_sample_no_occ_aware), :274-290 (cat_z_vals).
// The three scans that decide the searchsorted indices (vis_prob cumprod, transmittance cumprod, cdf cumsum) are
// accumulated in fp64 and rounded to fp32 per element -- the arithmetic of torch's CPU cumsum/cumprod on float32
// (SURVEY.md 8(c)) -- so the integer indices reproduce the reference's given identical (z, udf) inputs.
#include "../../include/nudf.h"
#include "common.cuh"
#include "raymath.cuh"

namespace nudf {

constexpr int SP_WARPS = 4;
constexpr unsigned FULLM = 0xffffffffu;

__device__ __forceinline__ double warp_scan_mul_d(double v, int lane) {
  for (int o = 1; o < 32; o <<= 1) {
    double t = __shfl_up_sync(FULLM, v, o);
    if (lane >= o) v *= t;
  }
  return v;
}
__device__ __forceinline__ double warp_scan_add_d(double v, int lane) {
  for (int o = 1; o < 32; o <<= 1) {
    double t = __shfl_up_sync(FULLM, v, o);
    if (lane >= o) v += t;
  }
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULLM, v, o);
  return v;
}

// out[i] = float( prod_{j<i} in[j] ), i < n  (exclusive; fp64 running product, each element rounded to fp32)
__device__ __forceinline__ void excl_cumprod_f64(const float* in, float* out, int n, int lane) {
  double carry = 1.0;
  for (int i0 = 0; i0 < n; i0 += 32) {
    int i = i0 + lane;
    double v = (i < n) ? (double)in[i] : 1.0;
    double inc = warp_scan_mul_d(v, lane);
    double exc = __shfl_up_sync(FULLM, inc, 1);
    if (lane == 0) exc = 1.0;
    if (i < n) out[i] = (float)(carry * exc);
    carry *= __shfl_sync(FULLM, inc, 31);
  }
  __syncwarp();
}

// Inverse-CDF sampling with deterministic u (sample_pdf, det=True).  bins[n], w[n-1] (raw weights, +1e-5 added here),
// cdf: scratch [n].  Writes samples[m] and optionally inds[m].
__device__ __forceinline__ void sample_pdf_warp(const float* bins, const float* w, float* cdf, int n, const float* u, int m,
                                                float* samples, int64_t* inds, int lane, int32_t* status = nullptr) {
  const int nw = n - 1;
  double s = 0.0;
  for (int j = lane; j < nw; j += 32) s += (double)(w[j] + 1e-5f);
  const float total = (float)warp_sum_d(s);
  // cdf[0] = 0, cdf[j+1] = float(sum_{k<=j} pdf_k) with an fp64 accumulator
  double carry = 0.0;
  if (lane == 0) cdf[0] = 0.0f;
  for (int j0 = 0; j0 < nw; j0 += 32) {
    int j = j0 + lane;
    float pdf = (j < nw) ? (w[j] + 1e-5f) / total : 0.0f;
    double inc = warp_scan_add_d((double)pdf, lane);
    if (j < nw) cdf[j + 1] = (float)(carry + inc);
    carry += __shfl_sync(FULLM, inc, 31);
  }
  __syncwarp();
  for (int k = lane; k < m; k += 32) {
    float uk = u[k];
    // searchsorted(cdf, u, right=True): number of entries <= u
    int lo = 0, hi = n;
    while (lo < hi) {
      int mid = (lo + hi) >> 1;
      if (cdf[mid] <= uk) lo = mid + 1; else hi = mid;
    }
    int below = lo - 1 > 0 ? lo - 1 : 0;
    int above = lo < n - 1 ? lo : n - 1;
    float c0 = cdf[below], c1 = cdf[above];
    float denom = c1 - c0;
    if (denom < 1e-5f) denom = 1.0f;
    float t = (uk - c0) / denom;
    float b0 = bins[below], b1 = bins[above];
    const float smp = __fadd_rn(b0, __fmul_rn(t, __fsub_rn(b1, b0)));
    samples[k] = smp;
    if (inds) inds[k] = lo;
    // the reference traps non-finite samples with pdb (udf_renderer_blending.py:97-101, 265-269): raise the device flag
    if (status != nullptr && !isfinite(smp)) atomicOr(status, NUDF_STATUS_NONFINITE_SAMPLES);
  }
}

// mode 0: up_sample_unbias ; mode 1: up_sample_no_occ_aware.  RULE is the alpha rule (AlphaRule, raymath.cuh) of the
// unbias branch's sdf2alpha calls (:256-257); the no-occ-aware branch has none.
template <int RULE>
__global__ void __launch_bounds__(SP_WARPS * 32)
up_sample_kernel(int mode, const float* __restrict__ rays_o, const float* __restrict__ rays_d, const float* __restrict__ z,
                 const float* __restrict__ udf, int n_rays, int n, int m, float sample_dist, float inv_s, float beta,
                 float gamma, const float* __restrict__ u_lin, float* __restrict__ new_z, int64_t* __restrict__ inds,
                 int32_t* __restrict__ status) {
  extern __shared__ float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * SP_WARPS + warp;
  if (r >= n_rays) return;
  float* base = smem + (size_t)warp * 8 * n;
  float* sz = base;            // z
  float* su = base + n;        // udf
  float* tcs = base + 2 * n;   // true_cos per section (n-1)
  float* fac = base + 3 * n;   // scan input
  float* vis = base + 4 * n;   // vis_prob
  float* alp = base + 5 * n;   // alpha per section
  float* wts = base + 6 * n;   // weights per section
  float* cdf = base + 7 * n;
  const float o[3] = {rays_o[r * 3 + 0], rays_o[r * 3 + 1], rays_o[r * 3 + 2]};
  const float d[3] = {rays_d[r * 3 + 0], rays_d[r * 3 + 1], rays_d[r * 3 + 2]};
  for (int i = lane; i < n; i += 32) { sz[i] = z[(int64_t)r * n + i]; su[i] = udf[(int64_t)r * n + i]; }
  __syncwarp();
  if (mode == 1) {
    // weights = alpha_occ[:, :-1] with raw = logistic(udf, beta) * gamma, alpha = 1 - exp(-relu(raw) * dists)
    for (int j = lane; j < n - 1; j += 32) {
      float dist = __fsub_rn(sz[j + 1], sz[j]);
      float e = expf(-beta * su[j]);
      float raw = 1.0f * beta * e / ((1.0f + e) * (1.0f + e)) * gamma;
      wts[j] = 1.0f - expf(-fmaxf(raw, 0.0f) * dist);
    }
    __syncwarp();
  } else {
    for (int j = lane; j < n - 1; j += 32) tcs[j] = __fsub_rn(su[j + 1], su[j]) / __fadd_rn(__fsub_rn(sz[j + 1], sz[j]), 1e-5f);
    __syncwarp();
    // visibility factors over all n samples
    for (int i = lane; i < n; i += 32) {
      float dist_raw = (i + 1 < n) ? __fsub_rn(sz[i + 1], sz[i]) : sample_dist;
      float raw, aocc;
      occ_forward(su[i], dist_raw, beta, gamma, &raw, &aocc);
      float vm = (i == 0) ? 1.0f : (tcs[i - 1] < 0.05f ? 1.0f : 0.0f);
      fac[i] = clampf_(1.0f - aocc + vm, 0.0f, 1.0f) + 1e-7f;
    }
    __syncwarp();
    excl_cumprod_f64(fac, vis, n, lane);
    for (int j = lane; j < n - 1; j += 32) {
      float p0[3], p1[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        p0[c] = __fadd_rn(o[c], __fmul_rn(d[c], sz[j]));
        p1[c] = __fadd_rn(o[c], __fmul_rn(d[c], sz[j + 1]));
      }
      float r0 = sqrtf(p0[0] * p0[0] + p0[1] * p0[1] + p0[2] * p0[2]);
      float r1 = sqrtf(p1[0] * p1[0] + p1[1] * p1[1] + p1[2] * p1[2]);
      float inside = (r0 < 1.0f || r1 < 1.0f) ? 1.0f : 0.0f;
      float cosj = -fabsf(tcs[j]);
      float prevc = (j > 0) ? -fabsf(tcs[j - 1]) : 0.0f;
      float cv = clampf_(fminf(prevc, cosj), -1e3f, 0.0f) * inside;
      float mid_udf = __fmul_rn(__fadd_rn(su[j], su[j + 1]), 0.5f);
      float dist = __fsub_rn(sz[j + 1], sz[j]);
      float ap = alpha_forward<RULE>(mid_udf, cv, dist, inv_s);
      float am = alpha_forward<RULE>(-mid_udf, cv, dist, inv_s);
      float sg = vis[j];
      float a = ap * sg + am * (1.0f - sg);
      alp[j] = a;
      fac[j] = 1.0f - a + 1e-7f;
    }
    __syncwarp();
    excl_cumprod_f64(fac, wts, n - 1, lane);
    for (int j = lane; j < n - 1; j += 32) wts[j] = alp[j] * wts[j];
    __syncwarp();
  }
  sample_pdf_warp(sz, wts, cdf, n, u_lin, m, new_z + (int64_t)r * m, inds ? inds + (int64_t)r * m : nullptr, lane, status);
}

__global__ void __launch_bounds__(SP_WARPS * 32)
sample_pdf_kernel(const float* __restrict__ bins, const float* __restrict__ weights, int n_rays, int n, int m,
                  const float* __restrict__ u_lin, float* __restrict__ samples, int64_t* __restrict__ inds,
                  int32_t* __restrict__ status) {
  extern __shared__ float smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r = blockIdx.x * SP_WARPS + warp;
  if (r >= n_rays) return;
  float* base = smem + (size_t)warp * 3 * n;
  float* sb = base; float* sw = base + n; float* cdf = base + 2 * n;
  for (int i = lane; i < n; i += 32) sb[i] = bins[(int64_t)r * n + i];
  for (int i = lane; i < n - 1; i += 32) sw[i] = weights[(int64_t)r * (n - 1) + i];
  __syncwarp();
  sample_pdf_warp(sb, sw, cdf, n, u_lin, m, samples + (int64_t)r * m, inds ? inds + (int64_t)r * m : nullptr, lane, status);
}

// Sorted merge of z[n] (sorted) and new_z[m] (sorted): rank by binary search; udf gathered alongside.
__global__ void merge_z_kernel(const float* __restrict__ z, const float* __restrict__ new_z, const float* __restrict__ udf,
                               const float* __restrict__ new_udf, int n_rays, int n, int m, float* __restrict__ z_out,
                               float* __restrict__ udf_out) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int tot = n + m;
  if (idx >= (int64_t)n_rays * tot) return;
  int r = (int)(idx / tot), e = (int)(idx - (int64_t)r * tot);
  const float* zr = z + (int64_t)r * n;
  const float* nr = new_z + (int64_t)r * m;
  float v; int pos; float uv = 0.f;
  if (e < n) {
    v = zr[e];
    int lo = 0, hi = m;                      // count of new values strictly less than v
    while (lo < hi) { int mid = (lo + hi) >> 1; if (nr[mid] < v) lo = mid + 1; else hi = mid; }
    pos = e + lo;
    if (udf) uv = udf[(int64_t)r * n + e];
  } else {
    int k = e - n;
    v = nr[k];
    int lo = 0, hi = n;                      // count of old values less than or equal to v
    while (lo < hi) { int mid = (lo + hi) >> 1; if (zr[mid] <= v) lo = mid + 1; else hi = mid; }
    pos = k + lo;
    if (new_udf) uv = new_udf[(int64_t)r * m + k];
  }
  z_out[(int64_t)r * tot + pos] = v;
  if (udf_out) udf_out[(int64_t)r * tot + pos] = uv;
}

}  // namespace nudf

using namespace nudf;

extern "C" {

int nudf_up_sample(int32_t mode, const float* rays_o, const float* rays_d, const float* z, const float* udf, int32_t n_rays,
                   int32_t n, int32_t m, float sample_dist, float inv_s, float beta, float gamma, const float* u_lin,
                   float* new_z, int64_t* inds, int32_t* status, void* stream) {
  NUDF_REQUIRE(mode == 0 || mode == 1 || mode == 2, "mode must be 0, 1 or 2");
  NUDF_REQUIRE(rays_o && rays_d && z && udf && new_z && u_lin, "null pointer");
  NUDF_REQUIRE(n >= 2 && m >= 1, "need n >= 2, m >= 1");
  if (n_rays <= 0) return 0;
  size_t smem = (size_t)SP_WARPS * 8 * n * sizeof(float);
  NUDF_REQUIRE(smem <= 200 * 1024, "too many samples per ray");
  // mode 2 is mode 0's up_sample_unbias under the 'theorical' alpha
  const bool theorical = mode == 2;
  auto kernel = theorical ? up_sample_kernel<ALPHA_THEORICAL> : up_sample_kernel<ALPHA_NUMERICAL>;
  if (smem > 48 * 1024)
    NUDF_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<(unsigned)cdiv(n_rays, SP_WARPS), SP_WARPS * 32, smem, (cudaStream_t)stream>>>(
      theorical ? 0 : mode, rays_o, rays_d, z, udf, n_rays, n, m, sample_dist, inv_s, beta, gamma, u_lin, new_z, inds, status);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_sample_pdf(const float* bins, const float* weights, int32_t n_rays, int32_t n, int32_t m, const float* u_lin,
                    float* samples, int64_t* inds, int32_t* status, void* stream) {
  NUDF_REQUIRE(bins && weights && samples && u_lin, "null pointer");
  NUDF_REQUIRE(n >= 2 && m >= 1, "need n >= 2, m >= 1");
  if (n_rays <= 0) return 0;
  size_t smem = (size_t)SP_WARPS * 3 * n * sizeof(float);
  NUDF_REQUIRE(smem <= 200 * 1024, "too many bins per ray");
  if (smem > 48 * 1024)
    NUDF_CUDA_OK(cudaFuncSetAttribute(sample_pdf_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  sample_pdf_kernel<<<(unsigned)cdiv(n_rays, SP_WARPS), SP_WARPS * 32, smem, (cudaStream_t)stream>>>(
      bins, weights, n_rays, n, m, u_lin, samples, inds, status);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_merge_z(const float* z, const float* new_z, const float* udf, const float* new_udf, int32_t n_rays, int32_t n,
                 int32_t m, float* z_out, float* udf_out, void* stream) {
  NUDF_REQUIRE(z && new_z && z_out, "null pointer");
  NUDF_REQUIRE(udf_out == nullptr || (udf && new_udf), "udf_out needs udf and new_udf");
  if (n_rays <= 0) return 0;
  int64_t tot = (int64_t)n_rays * (n + m);
  merge_z_kernel<<<(unsigned)cdiv(tot, 256), 256, 0, (cudaStream_t)stream>>>(z, new_z, udf, new_udf, n_rays, n, m, z_out, udf_out);
  NUDF_LAUNCH_OK();
  return 0;
}

}  // extern "C"

// Shared helpers for the nudf sm_90a kernels.
// Math helpers marked NUDF_HD are compiled for the host as well (tests/host/ builds them with g++ to check
// the per-sample formulas against the oracle on the CPU dev box, where no GPU exists).
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define NUDF_HD __host__ __device__ __forceinline__
#else
#define NUDF_HD inline
#endif

#define NUDF_MAX_LAYERS 16
#define NUDF_SQRT1_2 0.70710678118654752440f

namespace nudf {

// nn.Softplus(beta=100, threshold=20)  (reference models/fields.py:180):  z if 100 z > 20 else log1p(exp(100 z))/100.
// Device code uses the overflow-free form max(z,0) + log(1 + e^{-|100 z|})/100 with the MUFU-based __expf/__logf: the
// argument of the log is in [1,2], where __logf's absolute error is <= 2^-21.4, i.e. <= 4e-9 after the /100 -- an order
// of magnitude below fp32 resolution of the O(0.1..1) activations -- at ~1/5 of the instruction count of log1pf(expf()).
NUDF_HD float softplus100(float z) {
  float bz = 100.0f * z;
#if defined(__CUDA_ARCH__)
  float t = __expf(-fabsf(bz));
  float sp = fmaxf(z, 0.0f) + 0.01f * __logf(1.0f + t);
  return bz > 20.0f ? z : sp;
#else
  return bz > 20.0f ? z : log1pf(expf(bz)) * 0.01f;
#endif
}
// sigma(100 z) recovered from a = softplus100(z); exactly 1 in the linear regime (torch's softplus backward).
NUDF_HD float sig_from_softplus(float a) {
  float ba = 100.0f * a;
#if defined(__CUDA_ARCH__)
  return ba > 20.0f ? 1.0f : 1.0f - __expf(-ba);
#else
  return ba > 20.0f ? 1.0f : -expm1f(-ba);
#endif
}
NUDF_HD float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

NUDF_HD float clampf_(float x, float lo, float hi) { return fminf(fmaxf(x, lo), hi); }

}  // namespace nudf

#if defined(__CUDACC__)
#include <cuda_runtime.h>
#include <stdio.h>

#include <algorithm>

namespace nudf {

void set_error(const char* fmt, ...);
void count_launch();

// Per-kernel-family device timing for bench.py (nudf_set_launch_timing): while enabled, every launch wrapped in a
// LaunchTimer is bracketed by a cudaEvent pair recorded on the launching stream; nudf_read_launch_timing() synchronises
// and sums the pairs per family.  Off by default (zero overhead besides one branch).
enum LaunchFamily {
  FAM_UDF_FWD_CHAIN = 0,   // fused UDF value chain: no kernel of this build (the family order is part of the ABI)
  FAM_TC_REV = 1,          // one layer of the reverse sweep (grad_x udf) on the tensor cores
  FAM_TC_TAN = 2,          // one layer of the tangent chain
  FAM_TC_BWD = 3,          // one layer of the backward chain
  FAM_TC_OTHER = 4,        // other tensor-core layer GEMMs (colour / NeRF++ layers, UDF value chain)
  FAM_TC_WGRAD = 5,        // weight-gradient contractions on the tensor cores
  FAM_FFMA = 6,            // exact-fp32 FFMA GEMMs
  FAM_RAY = 7,             // ray kernels: compositing forward / backward, sampling, blending
  FAM_ELEMENTWISE = 8,     // element-wise kernels of the library (PE, fold / unfold, seeds, column sums)
  FAM_UDF_BWD_CHAIN = 9,   // fused tangent + backward chains: no kernel of this build
  FAM_COUNT = 10
};
bool launch_timing_on();
int launch_timer_begin(int family, cudaStream_t st);
void launch_timer_end(int slot, cudaStream_t st);
struct LaunchTimer {
  int slot; cudaStream_t st;
  LaunchTimer(int family, cudaStream_t s) : slot(-1), st(s) { if (launch_timing_on()) slot = launch_timer_begin(family, s); }
  ~LaunchTimer() { if (slot >= 0) launch_timer_end(slot, st); }
};

#define NUDF_CUDA_OK(expr)                                                              \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      nudf::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return -2;                                                                        \
    }                                                                                   \
  } while (0)

#define NUDF_LAUNCH_OK()                                                                \
  do {                                                                                  \
    nudf::count_launch();                                                               \
    cudaError_t _e = cudaGetLastError();                                                \
    if (_e != cudaSuccess) {                                                            \
      nudf::set_error("%s:%d: kernel launch -> %s", __FILE__, __LINE__, cudaGetErrorString(_e)); \
      return -2;                                                                        \
    }                                                                                   \
  } while (0)

#define NUDF_REQUIRE(cond, msg)                                                         \
  do {                                                                                  \
    if (!(cond)) {                                                                      \
      nudf::set_error("%s:%d: requirement failed: %s (%s)", __FILE__, __LINE__, #cond, msg); \
      return -1;                                                                        \
    }                                                                                   \
  } while (0)

// workspace of the deterministic split-K reductions (gemm_simt.cuh): ONE per device, so all library work on a device must be
// ordered on one stream (as torch's autograd runs it); allocated on first use, which must lie outside a CUDA-graph capture
constexpr int64_t SPLIT_WS_FLOATS = 8ll << 20;   // 32 MB
float* split_workspace(cudaStream_t st);

static inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int64_t round_up(int64_t a, int64_t b) { return cdiv(a, b) * b; }
// the grid of a grid-stride launch over n items, per_block items a block: at least 1 block, at most 8 * 65535
static inline unsigned grid_for(int64_t n, int per_block = 256) {
  return (unsigned)std::min<int64_t>(std::max<int64_t>(cdiv(n, per_block), 1), 65535ll * 8);
}
// the ctx / scratch layouts of the networks: offsets in floats, every block starts 16-byte aligned
struct Bump {
  int64_t off = 0;
  int64_t take(int64_t n) { int64_t o = off; off += round_up(n, 4); return o; }
};

__host__ __device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---- weight-norm fold / unfold of ALL layers of a network in one launch ------------------------------------------------------
// W = g v / ||v||  (row-wise; torch._weight_norm(v, g, dim=0), reference models/fields.py:110-113) and its adjoint
// dg = <dW, v>/||v||, dv = g/||v|| (dW - dg v/||v||).  A job = one layer; grid = (max rows over the jobs, number of jobs).
constexpr int NUDF_MAX_JOBS = 32;
struct FoldJob {
  const float* g; const float* v;      // [out], [out, in]
  const float* dw; float* dg; float* dv;   // unfold only
  float* w;                            // fold only: [out, ld], columns >= in zero-filled
  int out, in, ld;
};
struct FoldJobs { int n; FoldJob j[NUDF_MAX_JOBS]; };

static __global__ void fold_jobs_kernel(const __grid_constant__ FoldJobs jobs) {
  const FoldJob& J = jobs.j[blockIdx.y];
  const int row = blockIdx.x;
  if (row >= J.out) return;
  const float* vr = J.v + (int64_t)row * J.in;
  float ss = 0.f;
  for (int k = threadIdx.x; k < J.in; k += blockDim.x) ss += vr[k] * vr[k];
  __shared__ float red[32];
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (threadIdx.x == 0) red[0] = t;
  }
  __syncthreads();
  const float s = J.g[row] / sqrtf(red[0]);
  for (int k = threadIdx.x; k < J.ld; k += blockDim.x) J.w[(int64_t)row * J.ld + k] = k < J.in ? vr[k] * s : 0.f;
}
static __global__ void unfold_jobs_kernel(const __grid_constant__ FoldJobs jobs) {
  const FoldJob& J = jobs.j[blockIdx.y];
  const int row = blockIdx.x;
  if (row >= J.out) return;
  const float* vr = J.v + (int64_t)row * J.in;
  const float* dr = J.dw + (int64_t)row * J.ld;
  float ss = 0.f, dot = 0.f;
  for (int k = threadIdx.x; k < J.in; k += blockDim.x) { ss += vr[k] * vr[k]; dot += vr[k] * dr[k]; }
  __shared__ float red[2][32];
  for (int o = 16; o > 0; o >>= 1) { ss += __shfl_xor_sync(0xffffffffu, ss, o); dot += __shfl_xor_sync(0xffffffffu, dot, o); }
  if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = ss; red[1][threadIdx.x >> 5] = dot; }
  __syncthreads();
  if (threadIdx.x < 32) {
    float t0 = threadIdx.x < (blockDim.x >> 5) ? red[0][threadIdx.x] : 0.f;
    float t1 = threadIdx.x < (blockDim.x >> 5) ? red[1][threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) { t0 += __shfl_xor_sync(0xffffffffu, t0, o); t1 += __shfl_xor_sync(0xffffffffu, t1, o); }
    if (threadIdx.x == 0) { red[0][0] = t0; red[1][0] = t1; }
  }
  __syncthreads();
  const float n = sqrtf(red[0][0]);
  const float dgv = red[1][0] / n;
  if (threadIdx.x == 0) J.dg[row] = dgv;
  const float gn = J.g[row] / n;
  for (int k = threadIdx.x; k < J.in; k += blockDim.x) J.dv[(int64_t)row * J.in + k] = gn * (dr[k] - dgv * vr[k] / n);
}
// host: launch all jobs at once
static inline int run_fold_jobs(const FoldJobs& jobs, bool unfold, cudaStream_t st) {
  if (jobs.n <= 0) return 0;
  int max_out = 0;
  for (int i = 0; i < jobs.n; ++i) max_out = jobs.j[i].out > max_out ? jobs.j[i].out : max_out;
  const dim3 grid((unsigned)max_out, (unsigned)jobs.n);
  if (unfold) unfold_jobs_kernel<<<grid, 128, 0, st>>>(jobs);
  else fold_jobs_kernel<<<grid, 128, 0, st>>>(jobs);
  NUDF_LAUNCH_OK();
  return 0;
}

}  // namespace nudf
#endif

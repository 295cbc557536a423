// Surface point clouds of a UDF (neuraludf_b200/cloud.py drives them; DESIGN.md section 1 states the algorithm): the
// projection step p <- p - (u / |g|) g with its stable compaction, the final udf filter with the same compaction, and the
// seeded jittered resampling of the kept points.  Every fp32 operation is rounded once in the stated order with no
// contraction (__f*_rn), so that tests/proto/udf_cloud.py reproduces the kernels bit for bit from the same (u, g).  The
// step and the filter are compact.cuh's stable compaction: a point is an item with at most one output.
#include "../../include/nudf.h"
#include "common.cuh"
#include "compact.cuh"

namespace nudf {
namespace uc {

__device__ __forceinline__ bool in_box(const float q[3]) {
  // written so that a NaN coordinate is outside
  return q[0] >= -1.f && q[0] <= 1.f && q[1] >= -1.f && q[1] <= 1.f && q[2] >= -1.f && q[2] <= 1.f;
}

// the output of the compactions: the survivor q at out[3 j .. 3 j + 2], out a restrict pointer so that the inputs are
// read through the read-only path
using Out = float* __restrict__;
__device__ __forceinline__ void store_point(Out out, int64_t j, const float q[3]) {
  out[3 * j] = q[0];
  out[3 * j + 1] = q[1];
  out[3 * j + 2] = q[2];
}

// step 2: n = sqrt((gx gx + gy gy) + gz gz), q = p - (u / n) g; a point survives when u and g are finite, n != 0 and q
// lies in [-1,1]^3
struct StepOp {
  using Item = float[3];
  const float* p;
  const float* u;
  const float* g;
  __device__ __forceinline__ int eval(int64_t t, Item& q, bool) const {
    const float ut = u[t], gx = g[3 * t], gy = g[3 * t + 1], gz = g[3 * t + 2];
    const float n = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(gz, gz)));
    const float s = __fdiv_rn(ut, n);
    q[0] = __fsub_rn(p[3 * t], __fmul_rn(s, gx));
    q[1] = __fsub_rn(p[3 * t + 1], __fmul_rn(s, gy));
    q[2] = __fsub_rn(p[3 * t + 2], __fmul_rn(s, gz));
    return isfinite(ut) && isfinite(gx) && isfinite(gy) && isfinite(gz) && n != 0.f && in_box(q);
  }
  __device__ __forceinline__ void store(Out out, int64_t j, int64_t, const Item& q) const { store_point(out, j, q); }
};

// step 3: a point survives when u < thr (NaN does not)
struct FilterOp {
  using Item = float[3];
  const float* p;
  const float* u;
  float thr;
  __device__ __forceinline__ int eval(int64_t t, Item& q, bool) const {
    q[0] = p[3 * t];
    q[1] = p[3 * t + 1];
    q[2] = p[3 * t + 2];
    return u[t] < thr;
  }
  __device__ __forceinline__ void store(Out out, int64_t j, int64_t, const Item& q) const { store_point(out, j, q); }
};

// lowbias32, a public-domain bijective 32-bit integer mixer (C. Wellons); all arithmetic mod 2^32
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}

// the counter-based hash of the densify rounds: stream (seed, round, k), counter i
__device__ __forceinline__ uint32_t cloud_hash(uint32_t seed, uint32_t round, uint32_t i, uint32_t k) {
  return mix32(mix32(seed + 0x9e3779b9u * (4u * round + k)) ^ i);
}

// step 4: new point i = pool[cloud_hash(seed, round, i, 0) mod n_pool] + ((b_a 2^-24 - 1/2) voxel)_a, b_a the top 24 bits of
// cloud_hash(seed, round, i, 1 + a): t = b_a 2^-24 and t - 1/2 are exact in fp32, the product and the sum are rounded once
__global__ void k_resample(const float* __restrict__ pool, uint32_t n_pool, int64_t m, uint32_t seed, uint32_t round,
                           float voxel, float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    const uint32_t c = cloud_hash(seed, round, (uint32_t)i, 0) % n_pool;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float t = __fmul_rn(__uint2float_rn(cloud_hash(seed, round, (uint32_t)i, 1 + a) >> 8), 0x1p-24f);
      out[3 * i + a] = __fadd_rn(pool[3 * (int64_t)c + a], __fmul_rn(__fsub_rn(t, 0.5f), voxel));
    }
  }
}

}  // namespace uc
}  // namespace nudf

using namespace nudf;
using namespace nudf::uc;

int nudf_uc_step_count(const float* p, const float* u, const float* g, int64_t n, int32_t* counts, void* stream) {
  NUDF_REQUIRE(n >= 0 && (n == 0 || (p && u && g && counts)), "null pointer or negative count");
  if (n == 0) return 0;
  return seg_compact<Out>(StepOp{p, u, g}, n, counts, nullptr, nullptr, stream);
}

int nudf_uc_step_emit(const float* p, const float* u, const float* g, int64_t n, const int64_t* offsets, float* out,
                      void* stream) {
  NUDF_REQUIRE(n >= 0 && (n == 0 || (p && u && g && offsets && out)), "null pointer or negative count");
  if (n == 0) return 0;
  return seg_compact<Out>(StepOp{p, u, g}, n, nullptr, offsets, out, stream);
}

int nudf_uc_filter_count(const float* p, const float* u, int64_t n, float thr, int32_t* counts, void* stream) {
  NUDF_REQUIRE(n >= 0 && (n == 0 || (p && u && counts)), "null pointer or negative count");
  if (n == 0) return 0;
  return seg_compact<Out>(FilterOp{p, u, thr}, n, counts, nullptr, nullptr, stream);
}

int nudf_uc_filter_emit(const float* p, const float* u, int64_t n, float thr, const int64_t* offsets, float* out,
                        void* stream) {
  NUDF_REQUIRE(n >= 0 && (n == 0 || (p && u && offsets && out)), "null pointer or negative count");
  if (n == 0) return 0;
  return seg_compact<Out>(FilterOp{p, u, thr}, n, nullptr, offsets, out, stream);
}

int nudf_uc_resample(const float* pool, int64_t n_pool, int64_t m, uint32_t seed, int32_t round, float voxel, float* out,
                     void* stream) {
  NUDF_REQUIRE(m >= 0 && m <= 0xffffffffll, "m must lie in [0, 2^32)");
  NUDF_REQUIRE(round >= 0, "negative round");
  if (m == 0) return 0;
  NUDF_REQUIRE(n_pool >= 1 && n_pool <= 0xffffffffll, "the pool must hold 1 .. 2^32 - 1 points");
  NUDF_REQUIRE(pool && out, "null pointer");
  k_resample<<<grid_for(m), 256, 0, (cudaStream_t)stream>>>(pool, (uint32_t)n_pool, m, seed, (uint32_t)round, voxel, out);
  NUDF_LAUNCH_OK();
  return 0;
}

// Camera visibility, orientation and colour of surface points (neuraludf_b200/paint.py drives them; DESIGN.md section 1
// states the algorithm): unit normal lines from gradients, the ranking of candidate cameras, the sphere-traced visibility
// of (point, camera) pairs with its stable compaction, the orientation of the normals towards the chosen camera and the
// bilinear image gather.  Every fp32 operation is rounded once in the stated order with no contraction (__f*_rn), so that
// tests/proto/udf_paint.py reproduces the kernels bit for bit from the same inputs and udf values.  The round start and
// the trace step are compact.cuh's stable compaction: a point or a pair is an item with at most one output pair.
#include "../../include/nudf.h"
#include "common.cuh"
#include "compact.cuh"

namespace nudf {
namespace pt {

constexpr int kMaxViews = NUDF_PT_MAX_VIEWS;
constexpr int kMaxCand = NUDF_PT_MAX_CAND;

__device__ __forceinline__ float dot3(float ax, float ay, float az, float bx, float by, float bz) {
  return __fadd_rn(__fadd_rn(__fmul_rn(ax, bx), __fmul_rn(ay, by)), __fmul_rn(az, bz));
}

// x_r = ((P_r0 px + P_r1 py) + P_r2 pz) + P_r3 of the 3x4 row-major P
__device__ __forceinline__ void project(const float* P, float px, float py, float pz, float x[3]) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
    x[r] = __fadd_rn(dot3(P[4 * r], P[4 * r + 1], P[4 * r + 2], px, py, pz), P[4 * r + 3]);
}

// the pixel (u, w) = (x0 / x2, x1 / x2) of p in a view, true when it lies in front (x2 > 0) and inside [0,W-1] x [0,H-1]
// (a NaN coordinate is outside)
__device__ __forceinline__ bool pixel(const float* P, float px, float py, float pz, int H, int W, float& u, float& w) {
  float x[3];
  project(P, px, py, pz, x);
  u = __fdiv_rn(x[0], x[2]);
  w = __fdiv_rn(x[1], x[2]);
  return x[2] > 0.f && u >= 0.f && u <= (float)(W - 1) && w >= 0.f && w <= (float)(H - 1);
}

// d = c - p, L = sqrt((dx dx + dy dy) + dz dz), v = d / L; returns L
__device__ __forceinline__ float towards(const float* c, float px, float py, float pz, float v[3]) {
  const float dx = __fsub_rn(c[0], px), dy = __fsub_rn(c[1], py), dz = __fsub_rn(c[2], pz);
  const float L = __fsqrt_rn(dot3(dx, dy, dz, dx, dy, dz));
  v[0] = __fdiv_rn(dx, L);
  v[1] = __fdiv_rn(dy, L);
  v[2] = __fdiv_rn(dz, L);
  return L;
}

__device__ __forceinline__ void load3(const float* a, int64_t i, float& x, float& y, float& z) {
  x = a[3 * i];
  y = a[3 * i + 1];
  z = a[3 * i + 2];
}

// n = g / sqrt((gx gx + gy gy) + gz gz), 0 when that norm is 0 or not finite
__global__ void k_normals(const float* __restrict__ g, int64_t m, float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    float x, y, z;
    load3(g, i, x, y, z);
    const float L = __fsqrt_rn(dot3(x, y, z, x, y, z));
    const bool ok = isfinite(L) && L != 0.f;
    out[3 * i] = ok ? __fdiv_rn(x, L) : 0.f;
    out[3 * i + 1] = ok ? __fdiv_rn(y, L) : 0.f;
    out[3 * i + 2] = ok ? __fdiv_rn(z, L) : 0.f;
  }
}

// the cameras of a launch in shared memory: mats [V,12], centres [V,3]
struct SmemCams {
  float mats[kMaxViews * 12];
  float centres[kMaxViews * 3];
  __device__ __forceinline__ void load(const float* m, const float* c, int V) {
    for (int j = threadIdx.x; j < 12 * V; j += blockDim.x) mats[j] = m[j];
    for (int j = threadIdx.x; j < 3 * V; j += blockDim.x) centres[j] = c[j];
    __syncthreads();
  }
};

// candidates of each point: the cameras it projects in front of and inside, with |n . v| >= cos_min, the first K by
// |n . v| descending, ties to the lower index; -1 padding
__global__ void __launch_bounds__(256) k_rank(const float* __restrict__ p, const float* __restrict__ n, int64_t m,
                                              const float* __restrict__ mats, const float* __restrict__ centres, int V, int H,
                                              int W, float cos_min, int K, int32_t* __restrict__ cand) {
  __shared__ SmemCams cams;
  cams.load(mats, centres, V);
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    float px, py, pz, nx, ny, nz;
    load3(p, i, px, py, pz);
    load3(n, i, nx, ny, nz);
    float ba[kMaxCand];
    int bk[kMaxCand];
#pragma unroll
    for (int j = 0; j < kMaxCand; ++j) {
      ba[j] = -INFINITY;
      bk[j] = -1;
    }
    for (int k = 0; k < V; ++k) {
      float u, w, v[3];
      if (!pixel(cams.mats + 12 * k, px, py, pz, H, W, u, w)) continue;
      towards(cams.centres + 3 * k, px, py, pz, v);
      float a = fabsf(dot3(nx, ny, nz, v[0], v[1], v[2]));
      if (!(a >= cos_min)) continue;
      // insertion into the descending list: a goes before the first strictly smaller entry (so after equal ones, which
      // have lower indices), and every later entry moves down one slot
      int c = k;
      bool moving = false;
#pragma unroll
      for (int j = 0; j < kMaxCand; ++j) {
        if (moving || a > ba[j]) {
          const float ta = ba[j];
          const int tk = bk[j];
          ba[j] = a;
          bk[j] = c;
          a = ta;
          c = tk;
          moving = true;
        }
      }
    }
#pragma unroll
    for (int j = 0; j < kMaxCand; ++j)
      if (j < K) cand[i * K + j] = bk[j];
  }
}

struct Pair {
  int32_t idx, cam;
  float t, q[3];
};

// the output of the compactions: pair j in the four arrays
struct PairOut {
  int32_t *idx, *cam;
  float *t, *q;
  __device__ __forceinline__ void put(int64_t j, const Pair& o) const {
    idx[j] = o.idx;
    cam[j] = o.cam;
    t[j] = o.t;
    q[3 * j] = o.q[0];
    q[3 * j + 1] = o.q[1];
    q[3 * j + 2] = o.q[2];
  }
};

// round start: point i (unresolved, view[i] < 0) with candidate k = cand[i, r] >= 0 starts the pair (i, k) at
// t0 = t_start / |n . v| and q = p + t0 v
struct StartOp {
  using Item = Pair;
  const float *p, *n, *centres;
  const int32_t *cand, *view;
  int K, r;
  float t_start;
  __device__ __forceinline__ int eval(int64_t i, Pair& o, bool) const {
    if (view[i] >= 0) return 0;
    const int k = cand[i * K + r];
    if (k < 0) return 0;
    float px, py, pz, nx, ny, nz, v[3];
    load3(p, i, px, py, pz);
    load3(n, i, nx, ny, nz);
    towards(centres + 3 * k, px, py, pz, v);
    const float t = __fdiv_rn(t_start, fabsf(dot3(nx, ny, nz, v[0], v[1], v[2])));
    o = Pair{(int32_t)i, k, t, {__fadd_rn(px, __fmul_rn(t, v[0])), __fadd_rn(py, __fmul_rn(t, v[1])),
                                 __fadd_rn(pz, __fmul_rn(t, v[2]))}};
    return 1;
  }
  __device__ __forceinline__ void store(PairOut out, int64_t j, int64_t, const Pair& o) const { out.put(j, o); }
};

// trace step of pair a with the udf u[a] at its q: occluded (dropped) unless u >= hit; else t += u, q = p + t v, and the
// pair is visible (dropped; the emit pass sets view[idx] = cam) when |q|^2 > 1 or t >= |c - p|, else it stays active
struct StepOp {
  using Item = Pair;
  const float *p, *centres;
  const int32_t *idx, *cam;
  const float *t, *u;
  float hit;
  int32_t* view;
  __device__ __forceinline__ int eval(int64_t a, Pair& o, bool emit) const {
    const float ua = u[a];
    if (!(ua >= hit)) return 0;
    const int32_t i = idx[a], k = cam[a];
    float px, py, pz, v[3];
    load3(p, i, px, py, pz);
    const float L = towards(centres + 3 * k, px, py, pz, v);
    const float tn = __fadd_rn(t[a], ua);
    o = Pair{i, k, tn, {__fadd_rn(px, __fmul_rn(tn, v[0])), __fadd_rn(py, __fmul_rn(tn, v[1])),
                        __fadd_rn(pz, __fmul_rn(tn, v[2]))}};
    if (dot3(o.q[0], o.q[1], o.q[2], o.q[0], o.q[1], o.q[2]) > 1.f || tn >= L) {
      if (emit) view[i] = k;
      return 0;
    }
    return 1;
  }
  __device__ __forceinline__ void store(PairOut out, int64_t j, int64_t, const Pair& o) const { out.put(j, o); }
};

// n turned to n . v > 0 towards its view's centre (v as towards()); unchanged where view < 0
__global__ void k_orient(const float* __restrict__ p, const float* __restrict__ n, const int32_t* __restrict__ view,
                         int64_t m, const float* __restrict__ centres, float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    float px, py, pz, nx, ny, nz, v[3];
    load3(n, i, nx, ny, nz);
    const int k = view[i];
    if (k >= 0) {
      load3(p, i, px, py, pz);
      towards(centres + 3 * k, px, py, pz, v);
      if (dot3(nx, ny, nz, v[0], v[1], v[2]) < 0.f) {
        nx = -nx;
        ny = -ny;
        nz = -nz;
      }
    }
    out[3 * i] = nx;
    out[3 * i + 1] = ny;
    out[3 * i + 2] = nz;
  }
}

// bilinear sample of image view[i] at p's pixel (u, w), pixel centres on the integers: x0 = floor(u), a = u - x0,
// x1 = min(x0 + 1, W - 1) (rows alike, b); top = c00 + a (c01 - c00), bottom = c10 + a (c11 - c10),
// out = top + b (bottom - top).  0 where view < 0 or p does not land in front and inside the view.
__global__ void k_gather(const float* __restrict__ p, const int32_t* __restrict__ view, int64_t m,
                         const float* __restrict__ mats, const float* __restrict__ images, int H, int W,
                         float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < m; i += (int64_t)gridDim.x * blockDim.x) {
    const int k = view[i];
    float px, py, pz, u, w;
    load3(p, i, px, py, pz);
    if (k < 0 || !pixel(mats + 12 * k, px, py, pz, H, W, u, w)) {
      out[3 * i] = out[3 * i + 1] = out[3 * i + 2] = 0.f;
      continue;
    }
    const float fu = floorf(u), fw = floorf(w);
    const float a = __fsub_rn(u, fu), b = __fsub_rn(w, fw);
    const int x0 = (int)fu, y0 = (int)fw, x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
    const float* img = images + (int64_t)k * H * W * 3;
    const float* c00 = img + ((int64_t)y0 * W + x0) * 3;
    const float* c01 = img + ((int64_t)y0 * W + x1) * 3;
    const float* c10 = img + ((int64_t)y1 * W + x0) * 3;
    const float* c11 = img + ((int64_t)y1 * W + x1) * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float top = __fadd_rn(c00[ch], __fmul_rn(a, __fsub_rn(c01[ch], c00[ch])));
      const float bot = __fadd_rn(c10[ch], __fmul_rn(a, __fsub_rn(c11[ch], c10[ch])));
      out[3 * i + ch] = __fadd_rn(top, __fmul_rn(b, __fsub_rn(bot, top)));
    }
  }
}

}  // namespace pt
}  // namespace nudf

using namespace nudf;
using namespace nudf::pt;

#define PT_REQUIRE_VIEWS(V) NUDF_REQUIRE((V) >= 0 && (V) <= kMaxViews, "the view count must lie in [0, NUDF_PT_MAX_VIEWS]")

int nudf_pt_normals(const float* g, int64_t m, float* out, void* stream) {
  NUDF_REQUIRE(m >= 0 && (m == 0 || (g && out)), "null pointer or negative count");
  if (m == 0) return 0;
  k_normals<<<grid_for(m), 256, 0, (cudaStream_t)stream>>>(g, m, out);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_pt_rank(const float* p, const float* n, int64_t m, const float* mats, const float* centres, int32_t V, int32_t H,
                 int32_t W, float cos_min, int32_t K, int32_t* cand, void* stream) {
  PT_REQUIRE_VIEWS(V);
  NUDF_REQUIRE(K >= 1 && K <= kMaxCand, "K must lie in [1, NUDF_PT_MAX_CAND]");
  NUDF_REQUIRE(H >= 1 && W >= 1 && H <= (1 << 24) && W <= (1 << 24), "image size out of range");
  NUDF_REQUIRE(m >= 0 && m <= INT32_MAX, "the point count must lie in [0, 2^31)");
  if (m == 0) return 0;
  NUDF_REQUIRE(p && n && cand && (V == 0 || (mats && centres)), "null pointer");
  k_rank<<<grid_for(m), 256, 0, (cudaStream_t)stream>>>(p, n, m, mats, centres, V, H, W, cos_min, K, cand);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_pt_start_count(const float* p, const float* n, const int32_t* cand, int32_t K, int32_t r, const int32_t* view,
                        int64_t m, const float* centres, float t_start, int32_t* counts, void* stream) {
  NUDF_REQUIRE(K >= 1 && K <= kMaxCand && r >= 0 && r < K, "need 0 <= r < K <= NUDF_PT_MAX_CAND");
  NUDF_REQUIRE(m >= 0 && m <= INT32_MAX, "the point count must lie in [0, 2^31)");
  if (m == 0) return 0;
  NUDF_REQUIRE(p && n && cand && view && centres && counts, "null pointer");
  return seg_compact<PairOut>(StartOp{p, n, centres, cand, view, K, r, t_start}, m, counts, nullptr, PairOut{}, stream);
}

int nudf_pt_start_emit(const float* p, const float* n, const int32_t* cand, int32_t K, int32_t r, const int32_t* view,
                       int64_t m, const float* centres, float t_start, const int64_t* offsets, int32_t* out_idx,
                       int32_t* out_cam, float* out_t, float* out_q, void* stream) {
  NUDF_REQUIRE(K >= 1 && K <= kMaxCand && r >= 0 && r < K, "need 0 <= r < K <= NUDF_PT_MAX_CAND");
  NUDF_REQUIRE(m >= 0 && m <= INT32_MAX, "the point count must lie in [0, 2^31)");
  if (m == 0) return 0;
  NUDF_REQUIRE(p && n && cand && view && centres && offsets && out_idx && out_cam && out_t && out_q, "null pointer");
  return seg_compact<PairOut>(StartOp{p, n, centres, cand, view, K, r, t_start}, m, nullptr, offsets,
                 PairOut{out_idx, out_cam, out_t, out_q}, stream);
}

int nudf_pt_trace_count(const float* p, const float* centres, const int32_t* idx, const int32_t* cam, const float* t,
                        const float* u, int64_t n, float hit, int32_t* counts, void* stream) {
  NUDF_REQUIRE(n >= 0, "negative count");
  if (n == 0) return 0;
  NUDF_REQUIRE(p && centres && idx && cam && t && u && counts, "null pointer");
  return seg_compact<PairOut>(StepOp{p, centres, idx, cam, t, u, hit, nullptr}, n, counts, nullptr, PairOut{}, stream);
}

int nudf_pt_trace_emit(const float* p, const float* centres, const int32_t* idx, const int32_t* cam, const float* t,
                       const float* u, int64_t n, float hit, const int64_t* offsets, int32_t* view, int32_t* out_idx,
                       int32_t* out_cam, float* out_t, float* out_q, void* stream) {
  NUDF_REQUIRE(n >= 0, "negative count");
  if (n == 0) return 0;
  NUDF_REQUIRE(p && centres && idx && cam && t && u && offsets && view && out_idx && out_cam && out_t && out_q,
               "null pointer");
  return seg_compact<PairOut>(StepOp{p, centres, idx, cam, t, u, hit, view}, n, nullptr, offsets,
                 PairOut{out_idx, out_cam, out_t, out_q}, stream);
}

int nudf_pt_orient(const float* p, const float* n, const int32_t* view, int64_t m, const float* centres, float* out,
                   void* stream) {
  NUDF_REQUIRE(m >= 0, "negative count");
  if (m == 0) return 0;
  NUDF_REQUIRE(p && n && view && out, "null pointer");
  k_orient<<<grid_for(m), 256, 0, (cudaStream_t)stream>>>(p, n, view, m, centres, out);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_pt_gather(const float* p, const int32_t* view, int64_t m, const float* mats, const float* images, int32_t V,
                   int32_t H, int32_t W, float* out, void* stream) {
  PT_REQUIRE_VIEWS(V);
  NUDF_REQUIRE(H >= 1 && W >= 1 && H <= (1 << 24) && W <= (1 << 24), "image size out of range");
  NUDF_REQUIRE(m >= 0, "negative count");
  if (m == 0) return 0;
  NUDF_REQUIRE(p && view && out && (V == 0 || (mats && images)), "null pointer");
  k_gather<<<grid_for(m), 256, 0, (cudaStream_t)stream>>>(p, view, m, mats, images, H, W, out);
  NUDF_LAUNCH_OK();
  return 0;
}

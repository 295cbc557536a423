// Mask and visual-hull cleaning of a DTU mesh on the device: the per-vertex stages of the reference's
// evaluation/clean_dtu_mesh.py (clean_points_by_mask, clean_points_by_visualhull).  neuraludf_b200/clean.py drives them;
// tests/proto/mesh_clean.py restates both in NumPy.
//   1. dilate and threshold  grayscale max filter of every [H, W] uint8 mask over a structuring element given as one column
//                            interval per row (the ellipse is one), pixels outside the image not contributing (cv2.dilate's
//                            default border), then bit-packed: bit b of word w of a row is column 32 w + b, set where the
//                            dilated value is > 128 (mask pass) or < 128 (hull pass).  One block per 64 x 32 output tile:
//                            the tile plus its halo sits in shared memory and is turned, level by level, into a range-max
//                            table (level p holds max(src[x .. x + 2^p - 1]), built from level p - 1 by ping-pong), so an
//                            element row of length L costs two lookups at level floor(log2 L) instead of L.  Rows are
//                            visited in order of increasing length, so every level is built once.
//   2. project and vote      one thread per vertex, the views' 3 x 4 matrices in shared memory, the packed masks read
//                            through L2.  fp64, one rounding per operation: s_r = ((m_r0 x + m_r1 y) + m_r2 z) + m_r3,
//                            q = (s_0 / s_2, s_1 / s_2), u = rint(q_x) + 1, v = rint(q_y) + 1 (half to even, as np.round).
//                            A view counts when border <= u <= W - border and border <= v <= H - border and the padded mask
//                            (the bit mask inside a ring of ones) is set at (v, u).  NaN / inf / huge q fail the range test,
//                            which is where NumPy's int32 cast of them ends up too.
#include <algorithm>

#include "../../include/nudf.h"
#include "common.cuh"

namespace nudf {
namespace cl {

constexpr int kTileW = 64;           // output columns per block: two packed words per row
constexpr int kTileH = 32;           // output rows per block
constexpr int kThreads = 256;        // 4 rows at a time, kTileH / 4 rows per thread
constexpr int kRowsPerThread = kTileH / (kThreads / kTileW);
constexpr int kMaxK = 255;           // largest element height / width
constexpr int kMaxViews = 512;       // 512 x 12 doubles of matrices in shared memory

// the non-empty rows of the element sorted by length: element row dy[e], columns [j1[e], j1[e] + len[e])
struct Element {
  int32_t kw, kh, ax, ay, n;
  int16_t dy[kMaxK], j1[kMaxK], len[kMaxK];
};

template <bool BELOW>
__global__ void __launch_bounds__(kThreads) k_dilate(const uint8_t* __restrict__ img, int H, int W, int Wp, Element E,
                                                     uint32_t* __restrict__ out) {
  extern __shared__ uint8_t smem[];
  const int SW = kTileW + E.kw - 1, SH = kTileH + E.kh - 1, S = SW * SH;
  uint8_t* a = smem;
  uint8_t* b = smem + S;
  const int x0 = blockIdx.x * kTileW, y0 = blockIdx.y * kTileH;
  const uint8_t* src = img + (size_t)blockIdx.z * H * W;
  // smem (r, c) = source pixel (y0 - ay + r, x0 - ax + c); outside the image 0, the identity of max over uint8
  for (int i = threadIdx.x; i < S; i += kThreads) {
    const int r = i / SW, c = i - r * SW;
    const int y = y0 - E.ay + r, x = x0 - E.ax + c;
    a[i] = (y >= 0 && y < H && x >= 0 && x < W) ? src[(size_t)y * W + x] : 0;
  }
  __syncthreads();
  const int tx = threadIdx.x % kTileW, ty = threadIdx.x / kTileW;
  int acc[kRowsPerThread];
#pragma unroll
  for (int r = 0; r < kRowsPerThread; ++r) acc[r] = 0;
  int level = 0;
  for (int e = 0; e < E.n; ++e) {                    // block-uniform loop: the syncs below are reached by every thread
    const int len = E.len[e];
    const int p = 31 - __clz(len);
    while (level < p) {
      const int s = 1 << level;
      __syncthreads();                               // every read of level `level - 1` (now in b) is done
      for (int i = threadIdx.x; i < S; i += kThreads) {
        const int c = i % SW;
        b[i] = c + s < SW ? max(a[i], a[i + s]) : a[i];
      }
      __syncthreads();
      uint8_t* t = a; a = b; b = t;
      ++level;
    }
    const int c0 = tx + E.j1[e], c1 = tx + E.j1[e] + len - (1 << p);
    const uint8_t* row = a + (ty + E.dy[e]) * SW;
#pragma unroll
    for (int r = 0; r < kRowsPerThread; ++r) {
      const uint8_t* q = row + r * (kThreads / kTileW) * SW;
      acc[r] = max(acc[r], (int)max(q[c0], q[c1]));
    }
  }
  const int x = x0 + tx;
  const unsigned lane = threadIdx.x & 31;
#pragma unroll
  for (int r = 0; r < kRowsPerThread; ++r) {
    const int y = y0 + ty + r * (kThreads / kTileW);
    const bool bit = x < W && (BELOW ? acc[r] < 128 : acc[r] > 128);
    const unsigned word = __ballot_sync(0xffffffffu, bit);       // warp = 32 consecutive columns of one row
    if (lane == 0 && y < H && (x >> 5) < Wp) out[((size_t)blockIdx.z * H + y) * Wp + (x >> 5)] = word;
  }
}

__global__ void __launch_bounds__(256) k_vote(const double* __restrict__ pts, int64_t n, const double* __restrict__ mats,
                                              int V, const uint32_t* __restrict__ masks, int H, int W, int Wp, int border,
                                              int32_t* __restrict__ counts) {
  extern __shared__ double sm_mats[];
  for (int i = threadIdx.x; i < 12 * V; i += blockDim.x) sm_mats[i] = mats[i];
  __syncthreads();
  const double ulo = border, uhi = W - border, vlo = border, vhi = H - border;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const double x = pts[3 * t], y = pts[3 * t + 1], z = pts[3 * t + 2];
    int32_t c = 0;
    for (int v = 0; v < V; ++v) {
      const double* M = sm_mats + 12 * v;
      double s[3];
#pragma unroll
      for (int r = 0; r < 3; ++r)
        s[r] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(M[4 * r], x), __dmul_rn(M[4 * r + 1], y)), __dmul_rn(M[4 * r + 2], z)),
                         M[4 * r + 3]);
      const double u = rint(__ddiv_rn(s[0], s[2])) + 1.0, w = rint(__ddiv_rn(s[1], s[2])) + 1.0;
      if (!(u >= ulo && u <= uhi && w >= vlo && w <= vhi)) continue;     // NaN fails here
      const int iu = (int)u, iv = (int)w;
      // padded (iv, iu): the ring of ones at row 0 / column 0 (rows H + 1, columns W + 1 are out of range), else the mask
      if (iu == 0 || iv == 0) { ++c; continue; }
      const int col = iu - 1;
      c += (masks[((size_t)v * H + (iv - 1)) * Wp + (col >> 5)] >> (col & 31)) & 1u;
    }
    counts[t] = c;
  }
}

}  // namespace cl
}  // namespace nudf

using namespace nudf;
using namespace nudf::cl;

int nudf_cl_dilate(const uint8_t* masks, int32_t n_views, int32_t height, int32_t width, const int32_t* row_lo,
                   const int32_t* row_hi, int32_t kh, int32_t kw, int32_t anchor_x, int32_t anchor_y, int32_t below,
                   uint32_t* packed, void* stream) {
  NUDF_REQUIRE(masks && row_lo && row_hi && packed, "null pointer");
  NUDF_REQUIRE(n_views >= 0 && height >= 0 && width >= 0, "negative size");
  NUDF_REQUIRE(n_views <= 65535 && height <= 65535 * kTileH, "too many views or rows");
  NUDF_REQUIRE(kh >= 1 && kw >= 1 && kh <= kMaxK && kw <= kMaxK, "element sides must be in [1, 255]");
  NUDF_REQUIRE(anchor_x >= 0 && anchor_x < kw && anchor_y >= 0 && anchor_y < kh, "anchor outside the element");
  Element E{};
  E.kw = kw, E.kh = kh, E.ax = anchor_x, E.ay = anchor_y, E.n = 0;
  for (int i = 0; i < kh; ++i) {
    NUDF_REQUIRE(row_lo[i] >= 0 && row_hi[i] <= kw, "element row interval outside [0, kw]");
    if (row_hi[i] > row_lo[i]) {
      E.dy[E.n] = (int16_t)i, E.j1[E.n] = (int16_t)row_lo[i], E.len[E.n] = (int16_t)(row_hi[i] - row_lo[i]);
      ++E.n;
    }
  }
  {  // stable sort of the rows by length: the levels of the range-max table are then built in order
    int idx[kMaxK];
    for (int e = 0; e < E.n; ++e) idx[e] = e;
    std::stable_sort(idx, idx + E.n, [&](int p, int q) { return E.len[p] < E.len[q]; });
    Element s = E;
    for (int e = 0; e < E.n; ++e) s.dy[e] = E.dy[idx[e]], s.j1[e] = E.j1[idx[e]], s.len[e] = E.len[idx[e]];
    E = s;
  }
  if (n_views == 0 || height == 0 || width == 0) return 0;
  const size_t smem = 2 * (size_t)(kTileW + kw - 1) * (kTileH + kh - 1);
  const int Wp = (int)cdiv(width, 32);
  dim3 grid((unsigned)cdiv(width, kTileW), (unsigned)cdiv(height, kTileH), (unsigned)n_views);
  cudaStream_t st = (cudaStream_t)stream;
  if (below) {
    NUDF_CUDA_OK(cudaFuncSetAttribute(k_dilate<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_dilate<true><<<grid, kThreads, smem, st>>>(masks, height, width, Wp, E, packed);
  } else {
    NUDF_CUDA_OK(cudaFuncSetAttribute(k_dilate<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_dilate<false><<<grid, kThreads, smem, st>>>(masks, height, width, Wp, E, packed);
  }
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_cl_vote(const double* points, int64_t n, const double* mats, int32_t n_views, const uint32_t* packed,
                 int32_t height, int32_t width, int32_t border, int32_t* counts, void* stream) {
  NUDF_REQUIRE(points && mats && packed && counts, "null pointer");
  NUDF_REQUIRE(n >= 0 && n_views >= 0 && height >= 0 && width >= 0 && border >= 0, "negative size");
  NUDF_REQUIRE(n_views <= kMaxViews, "at most 512 views");
  if (n == 0) return 0;
  const size_t smem = sizeof(double) * 12 * (size_t)n_views;
  k_vote<<<grid_for(n), 256, smem, (cudaStream_t)stream>>>(points, n, mats, n_views, packed, height, width,
                                                           (int)cdiv(width, 32), border, counts);
  NUDF_LAUNCH_OK();
  return 0;
}

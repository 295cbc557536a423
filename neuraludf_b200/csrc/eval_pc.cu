// Chamfer evaluation of a reconstruction against a ground-truth point cloud on the device: the shared stages of the DTU and
// DeepFashion3D evaluation scripts (evaluation/eval_dtu_python.py, eval_deepfashion_python.py).  neuraludf_b200/evaluate.py
// drives them; tests/proto/eval_pc.py restates every stage in NumPy / sklearn.
//   1. surface sampling   per triangle with area2 > 0: n1 = floor(l1 / thr), n2 = floor(l2 / thr), thr = density *
//                         sqrt(l1 l2 / area2); the points (v1 a + v2 b) + v0 for a = (i + .5) / max(n1, 1e-7),
//                         b = (j + .5) / max(n2, 1e-7), 0 <= i <= n1, 0 <= j <= n2, a + b < 1, row-major.  Every operation is
//                         a separately rounded fp64 __d*_rn in NumPy's order, so the samples are bit-identical.  Count, then
//                         (caller's exclusive scan) emit; one warp per triangle, lanes over the rows i.
//   2. radius graph       uniform grid of cell edge r (1 + 1e-6) over the shuffled points (a pair within r in fp64 is then
//                         at most one cell apart on every axis); CSR lists of each point's LOWER-rank neighbours with
//                         (dx^2 + dy^2) + dz^2 <= r * r -- sklearn's KD-tree test, inclusive at r.
//   3. greedy downsample  the scripts' loop (walk the shuffled points; a point still marked keeps itself and unmarks its
//                         r-neighbours) keeps the lexicographically-first maximal independent set of the radius graph.  In
//                         rounds: an undecided point is OUT once a lower-rank neighbour is IN, IN once all of them are OUT.
//                         Decisions are final and correct whenever they are taken, so the in-place update is race-tolerant;
//                         the lowest-rank undecided point always decides, and a random order needs O(log^2 n) rounds w.h.p.
//                         (Blelloch, Fineman & Shun, SPAA 2012).
//   4. nearest distance   exact, bounded: targets Morton-sorted into 32-point leaves under an implicit complete binary tree
//                         of AABBs (node i has children 2i+1, 2i+2; leaf l is node L-1+l); per query a depth-first
//                         branch-and-bound seeded with max_dist, queries in Morton order for warp coherence.  The distance is
//                         sqrt((dx^2 + dy^2) + dz^2) in fp64 as in the KD-tree; a query with no target below max_dist gets +inf.
#include <algorithm>

#include "../../include/nudf.h"
#include "common.cuh"

namespace nudf {
namespace pc {

constexpr int kLeaf = 32;          // targets per BVH leaf
constexpr int kStack = 40;         // traversal stack: >= tree depth (log2 of the leaf count)

__device__ __forceinline__ double sq3(double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z));
}

// ---- 1. surface sampling --------------------------------------------------------------------------------------------------
struct Tri {
  double v0[3], e1[3], e2[3];
  double n1, n2, den1, den2;
};

// false for a triangle the scripts drop (area2 == 0, or a non-finite area)
__device__ __forceinline__ bool tri_setup(const double* __restrict__ V, const int64_t* __restrict__ F, int64_t f, double density,
                                          Tri& T) {
  const int64_t a = F[3 * f], b = F[3 * f + 1], c = F[3 * f + 2];
  for (int k = 0; k < 3; ++k) {
    T.v0[k] = V[3 * a + k];
    T.e1[k] = __dsub_rn(V[3 * b + k], T.v0[k]);
    T.e2[k] = __dsub_rn(V[3 * c + k], T.v0[k]);
  }
  const double l1 = __dsqrt_rn(sq3(T.e1[0], T.e1[1], T.e1[2]));
  const double l2 = __dsqrt_rn(sq3(T.e2[0], T.e2[1], T.e2[2]));
  // np.cross: a1 b2 - a2 b1, a2 b0 - a0 b2, a0 b1 - a1 b0
  const double c0 = __dsub_rn(__dmul_rn(T.e1[1], T.e2[2]), __dmul_rn(T.e1[2], T.e2[1]));
  const double c1 = __dsub_rn(__dmul_rn(T.e1[2], T.e2[0]), __dmul_rn(T.e1[0], T.e2[2]));
  const double c2 = __dsub_rn(__dmul_rn(T.e1[0], T.e2[1]), __dmul_rn(T.e1[1], T.e2[0]));
  const double area2 = __dsqrt_rn(sq3(c0, c1, c2));
  if (!(area2 > 0.0)) return false;
  const double thr = __dmul_rn(density, __dsqrt_rn(__ddiv_rn(__dmul_rn(l1, l2), area2)));
  T.n1 = floor(__ddiv_rn(l1, thr));
  T.n2 = floor(__ddiv_rn(l2, thr));
  if (!(T.n1 >= 0.0 && T.n2 >= 0.0 && T.n1 < 9.0e15 && T.n2 < 9.0e15)) return false;   // non-finite geometry: no samples
  T.den1 = T.n1 > 1e-7 ? T.n1 : 1e-7;      // max(n, 1e-7)
  T.den2 = T.n2 > 1e-7 ? T.n2 : 1e-7;
  return true;
}

// samples of row i: the number of j in [0, n2] with a + b < 1.  a + b is non-decreasing in j under round-to-nearest, so the
// kept j form a prefix and a binary search on the exact fp64 predicate finds its length (no closed form: it can disagree at ties).
__device__ __forceinline__ int64_t row_count(const Tri& T, double a) {
  int64_t lo = 0, hi = (int64_t)T.n2 + 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    const double b = __ddiv_rn(__dadd_rn((double)mid, 0.5), T.den2);
    if (__dadd_rn(a, b) < 1.0) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ double row_a(const Tri& T, int64_t i) { return __ddiv_rn(__dadd_rn((double)i, 0.5), T.den1); }

__global__ void k_sample_count(const double* __restrict__ V, const int64_t* __restrict__ F, int64_t n_faces, double density,
                               int64_t* __restrict__ counts) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t f = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; f < n_faces; f += warps) {
    Tri T;
    int64_t c = 0;
    if (tri_setup(V, F, f, density, T))
      for (int64_t i = lane; i <= (int64_t)T.n1; i += 32) c += row_count(T, row_a(T, i));
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) counts[f] = c;
  }
}

__global__ void k_sample_emit(const double* __restrict__ V, const int64_t* __restrict__ F, int64_t n_faces, double density,
                              const int64_t* __restrict__ offsets, double* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t f = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5; f < n_faces; f += warps) {
    Tri T;
    if (!tri_setup(V, F, f, density, T)) continue;          // warp-uniform
    int64_t base = offsets[f];
    for (int64_t i0 = 0; i0 <= (int64_t)T.n1; i0 += 32) {
      const int64_t i = i0 + lane;
      const double a = row_a(T, i);
      const int64_t c = i <= (int64_t)T.n1 ? row_count(T, a) : 0;
      int64_t incl = c;                                      // inclusive warp scan of the row counts
      for (int o = 1; o < 32; o <<= 1) {
        const int64_t y = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += y;
      }
      double* q = out + 3 * (base + incl - c);
      for (int64_t j = 0; j < c; ++j) {
        const double b = __ddiv_rn(__dadd_rn((double)j, 0.5), T.den2);
#pragma unroll
        for (int k = 0; k < 3; ++k) q[3 * j + k] = __dadd_rn(__dadd_rn(__dmul_rn(T.e1[k], a), __dmul_rn(T.e2[k], b)), T.v0[k]);
      }
      base += __shfl_sync(0xffffffffu, incl, 31);
    }
  }
}

// ---- 2. radius graph ------------------------------------------------------------------------------------------------------
struct Grid {
  double lo[3], h;
  int64_t n[3];
};

__global__ void k_cell_keys(const double* __restrict__ p, int64_t n, Grid G, int64_t* __restrict__ keys) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    int64_t c[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double u = floor(__ddiv_rn(__dsub_rn(p[3 * t + k], G.lo[k]), G.h));
      c[k] = u <= 0.0 ? 0 : (u >= (double)(G.n[k] - 1) ? G.n[k] - 1 : (int64_t)u);
    }
    keys[t] = (c[0] * G.n[1] + c[1]) * G.n[2] + c[2];
  }
}

__device__ __forceinline__ int64_t lower_bound(const int64_t* __restrict__ a, int64_t n, int64_t key) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// thread t: the point at sorted position t (rank order[t]); scans the 27 cells around it (9 runs of up to 3 consecutive keys)
template <bool EMIT>
__global__ void k_radius(const double* __restrict__ ps, const int64_t* __restrict__ order, const int64_t* __restrict__ skeys,
                         int64_t n, const int64_t* __restrict__ cells, const int64_t* __restrict__ cstart, int64_t n_cells, Grid G,
                         double r2, int32_t* __restrict__ counts, const int64_t* __restrict__ offsets, int32_t* __restrict__ nbr) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t me = order[t], key = skeys[t];
    const int64_t iz = key % G.n[2], iy = (key / G.n[2]) % G.n[1], ix = key / (G.n[1] * G.n[2]);
    const double x = ps[3 * t], y = ps[3 * t + 1], z = ps[3 * t + 2];
    const int64_t z0 = iz > 0 ? iz - 1 : 0, z1 = iz + 1 < G.n[2] ? iz + 1 : iz;
    int64_t cnt = 0, pos = EMIT ? offsets[me] : 0;
    for (int64_t jx = ix - 1; jx <= ix + 1; ++jx) {
      if (jx < 0 || jx >= G.n[0]) continue;
      for (int64_t jy = iy - 1; jy <= iy + 1; ++jy) {
        if (jy < 0 || jy >= G.n[1]) continue;
        const int64_t row = (jx * G.n[1] + jy) * G.n[2];
        for (int64_t c = lower_bound(cells, n_cells, row + z0); c < n_cells && cells[c] <= row + z1; ++c) {
          for (int64_t s = cstart[c]; s < cstart[c + 1]; ++s) {
            const int64_t o = order[s];
            if (o >= me) continue;
            const double d2 = sq3(__dsub_rn(x, ps[3 * s]), __dsub_rn(y, ps[3 * s + 1]), __dsub_rn(z, ps[3 * s + 2]));
            if (d2 <= r2) {
              if (EMIT) nbr[pos++] = (int32_t)o;
              else ++cnt;
            }
          }
        }
      }
    }
    if (!EMIT) counts[me] = (int32_t)cnt;
  }
}

// ---- 3. greedy downsampling: lexicographically-first MIS in rounds ---------------------------------------------------------
enum : uint8_t { UNDECIDED = 0, KEPT = 1, DROPPED = 2 };

__global__ void k_mis_round(const int64_t* __restrict__ off, const int32_t* __restrict__ nbr, int64_t n, uint8_t* state,
                            int32_t* __restrict__ pending) {
  volatile uint8_t* vs = state;
  for (int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; v < n; v += (int64_t)gridDim.x * blockDim.x) {
    if (vs[v] != UNDECIDED) continue;
    bool all_out = true, any_in = false;
    for (int64_t e = off[v]; e < off[v + 1]; ++e) {
      const uint8_t s = vs[nbr[e]];
      if (s == KEPT) { any_in = true; break; }
      if (s == UNDECIDED) all_out = false;
    }
    if (any_in) vs[v] = DROPPED;
    else if (all_out) vs[v] = KEPT;
    else *pending = 1;
  }
}

// ---- 4. bounded exact nearest distance -------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t spread21(uint64_t v) {
  v &= 0x1fffffull;
  v = (v | (v << 32)) & 0x1f00000000ffffull;
  v = (v | (v << 16)) & 0x1f0000ff0000ffull;
  v = (v | (v << 8)) & 0x100f00f00f00f00full;
  v = (v | (v << 4)) & 0x10c30c30c30c30c3ull;
  v = (v | (v << 2)) & 0x1249249249249249ull;
  return v;
}

__global__ void k_morton(const double* __restrict__ p, int64_t n, double lx, double ly, double lz, double scale,
                         int64_t* __restrict__ codes) {
  const double lo[3] = {lx, ly, lz};
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    uint64_t code = 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double u = (p[3 * t + k] - lo[k]) * scale;
      const uint64_t q = u > 0.0 ? (u < 2097151.0 ? (uint64_t)u : 2097151ull) : 0ull;   // NaN -> 0
      code |= spread21(q) << (2 - k);
    }
    codes[t] = (int64_t)code;
  }
}

// boxes[node] = {lo x, y, z, hi x, y, z}; an empty leaf is {+inf, -inf} (its lower bound is +inf)
__global__ void k_bvh_leaves(const double* __restrict__ ts, int64_t n, int64_t n_leaves, double* __restrict__ boxes) {
  for (int64_t l = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; l < n_leaves; l += (int64_t)gridDim.x * blockDim.x) {
    double lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    const int64_t e = min(n, (l + 1) * kLeaf);
    for (int64_t s = l * kLeaf; s < e; ++s)
      for (int k = 0; k < 3; ++k) { lo[k] = fmin(lo[k], ts[3 * s + k]); hi[k] = fmax(hi[k], ts[3 * s + k]); }
    double* b = boxes + 6 * (n_leaves - 1 + l);
    for (int k = 0; k < 3; ++k) { b[k] = lo[k]; b[3 + k] = hi[k]; }
  }
}

__global__ void k_bvh_level(double* __restrict__ boxes, int64_t first, int64_t count) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < count; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = first + t;
    const double* a = boxes + 6 * (2 * i + 1);
    const double* b = boxes + 6 * (2 * i + 2);
    for (int k = 0; k < 3; ++k) {
      boxes[6 * i + k] = fmin(a[k], b[k]);
      boxes[6 * i + 3 + k] = fmax(a[3 + k], b[3 + k]);
    }
  }
}

// lower bound of the computed distance^2 of any point of the box: per axis the gap max(lo - q, q - hi, 0), squared and summed
// in the distance's own order.  Rounding is monotone, so it never exceeds the computed distance^2 of a point inside the box.
__device__ __forceinline__ double box_lb(const double* __restrict__ b, double x, double y, double z) {
  const double gx = x < b[0] ? __dsub_rn(b[0], x) : (x > b[3] ? __dsub_rn(x, b[3]) : 0.0);
  const double gy = y < b[1] ? __dsub_rn(b[1], y) : (y > b[4] ? __dsub_rn(y, b[4]) : 0.0);
  const double gz = z < b[2] ? __dsub_rn(b[2], z) : (z > b[5] ? __dsub_rn(z, b[5]) : 0.0);
  return sq3(gx, gy, gz);
}

__global__ void __launch_bounds__(128) k_nearest(const double* __restrict__ qs, int64_t n_q, const int64_t* __restrict__ qorder,
                                                 const double* __restrict__ ts, int64_t n_t, const double* __restrict__ boxes,
                                                 int64_t n_leaves, double bound2, double max_dist, double* __restrict__ dist) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n_q; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t q = qorder ? qorder[t] : t;
    const double x = qs[3 * q], y = qs[3 * q + 1], z = qs[3 * q + 2];
    double best = bound2;
    bool found = false;
    int64_t stack[kStack];
    double stack_lb[kStack];
    int sp = 0;
    int64_t node = 0;
    bool go = box_lb(boxes, x, y, z) <= best;
    while (go) {
      if (node >= n_leaves - 1) {
        const int64_t l = node - (n_leaves - 1);
        const int64_t e = min(n_t, (l + 1) * kLeaf);
        for (int64_t s = l * kLeaf; s < e; ++s) {
          const double d2 = sq3(__dsub_rn(x, ts[3 * s]), __dsub_rn(y, ts[3 * s + 1]), __dsub_rn(z, ts[3 * s + 2]));
          if (d2 <= best) { best = d2; found = true; }
        }
      } else {
        int64_t c0 = 2 * node + 1, c1 = 2 * node + 2;
        double l0 = box_lb(boxes + 6 * c0, x, y, z), l1 = box_lb(boxes + 6 * c1, x, y, z);
        if (l1 < l0) { const int64_t ct = c0; c0 = c1; c1 = ct; const double lt = l0; l0 = l1; l1 = lt; }
        if (l0 <= best) {
          if (l1 <= best) { stack[sp] = c1; stack_lb[sp] = l1; ++sp; }
          node = c0;
          continue;
        }
      }
      go = false;
      while (sp > 0) {
        --sp;
        if (stack_lb[sp] <= best) { node = stack[sp]; go = true; break; }
      }
    }
    const double d = __dsqrt_rn(best);
    dist[q] = (found && d < max_dist) ? d : INFINITY;
  }
}

static inline unsigned grid_for(int64_t n, int per_block = 256) {
  return (unsigned)std::min<int64_t>(std::max<int64_t>(cdiv(n, per_block), 1), 65535ll * 8);
}

}  // namespace pc
}  // namespace nudf

using namespace nudf;
using namespace nudf::pc;

int nudf_pc_sample_count(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, double density,
                         int64_t* counts, void* stream) {
  NUDF_REQUIRE(verts && faces && counts && n_verts >= 0 && n_faces >= 0, "null pointer or negative count");
  NUDF_REQUIRE(density > 0.0, "density must be positive");
  if (n_faces == 0) return 0;
  k_sample_count<<<grid_for(32 * n_faces), 256, 0, (cudaStream_t)stream>>>(verts, faces, n_faces, density, counts);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_pc_sample_emit(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, double density,
                        const int64_t* offsets, double* points, void* stream) {
  NUDF_REQUIRE(verts && faces && offsets && points && n_verts >= 0 && n_faces >= 0, "null pointer or negative count");
  NUDF_REQUIRE(density > 0.0, "density must be positive");
  if (n_faces == 0) return 0;
  k_sample_emit<<<grid_for(32 * n_faces), 256, 0, (cudaStream_t)stream>>>(verts, faces, n_faces, density, offsets, points);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_pc_cell_keys(const double* points, int64_t n, const double* lo, double cell, const int64_t* dims, int64_t* keys,
                      void* stream) {
  NUDF_REQUIRE(points && lo && dims && keys && n >= 0, "null pointer or negative count");
  NUDF_REQUIRE(cell > 0.0 && dims[0] > 0 && dims[1] > 0 && dims[2] > 0, "cell edge and grid dimensions must be positive");
  NUDF_REQUIRE(dims[0] <= (INT64_C(1) << 62) / dims[1] / dims[2], "grid has too many cells for 64-bit keys");
  if (n == 0) return 0;
  Grid G{{lo[0], lo[1], lo[2]}, cell, {dims[0], dims[1], dims[2]}};
  k_cell_keys<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(points, n, G, keys);
  NUDF_LAUNCH_OK();
  return 0;
}

static int radius_pass(bool emit, const double* sorted_points, const int64_t* order, const int64_t* sorted_keys, int64_t n,
                       const int64_t* cells, const int64_t* cell_start, int64_t n_cells, const double* lo, double cell,
                       const int64_t* dims, double radius, int32_t* counts, const int64_t* offsets, int32_t* nbr, void* stream) {
  NUDF_REQUIRE(sorted_points && order && sorted_keys && cells && cell_start && lo && dims && n >= 0 && n_cells >= 0,
               "null pointer or negative count");
  NUDF_REQUIRE(n < (INT64_C(1) << 31), "at most 2^31 - 1 points");
  NUDF_REQUIRE(radius > 0.0 && cell > 0.0, "radius and cell edge must be positive");
  if (n == 0) return 0;
  Grid G{{lo[0], lo[1], lo[2]}, cell, {dims[0], dims[1], dims[2]}};
  const double r2 = radius * radius;
  if (emit)
    k_radius<true><<<grid_for(n, 128), 128, 0, (cudaStream_t)stream>>>(sorted_points, order, sorted_keys, n, cells, cell_start,
                                                                       n_cells, G, r2, nullptr, offsets, nbr);
  else
    k_radius<false><<<grid_for(n, 128), 128, 0, (cudaStream_t)stream>>>(sorted_points, order, sorted_keys, n, cells, cell_start,
                                                                        n_cells, G, r2, counts, nullptr, nullptr);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_pc_radius_count(const double* sorted_points, const int64_t* order, const int64_t* sorted_keys, int64_t n,
                         const int64_t* cells, const int64_t* cell_start, int64_t n_cells, const double* lo, double cell,
                         const int64_t* dims, double radius, int32_t* counts, void* stream) {
  NUDF_REQUIRE(counts, "null pointer");
  return radius_pass(false, sorted_points, order, sorted_keys, n, cells, cell_start, n_cells, lo, cell, dims, radius, counts,
                     nullptr, nullptr, stream);
}

int nudf_pc_radius_emit(const double* sorted_points, const int64_t* order, const int64_t* sorted_keys, int64_t n,
                        const int64_t* cells, const int64_t* cell_start, int64_t n_cells, const double* lo, double cell,
                        const int64_t* dims, double radius, const int64_t* offsets, int32_t* nbr, void* stream) {
  NUDF_REQUIRE(offsets && nbr, "null pointer");
  return radius_pass(true, sorted_points, order, sorted_keys, n, cells, cell_start, n_cells, lo, cell, dims, radius, nullptr,
                     offsets, nbr, stream);
}

int nudf_pc_greedy_mis(const int64_t* offsets, const int32_t* nbr, int64_t n, uint8_t* state, int32_t* flag_ws,
                       int32_t* rounds, void* stream) {
  NUDF_REQUIRE(offsets && state && flag_ws && n >= 0, "null pointer or negative count");
  if (rounds) *rounds = 0;
  if (n == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  NUDF_CUDA_OK(cudaMemsetAsync(state, UNDECIDED, (size_t)n, st));
  // Termination: in every round the lowest-rank undecided point has only decided lower-rank neighbours, so it decides;
  // at most n rounds, O(log^2 n) w.h.p. for a random order.  Each round costs one host read of flag_ws.
  int32_t pending = 1, r = 0;
  while (pending) {
    NUDF_CUDA_OK(cudaMemsetAsync(flag_ws, 0, sizeof(int32_t), st));
    k_mis_round<<<grid_for(n), 256, 0, st>>>(offsets, nbr, n, state, flag_ws);
    NUDF_LAUNCH_OK();
    ++r;
    NUDF_CUDA_OK(cudaMemcpyAsync(&pending, flag_ws, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    NUDF_CUDA_OK(cudaStreamSynchronize(st));
  }
  if (rounds) *rounds = r;
  return 0;
}

int nudf_pc_morton(const double* points, int64_t n, const double* lo, double scale, int64_t* codes, void* stream) {
  NUDF_REQUIRE(points && lo && codes && n >= 0, "null pointer or negative count");
  if (n == 0) return 0;
  k_morton<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(points, n, lo[0], lo[1], lo[2], scale, codes);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_pc_bvh_build(const double* sorted_targets, int64_t n, int64_t n_leaves, double* boxes, void* stream) {
  NUDF_REQUIRE(sorted_targets && boxes && n > 0, "null pointer or no targets");
  NUDF_REQUIRE(n_leaves >= 1 && (n_leaves & (n_leaves - 1)) == 0 && n_leaves * kLeaf >= n,
               "n_leaves must be a power of two with n_leaves * 32 >= n");
  NUDF_REQUIRE(n_leaves <= (INT64_C(1) << (kStack - 2)), "too many leaves");
  cudaStream_t st = (cudaStream_t)stream;
  k_bvh_leaves<<<grid_for(n_leaves), 256, 0, st>>>(sorted_targets, n, n_leaves, boxes);
  NUDF_LAUNCH_OK();
  for (int64_t count = n_leaves >> 1; count >= 1; count >>= 1) {   // level with `count` nodes starts at node count - 1
    k_bvh_level<<<grid_for(count), 256, 0, st>>>(boxes, count - 1, count);
    NUDF_LAUNCH_OK();
  }
  return 0;
}

int nudf_pc_nearest(const double* queries, int64_t n_queries, const int64_t* query_order, const double* sorted_targets,
                    int64_t n_targets, const double* boxes, int64_t n_leaves, double max_dist, double* dist, void* stream) {
  NUDF_REQUIRE(queries && sorted_targets && boxes && dist && n_queries >= 0 && n_targets > 0, "null pointer or no targets");
  NUDF_REQUIRE(n_leaves >= 1 && (n_leaves & (n_leaves - 1)) == 0 && n_leaves * kLeaf >= n_targets, "bad leaf count");
  NUDF_REQUIRE(max_dist > 0.0, "max_dist must be positive (+inf: unbounded)");
  if (n_queries == 0) return 0;
  // prune above max_dist^2 (1 + 1e-12): any computed distance^2 whose root is below max_dist lies below it
  const double bound2 = isinf(max_dist) ? INFINITY : max_dist * max_dist * (1.0 + 1e-12);
  k_nearest<<<grid_for(n_queries, 128), 128, 0, (cudaStream_t)stream>>>(queries, n_queries, query_order, sorted_targets,
                                                                         n_targets, boxes, n_leaves, bound2, max_dist, dist);
  NUDF_LAUNCH_OK();
  return 0;
}

// Narrow-band evaluation of an N^3 lattice, coarse to fine: the stages of grid.udf_band (the lattice on [-1,1]^3,
// voxel = 2 / (N - 1)) and grid.iso_band (the lattice of three fp32 axis tables on any box).  tests/proto/udf_band.py and
// tests/proto/iso_band.py restate every kernel in NumPy with the same fp64 operation order.
//   lattice of stride s   per axis the coordinates 0, s, 2 s, ... and N - 1 (the clamped last plane when (N - 1) % s != 0);
//   block of stride s     the box [a, min(a + s, N - 1)] per axis, a a multiple of s below N - 1: cdiv(N - 1, s) per axis,
//                         numbered ((bx * nb) + by) * nb + bz;
//   block test            a candidate block (every block at the first level, else a block inside a kept block of the
//                         previous stride) is kept when  min(corner value) - L r < tau,  r = the largest distance from a
//                         point of the box to its nearest corner (half its diagonal, the box's own extents).  If the field
//                         is L-Lipschitz, a culled block holds no point with a value < tau.  fp64, one rounding per
//                         operation, with slack against every rounding involved (the spacing rules below).  A NaN corner
//                         keeps the block.
//   point emission        a kept block of stride s emits the points of the stride-t lattice (t divides s) in its closed box
//                         that are not on the stride-s lattice; a point on a face or edge shared with other kept blocks is
//                         emitted by the lowest-numbered of them.  Count, scan, emit: blocks in ascending order, each in
//                         (x, y, z) lexicographic order, so the output is deterministic.
// Coordinate rules (sub-lattice and emission):
//   Cube    fl(fl(i * fl32(voxel)) - 1), no contraction: bit-identical to grid.lattice_points;
//   Table   ax[a][i] from three device fp32 tables [N]: the torch.linspace tables of grid.axis_tables, which the dense
//           threshold sweep (extract_geometry) evaluates, so the points are that sweep's bit for bit.
// Spacing rules (block test):
//   Cube    r = 0.5 sqrt(ex^2 + ey^2 + ez^2) voxel (e: the box's index extents), enlarged by 1e-6 relative plus 1e-6
//           absolute (the fp32 lattice coordinates are within 6e-8 of i voxel - 1 per axis); tau enlarged by 1e-6 relative
//           (the dense udf band compares fp32 values with an fp32 threshold); edge slope |du| / (e_a voxel);
//   Table   r = 0.5 sqrt(dx^2 + dy^2 + dz^2), d_a = |ax[a][hi] - ax[a][lo]| in fp64 (the box's own table coordinates),
//           enlarged by 1e-6 relative plus the caller's `pad` (the distance by which rounding in the tables may put a
//           lattice point outside its block's corner box: grid.iso_band measures it on the tables); tau is the caller's,
//           slack included (grid.iso_band: level + L D plus 1e-6 (|level| + L D)); edge slope |du| / (e_a h_a), h_a the
//           largest step of table a, a lower bound on the slope since the edge is at most e_a h_a long.
//
// Why the table rule meshes a threshold lattice exactly (grid.iso_band, mesh.iso_mesh_band): let every step of table a be
// at most h_a, D = sqrt(h_x^2 + h_y^2 + h_z^2) (two corners of one lattice cell are at most D apart) and tau > level + L D.
// If the field is L-Lipschitz at the lattice points and the query gives a point the same bits in any batch, every point
// with a value below tau is evaluated with the dense sweep's bits, and every point left out (+inf) has a dense value
// >= tau > level + L D.  A cell the dense lattice makes active has a corner at or below the level, so all its corners are
// below tau and evaluated.  A cell with a culled corner has, for the same reason, every dense corner value above the level,
// so it is inactive in both lattices.  The threshold marching cubes (nudf_iso_*) reads df only at the corners of active
// cells, so it gives the same active cells, faces, vertex keys and fp64 vertices on both.
#include <type_traits>

#include "../../include/nudf.h"
#include "common.cuh"
#include "df_access.cuh"

namespace nudf {
namespace nb {

struct Lat {
  int64_t N;     // lattice points per axis
  int64_t s;     // block stride
  int64_t nb;    // blocks per axis
  __device__ __forceinline__ int64_t lo(int64_t b) const { return b * s; }
  __device__ __forceinline__ int64_t hi(int64_t b) const { return min(b * s + s, N - 1); }
};

__device__ __forceinline__ float coord(int64_t i, float vf) { return __fsub_rn(__fmul_rn((float)i, vf), 1.0f); }

struct CubeCoord {
  float vf;  // fl32(voxel)
  __device__ __forceinline__ float operator()(int a, int64_t i) const { return coord(i, vf); }
};

struct TableCoord {
  const float* ax[3];
  __device__ __forceinline__ float operator()(int a, int64_t i) const { return ax[a][i]; }
};

template <class C>
__device__ __forceinline__ void write_point(int64_t x, int64_t y, int64_t z, int64_t N, const C& cr, int64_t* idx, float* pts,
                                            int64_t o) {
  idx[o] = (x * N + y) * N + z;
  pts[3 * o] = cr(0, x);
  pts[3 * o + 1] = cr(1, y);
  pts[3 * o + 2] = cr(2, z);
}

template <class C>
__global__ void k_sublattice(int64_t N, int64_t s, int64_t m, C cr, int64_t* __restrict__ idx, float* __restrict__ pts) {
  const int64_t n = m * m * m;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t a = t / (m * m), b = (t / m) % m, c = t % m;
    write_point(min(a * s, N - 1), min(b * s, N - 1), min(c * s, N - 1), N, cr, idx, pts, t);
  }
}

struct CubeSpacing {
  double voxel;
  __device__ __forceinline__ double thr(double tau) const { return __dmul_rn(tau, 1.000001); }
  // r with slack, for the box [x0, x0 + ex] x [y0, y0 + ey] x [z0, z0 + ez]
  __device__ __forceinline__ double radius(int64_t, int64_t, int64_t, int64_t ex, int64_t ey, int64_t ez) const {
    const double r = __dmul_rn(__dmul_rn(0.5, __dsqrt_rn((double)(ex * ex + ey * ey + ez * ez))), voxel);
    return __dadd_rn(__dmul_rn(r, 1.000001), 1e-6);
  }
  __device__ __forceinline__ double edge(int, int64_t e) const { return (double)e * voxel; }
};

struct TableSpacing {
  const float* ax[3];
  double h[3];   // the largest step of each table
  double pad;    // added to r: the tables' excursion outside a block's corner box
  __device__ __forceinline__ double thr(double tau) const { return tau; }
  __device__ __forceinline__ double extent(int a, int64_t lo, int64_t e) const {
    return fabs(__dsub_rn((double)ax[a][lo + e], (double)ax[a][lo]));
  }
  __device__ __forceinline__ double radius(int64_t x0, int64_t y0, int64_t z0, int64_t ex, int64_t ey, int64_t ez) const {
    const double dx = extent(0, x0, ex), dy = extent(1, y0, ey), dz = extent(2, z0, ez);
    const double q = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
    return __dadd_rn(__dmul_rn(__dmul_rn(0.5, __dsqrt_rn(q)), 1.000001), pad);
  }
  __device__ __forceinline__ double edge(int a, int64_t e) const { return __dmul_rn((double)e, h[a]); }
};

// A: the lattice reader (df_access.cuh): DenseDf for grid.udf_band / iso_band, BrickDf for grid.udf_band_sparse /
// iso_band_sparse
template <class A, class S>
__global__ void k_block_test(A df, Lat B, const uint8_t* __restrict__ parent, int64_t ps, int64_t pnb,
                             S sp, double lip, double tau, uint8_t* __restrict__ flags, unsigned* __restrict__ max_slope) {
  const int64_t n = B.nb * B.nb * B.nb, N = B.N;
  const double thr = sp.thr(tau);
  for (int64_t base = blockIdx.x * (int64_t)blockDim.x; base < n; base += (int64_t)gridDim.x * blockDim.x) {
    const int64_t t = base + threadIdx.x;
    float slope = 0.f;                               // the warp reduces its maximum below: every lane reaches it
    if (t < n) {
      const int64_t bx = t / (B.nb * B.nb), by = (t / B.nb) % B.nb, bz = t % B.nb;
      bool cand = true;
      if (parent) cand = parent[((B.lo(bx) / ps) * pnb + B.lo(by) / ps) * pnb + B.lo(bz) / ps] != 0;
      uint8_t keep = 0;
      if (cand) {
        const int64_t x0 = B.lo(bx), y0 = B.lo(by), z0 = B.lo(bz);
        const int64_t ex = B.hi(bx) - x0, ey = B.hi(by) - y0, ez = B.hi(bz) - z0;
        float u[8];
#pragma unroll
        for (int c = 0; c < 8; ++c)
          u[c] = df(((x0 + ((c >> 2) & 1) * ex) * N + (y0 + ((c >> 1) & 1) * ey)) * N + z0 + (c & 1) * ez);
        bool nan = false;
        double mn = u[0];
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          nan |= u[c] != u[c];
          mn = fmin(mn, (double)u[c]);
        }
        const double rr = sp.radius(x0, y0, z0, ex, ey, ez);
        const double bound = __dsub_rn(mn, __dmul_rn(lip, rr));
        keep = (nan || !(bound >= thr)) ? 1 : 0;
        // the 12 box edges: |du| / (edge length, or its upper bound) between finite corners
        const int64_t e[3] = {ex, ey, ez};
#pragma unroll
        for (int c = 0; c < 8; ++c)
#pragma unroll
          for (int ax = 0; ax < 3; ++ax) {
            const int bit = 4 >> ax;
            if (c & bit) continue;
            const float a = u[c], b = u[c | bit];
            if (isfinite(a) && isfinite(b))
              slope = fmaxf(slope, (float)(fabs((double)b - (double)a) / sp.edge(ax, e[ax])));
          }
      }
      if (flags) flags[t] = keep;
    }
    // non-negative floats order like their bit patterns: one atomic per warp
    const unsigned w = __reduce_max_sync(0xffffffffu, __float_as_uint(slope));
    if ((threadIdx.x & 31) == 0 && w) atomicMax(max_slope, w);
  }
}

// visits the points of stride-t lattice that block (bx, by, bz) of stride s emits, in emission order
template <class F>
__device__ __forceinline__ void block_points(const uint8_t* __restrict__ flags, const Lat& B, int64_t t, int64_t blk, F&& f) {
  const int64_t b[3] = {blk / (B.nb * B.nb), (blk / B.nb) % B.nb, blk % B.nb};
  int64_t lo[3], hi[3], m[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    lo[a] = B.lo(b[a]);
    hi[a] = B.hi(b[a]);
    m[a] = (hi[a] - lo[a] + t - 1) / t + 1;
  }
  for (int64_t jx = 0; jx < m[0]; ++jx)
    for (int64_t jy = 0; jy < m[1]; ++jy)
      for (int64_t jz = 0; jz < m[2]; ++jz) {
        const int64_t j[3] = {jx, jy, jz};
        int cls[3];                                    // -1: on the box's lower face, +1: upper face, 0: inside
        bool corner = true;
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          cls[a] = j[a] == 0 ? -1 : (j[a] == m[a] - 1 ? 1 : 0);
          corner &= cls[a] != 0;
        }
        if (corner) continue;                          // on the stride-s lattice: evaluated already
        bool owned = true;
        for (int d = 1; d < 27 && owned; ++d) {        // the other blocks holding the point: offsets along face axes
          const int dd[3] = {d / 9 - 1, (d / 3) % 3 - 1, d % 3 - 1};
          if (dd[0] == 0 && dd[1] == 0 && dd[2] == 0) continue;
          bool ok = true;
          int64_t q[3];
#pragma unroll
          for (int a = 0; a < 3; ++a) {
            ok &= dd[a] == 0 || dd[a] == cls[a];
            q[a] = b[a] + dd[a];
            ok &= q[a] >= 0 && q[a] < B.nb;
          }
          if (!ok) continue;
          const int64_t qb = (q[0] * B.nb + q[1]) * B.nb + q[2];
          if (qb < blk && flags[qb]) owned = false;
        }
        if (owned) f(min(lo[0] + jx * t, hi[0]), min(lo[1] + jy * t, hi[1]), min(lo[2] + jz * t, hi[2]));
      }
}

__global__ void k_count(const uint8_t* __restrict__ flags, Lat B, int64_t t, const int64_t* __restrict__ kept, int64_t n,
                        int32_t* __restrict__ counts) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int32_t c = 0;
    block_points(flags, B, t, kept[i], [&](int64_t, int64_t, int64_t) { ++c; });
    counts[i] = c;
  }
}

template <class C>
__global__ void k_emit(const uint8_t* __restrict__ flags, Lat B, int64_t t, const int64_t* __restrict__ kept, int64_t n,
                       const int64_t* __restrict__ offsets, C cr, int64_t* __restrict__ idx, float* __restrict__ pts) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t o = offsets[i];
    block_points(flags, B, t, kept[i], [&](int64_t x, int64_t y, int64_t z) { write_point(x, y, z, B.N, cr, idx, pts, o++); });
  }
}

}  // namespace nb
}  // namespace nudf

using namespace nudf;
using namespace nudf::nb;

static inline bool is_table(const nudf_band_coords& co) { return co.ax[0] || co.ax[1] || co.ax[2]; }

static int check_coords(const nudf_band_coords* co) {
  NUDF_REQUIRE(co && (!is_table(*co) || (co->ax[0] && co->ax[1] && co->ax[2])), "null pointer");
  NUDF_REQUIRE(!is_table(*co) || (co->h[0] >= 0.0 && co->h[1] >= 0.0 && co->h[2] >= 0.0 && co->pad >= 0.0),
               "negative spacing or pad");
  return 0;
}

// Checks the descriptor, then returns launch(TableCoord) or launch(CubeCoord) (-1: invalid).
template <class F>
static int with_coords(const nudf_band_coords* co, F&& launch) {
  if (check_coords(co)) return -1;
  if (is_table(*co)) return launch(TableCoord{{co->ax[0], co->ax[1], co->ax[2]}});
  return launch(CubeCoord{(float)co->voxel});
}

int nudf_nb_sublattice(int32_t n, int32_t s, const nudf_band_coords* co, int64_t* idx, float* pts, void* stream) {
  return with_coords(co, [&](auto cr) {
    NUDF_REQUIRE(idx && pts, "null pointer");
    NUDF_REQUIRE(n >= 2 && s >= 1, "need N >= 2 and stride >= 1");
    const int64_t m = cdiv(n - 1, s) + 1;
    k_sublattice<<<grid_for(m * m * m), 256, 0, (cudaStream_t)stream>>>(n, s, m, cr, idx, pts);
    NUDF_LAUNCH_OK();
    return 0;
  });
}

// every reader with either spacing rule: the table rule on a brick store keeps the blocks it keeps on the dense band
int nudf_nb_block_test(const nudf_lattice* lat, int32_t s, const uint8_t* parent_flags, int32_t parent_s,
                       const nudf_band_coords* co, double lipschitz, double tau, uint8_t* flags, uint32_t* max_slope,
                       void* stream) {
  if (check_coords(co)) return -1;
  return with_lattice(lat, [&](auto df) {
    NUDF_REQUIRE(max_slope, "null pointer");
    NUDF_REQUIRE(lat->n0 == lat->n1 && lat->n1 == lat->n2, "the band lattice must be cubic");
    NUDF_REQUIRE(s >= 1, "need stride >= 1");
    NUDF_REQUIRE(!parent_flags || (parent_s > s && parent_s % s == 0), "the parent stride must be a multiple of the stride");
    NUDF_REQUIRE(lipschitz >= 0.0, "negative Lipschitz constant");
    const int32_t n = lat->n0;
    const Lat B{n, s, cdiv(n - 1, s)};
    const int64_t pnb = parent_flags ? cdiv(n - 1, parent_s) : 0;
    auto launch = [&](auto sp) {
      k_block_test<<<grid_for(B.nb * B.nb * B.nb), 256, 0, (cudaStream_t)stream>>>(df, B, parent_flags, parent_s, pnb, sp,
                                                                                   lipschitz, tau, flags, max_slope);
      NUDF_LAUNCH_OK();
      return 0;
    };
    if (is_table(*co)) return launch(TableSpacing{{co->ax[0], co->ax[1], co->ax[2]}, {co->h[0], co->h[1], co->h[2]}, co->pad});
    return launch(CubeSpacing{co->voxel});
  });
}

int nudf_nb_count(const uint8_t* flags, int32_t n, int32_t s, int32_t t, const int64_t* kept, int64_t n_kept,
                  int32_t* counts, void* stream) {
  NUDF_REQUIRE(flags && (n_kept == 0 || (kept && counts)), "null pointer");
  NUDF_REQUIRE(n >= 2 && t >= 1 && s > t && s % t == 0, "the stride must be a multiple of the next stride");
  if (n_kept == 0) return 0;
  k_count<<<grid_for(n_kept), 256, 0, (cudaStream_t)stream>>>(flags, Lat{n, s, cdiv(n - 1, s)}, t, kept, n_kept, counts);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_nb_emit(const uint8_t* flags, int32_t n, int32_t s, int32_t t, const int64_t* kept, int64_t n_kept,
                 const int64_t* offsets, const nudf_band_coords* co, int64_t* idx, float* pts, void* stream) {
  return with_coords(co, [&](auto cr) {
    NUDF_REQUIRE(flags && (n_kept == 0 || (kept && offsets && idx && pts)), "null pointer");
    NUDF_REQUIRE(n >= 2 && t >= 1 && s > t && s % t == 0, "the stride must be a multiple of the next stride");
    if (n_kept == 0) return 0;
    k_emit<<<grid_for(n_kept), 256, 0, (cudaStream_t)stream>>>(flags, Lat{n, s, cdiv(n - 1, s)}, t, kept, n_kept, offsets, cr,
                                                              idx, pts);
    NUDF_LAUNCH_OK();
    return 0;
  });
}

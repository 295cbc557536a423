// Mesh post-processing after the MC's vertex filter (extract_mesh.py:215-265), the stages of neuraludf_b200/mesh_post.py.
// tests/proto/mesh_post.py restates every kernel in NumPy with the same fp64 operation order; sorting, unique and
// compaction run in torch between the launches.
//   face pass       remap a face through the vertex merge, test it for degeneracy, emit its sorted vertex triple and its
//                   three edge codes ((lo * V + hi) * 2 + (1 when the face runs hi -> lo)).  Degenerate: a = v1 - v0,
//                   b = v2 - v0, c = a x b; kept when |a|, |b|, |c| / |a| and |c| / |b| all exceed 1e-8, with
//                   |x| = sqrt((x0 x0 + x1 x1) + x2 x2).
//   holes           one thread per boundary edge (u, v), u < v, over the CSR of boundary neighbours (ascending): walk from v
//                   away from u through vertices of boundary degree 2; a return to u after 3 or 4 vertices is a hole, owned
//                   by its smallest edge key.  The owner emits one face (triangle) or two (quad, split along the shorter
//                   diagonal by squared length, a tie to the diagonal through the smallest vertex), traversing the owner
//                   edge against its direction in its face.  Count, scan, emit: the output follows the boundary edge order.
//   smoothing       one Jacobi step over the border vertices: v + lambda (sum of neighbours / count - v), neighbours summed
//                   in ascending index order; everything read from the previous step's buffer.
// Every fp64 operation is an explicit __d*_rn: no contraction, so the device and NumPy give the same bits.
#include "../../include/nudf.h"
#include "common.cuh"

namespace nudf {
namespace mp {

__device__ __forceinline__ double norm3(double x, double y, double z) {
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
}

__global__ void k_faces(const double* __restrict__ verts, int64_t nv, const int64_t* __restrict__ faces, int64_t nf,
                        const int64_t* __restrict__ remap, int64_t* __restrict__ out, int64_t* __restrict__ sorted,
                        int64_t* __restrict__ codes, uint8_t* __restrict__ nondeg) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nf; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t g[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      g[k] = faces[3 * i + k];
      if (remap) g[k] = remap[g[k]];
      out[3 * i + k] = g[k];
    }
    const int64_t lo = min(g[0], min(g[1], g[2])), hi = max(g[0], max(g[1], g[2]));
    sorted[3 * i] = lo;
    sorted[3 * i + 1] = g[0] + g[1] + g[2] - lo - hi;
    sorted[3 * i + 2] = hi;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int64_t a = g[k], b = g[(k + 1) % 3];
      codes[3 * i + k] = (min(a, b) * nv + max(a, b)) * 2 + (a > b ? 1 : 0);
    }
    double p[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k)
#pragma unroll
      for (int d = 0; d < 3; ++d) p[k][d] = verts[3 * g[k] + d];
    double a[3], b[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      a[d] = __dsub_rn(p[1][d], p[0][d]);
      b[d] = __dsub_rn(p[2][d], p[0][d]);
    }
    const double cx = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
    const double cy = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
    const double cz = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
    const double la = norm3(a[0], a[1], a[2]), lb = norm3(b[0], b[1], b[2]), lc = norm3(cx, cy, cz);
    const double t = 1e-8;
    nondeg[i] = (la > t && lb > t && __ddiv_rn(lc, la) > t && __ddiv_rn(lc, lb) > t) ? 1 : 0;
  }
}

__device__ __forceinline__ int64_t ekey(int64_t a, int64_t b, int64_t nv) { return min(a, b) * nv + max(a, b); }

// the hole owned by boundary edge (u, v): its vertex count (3 or 4; 0: none) and the cycle u, v, ... in walk order
__device__ __forceinline__ int walk(int64_t u, int64_t v, const int64_t* __restrict__ rowptr, const int64_t* __restrict__ cols,
                                    int64_t nv, int64_t* cyc) {
  auto deg = [&](int64_t x) { return rowptr[x + 1] - rowptr[x]; };
  if (deg(u) != 2 || deg(v) != 2) return 0;
  cyc[0] = u;
  cyc[1] = v;
  int64_t prev = u, cur = v;
  int len = 0;
  for (int step = 0; step < 3 && !len; ++step) {
    const int64_t n0 = cols[rowptr[cur]], n1 = cols[rowptr[cur] + 1];
    const int64_t nxt = n0 == prev ? n1 : n0;
    if (nxt == u) {
      if (step >= 1) len = step + 2;
      break;
    }
    if (step == 2 || deg(nxt) != 2) return 0;
    cyc[step + 2] = nxt;
    prev = cur;
    cur = nxt;
  }
  if (!len) return 0;
  const int64_t k0 = ekey(u, v, nv);
  for (int j = 1; j < len; ++j)
    if (ekey(cyc[j], cyc[(j + 1) % len], nv) <= k0) return 0;
  return len;
}

__global__ void k_hole_count(const int64_t* __restrict__ edges, int64_t ne, const int64_t* __restrict__ rowptr,
                             const int64_t* __restrict__ cols, int64_t nv, int32_t* __restrict__ counts) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < ne; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t cyc[4];
    const int len = walk(edges[2 * i], edges[2 * i + 1], rowptr, cols, nv, cyc);
    counts[i] = len == 3 ? 1 : (len == 4 ? 2 : 0);
  }
}

__device__ __forceinline__ double sqdist(const double* __restrict__ verts, int64_t a, int64_t b) {
  const double dx = __dsub_rn(verts[3 * a], verts[3 * b]), dy = __dsub_rn(verts[3 * a + 1], verts[3 * b + 1]);
  const double dz = __dsub_rn(verts[3 * a + 2], verts[3 * b + 2]);
  return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

__global__ void k_hole_emit(const double* __restrict__ verts, const int64_t* __restrict__ edges, const uint8_t* __restrict__ dirs,
                            int64_t ne, const int64_t* __restrict__ rowptr, const int64_t* __restrict__ cols, int64_t nv,
                            const int64_t* __restrict__ offsets, int64_t* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < ne; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t w[4];
    const int len = walk(edges[2 * i], edges[2 * i + 1], rowptr, cols, nv, w);
    if (!len) continue;
    int64_t c[4];                                  // oriented: against the owner edge's direction in its face
    c[0] = w[0];
    for (int j = 1; j < len; ++j) c[j] = dirs[i] ? w[j] : w[len - j];
    int64_t* o = out + 3 * offsets[i];
    if (len == 3) {
      o[0] = c[0], o[1] = c[1], o[2] = c[2];
      continue;
    }
    const double d02 = sqdist(verts, c[0], c[2]), d13 = sqdist(verts, c[1], c[3]);
    const int r = (d13 < d02 || (d13 == d02 && min(c[1], c[3]) < min(c[0], c[2]))) ? 1 : 0;
    const int64_t d0 = c[r], d1 = c[r + 1], d2 = c[r + 2], d3 = c[(r + 3) & 3];
    o[0] = d0, o[1] = d1, o[2] = d2;
    o[3] = d0, o[4] = d2, o[5] = d3;
  }
}

__global__ void k_smooth(const double* __restrict__ vin, double* __restrict__ vout, const int64_t* __restrict__ border,
                         int64_t nb, const int64_t* __restrict__ rowptr, const int64_t* __restrict__ cols, double lambda) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nb; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = border[i], r0 = rowptr[b], r1 = rowptr[b + 1];
    double s[3] = {0.0, 0.0, 0.0};
    for (int64_t r = r0; r < r1; ++r) {
      const int64_t n = cols[r];
#pragma unroll
      for (int d = 0; d < 3; ++d) s[d] = __dadd_rn(s[d], vin[3 * n + d]);
    }
    const double cnt = (double)(r1 - r0);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const double v = vin[3 * b + d];
      vout[3 * b + d] = __dadd_rn(v, __dmul_rn(lambda, __dsub_rn(__ddiv_rn(s[d], cnt), v)));
    }
  }
}

}  // namespace mp
}  // namespace nudf

using namespace nudf;
using namespace nudf::mp;

int nudf_mp_faces(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, const int64_t* remap,
                  int64_t* out_faces, int64_t* sorted_faces, int64_t* edge_codes, uint8_t* nondegenerate, void* stream) {
  NUDF_REQUIRE(n_faces >= 0 && n_verts >= 0, "negative size");
  if (n_faces == 0) return 0;
  NUDF_REQUIRE(verts && faces && out_faces && sorted_faces && edge_codes && nondegenerate, "null pointer");
  NUDF_REQUIRE(n_verts < (int64_t(1) << 30), "edge codes need fewer than 2^30 vertices");
  k_faces<<<grid_for(n_faces), 256, 0, (cudaStream_t)stream>>>(verts, n_verts, faces, n_faces, remap, out_faces, sorted_faces,
                                                              edge_codes, nondegenerate);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_mp_hole_count(const int64_t* edges, int64_t n_edges, const int64_t* rowptr, const int64_t* cols, int64_t n_verts,
                       int32_t* counts, void* stream) {
  NUDF_REQUIRE(n_edges >= 0, "negative size");
  if (n_edges == 0) return 0;
  NUDF_REQUIRE(edges && rowptr && cols && counts, "null pointer");
  k_hole_count<<<grid_for(n_edges), 256, 0, (cudaStream_t)stream>>>(edges, n_edges, rowptr, cols, n_verts, counts);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_mp_hole_emit(const double* verts, const int64_t* edges, const uint8_t* dirs, int64_t n_edges, const int64_t* rowptr,
                      const int64_t* cols, int64_t n_verts, const int64_t* offsets, int64_t* faces, void* stream) {
  NUDF_REQUIRE(n_edges >= 0, "negative size");
  if (n_edges == 0) return 0;
  NUDF_REQUIRE(verts && edges && dirs && rowptr && cols && offsets && faces, "null pointer");
  k_hole_emit<<<grid_for(n_edges), 256, 0, (cudaStream_t)stream>>>(verts, edges, dirs, n_edges, rowptr, cols, n_verts, offsets,
                                                                  faces);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_mp_smooth_step(const double* verts_in, double* verts_out, const int64_t* border, int64_t n_border,
                        const int64_t* rowptr, const int64_t* cols, double lambda, void* stream) {
  NUDF_REQUIRE(n_border >= 0, "negative size");
  if (n_border == 0) return 0;
  NUDF_REQUIRE(verts_in && verts_out && verts_in != verts_out && border && rowptr && cols, "null pointer or in-place step");
  k_smooth<<<grid_for(n_border), 256, 0, (cudaStream_t)stream>>>(verts_in, verts_out, border, n_border, rowptr, cols, lambda);
  NUDF_LAUNCH_OK();
  return 0;
}

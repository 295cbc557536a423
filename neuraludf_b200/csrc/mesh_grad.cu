// The gradient branch of get_mesh_udf_fast (extract_mesh.py:267-304), the stages of neuraludf_b200/extract_mesh.py.
// tests/proto/mesh_grad.py restates every kernel in NumPy with the same operation order.
//   vertex normals  face pass: the fp64 unit normal n = c / max(|c|, 1e-300), c = (v1 - v0) x (v2 - v0), and the angle at
//                   each corner k, acos(clip(u.w / max(|u| |w|, 1e-300), -1, 1)) with u, w the edges from corner k to
//                   corners k + 1 and k + 2; it writes n * angle_k per corner.  Vertex pass: each vertex sums the terms of
//                   its incidences in ascending (corner, face) order (a CSR sorted in torch), divides by max(|sum|, 1e-300)
//                   and rounds once to fp32.  |x| = sqrt((x0 x0 + x1 x1) + x2 x2), x.y = (x0 y0 + x1 y1) + x2 y2.
//   refine          mode 1 (no probe values): the probe points v + fl(eps n) and v - fl(eps n).  Mode 2: new_verts =
//                   (v - (eps s1) n) + (eps s2) n, each product and sum rounded on its own, and the next indices
//                   trunc(fl(x + 1) / fl(voxel)) per axis with their six clamped neighbours, block-major.
// Every operation is an explicit __d*_rn / __f*_rn: no contraction, so the device and NumPy give the same bits (acos aside:
// CUDA's and the host libm's may differ in the last fp64 bit).
#include "../../include/nudf.h"
#include "common.cuh"

namespace nudf {
namespace mg {

__device__ __forceinline__ double dot3(const double* a, const double* b) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}

__global__ void k_face_terms(const double* __restrict__ verts, const int64_t* __restrict__ faces, int64_t nf,
                             double* __restrict__ terms) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nf; i += (int64_t)gridDim.x * blockDim.x) {
    double p[3][3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const int64_t g = faces[3 * i + k];
#pragma unroll
      for (int d = 0; d < 3; ++d) p[k][d] = verts[3 * g + d];
    }
    double a[3], b[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      a[d] = __dsub_rn(p[1][d], p[0][d]);
      b[d] = __dsub_rn(p[2][d], p[0][d]);
    }
    double n[3] = {__dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1])),
                   __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2])),
                   __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]))};
    const double ln = fmax(__dsqrt_rn(dot3(n, n)), 1e-300);
#pragma unroll
    for (int d = 0; d < 3; ++d) n[d] = __ddiv_rn(n[d], ln);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      double u[3], w[3];
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        u[d] = __dsub_rn(p[(k + 1) % 3][d], p[k][d]);
        w[d] = __dsub_rn(p[(k + 2) % 3][d], p[k][d]);
      }
      const double den = fmax(__dmul_rn(__dsqrt_rn(dot3(u, u)), __dsqrt_rn(dot3(w, w))), 1e-300);
      double c = __ddiv_rn(dot3(u, w), den);
      c = c < -1.0 ? -1.0 : (c > 1.0 ? 1.0 : c);               // np.clip: a NaN stays NaN
      const double ang = acos(c);
#pragma unroll
      for (int d = 0; d < 3; ++d) terms[9 * i + 3 * k + d] = __dmul_rn(n[d], ang);
    }
  }
}

__global__ void k_vertex_normals(const int64_t* __restrict__ rowptr, const int64_t* __restrict__ inc, int64_t nv, int64_t nf,
                                 const double* __restrict__ terms, float* __restrict__ normals) {
  for (int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; v < nv; v += (int64_t)gridDim.x * blockDim.x) {
    double s[3] = {0.0, 0.0, 0.0};
    for (int64_t r = rowptr[v]; r < rowptr[v + 1]; ++r) {
      const int64_t e = inc[r], c = e / nf, f = e - c * nf;
#pragma unroll
      for (int d = 0; d < 3; ++d) s[d] = __dadd_rn(s[d], terms[9 * f + 3 * c + d]);
    }
    const double l = fmax(__dsqrt_rn(dot3(s, s)), 1e-300);
#pragma unroll
    for (int d = 0; d < 3; ++d) normals[3 * v + d] = __double2float_rn(__ddiv_rn(s[d], l));
  }
}

__global__ void k_probes(const float* __restrict__ verts, const float* __restrict__ normals, int64_t nv, float eps,
                         float* __restrict__ probes) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < 3 * nv; t += (int64_t)gridDim.x * blockDim.x) {
    const float o = __fmul_rn(eps, normals[t]);
    probes[t] = __fadd_rn(verts[t], o);
    probes[3 * nv + t] = __fsub_rn(verts[t], o);
  }
}

// numpy's astype(int64) on x86: trunc toward zero, NaN and out-of-range values give INT64_MIN
__device__ __forceinline__ int64_t trunc_i64(float q) {
  return (q >= -9.2233720e18f && q < 9.2233720e18f) ? __float2ll_rz(q) : (int64_t)0x8000000000000000ull;
}

// i * n * n + j * n + k in int64 with numpy's wrap-around
__device__ __forceinline__ int64_t flat(int64_t i, int64_t j, int64_t k, int64_t n) {
  const uint64_t un = (uint64_t)n;
  return (int64_t)((uint64_t)i * un * un + (uint64_t)j * un + (uint64_t)k);
}

__global__ void k_refine(const float* __restrict__ verts, const float* __restrict__ normals, int64_t nv, float eps,
                         const float* __restrict__ s1, const float* __restrict__ s2, int64_t n_mc, float voxel,
                         float* __restrict__ new_verts, int64_t* __restrict__ next_indices) {
  for (int64_t v = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; v < nv; v += (int64_t)gridDim.x * blockDim.x) {
    const float e1 = __fmul_rn(eps, s1[v]), e2 = __fmul_rn(eps, s2[v]);
    int64_t q[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const float n = normals[3 * v + d];
      const float x = __fadd_rn(__fsub_rn(verts[3 * v + d], __fmul_rn(e1, n)), __fmul_rn(e2, n));
      new_verts[3 * v + d] = x;
      q[d] = trunc_i64(__fdiv_rn(__fsub_rn(x, -1.0f), voxel));
    }
    const int64_t i = q[0], j = q[1], k = q[2], hi = n_mc - 1;
    const int64_t im = (int64_t)((uint64_t)i - 1), jm = (int64_t)((uint64_t)j - 1), km = (int64_t)((uint64_t)k - 1);
    int64_t* o = next_indices + v;
    o[0] = flat(i, j, k, n_mc);
    o[nv] = flat(min(i + 1, hi), j, k, n_mc);
    o[2 * nv] = flat(i, min(j + 1, hi), k, n_mc);
    o[3 * nv] = flat(i, j, min(k + 1, hi), n_mc);
    o[4 * nv] = flat(max(im, (int64_t)0), j, k, n_mc);
    o[5 * nv] = flat(i, max(jm, (int64_t)0), k, n_mc);
    o[6 * nv] = flat(i, j, max(km, (int64_t)0), n_mc);
  }
}

}  // namespace mg
}  // namespace nudf

using namespace nudf;
using namespace nudf::mg;

int nudf_mg_vertex_normals(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, const int64_t* rowptr,
                           const int64_t* incidences, double* face_terms, float* normals, void* stream) {
  NUDF_REQUIRE(n_faces >= 0 && n_verts >= 0, "negative size");
  if (n_verts == 0) return 0;
  NUDF_REQUIRE(rowptr && normals, "null pointer");
  NUDF_REQUIRE(n_faces == 0 || (verts && faces && incidences && face_terms), "null pointer");
  if (n_faces > 0) {
    k_face_terms<<<grid_for(n_faces), 256, 0, (cudaStream_t)stream>>>(verts, faces, n_faces, face_terms);
    NUDF_LAUNCH_OK();
  }
  k_vertex_normals<<<grid_for(n_verts), 256, 0, (cudaStream_t)stream>>>(rowptr, incidences, n_verts, n_faces > 0 ? n_faces : 1,
                                                                       face_terms, normals);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_mg_refine(const float* verts, const float* normals, int64_t n_verts, float eps, const float* s1, const float* s2,
                   int32_t n_mc, float* probes, float* new_verts, int64_t* next_indices, void* stream) {
  NUDF_REQUIRE(n_verts >= 0, "negative size");
  NUDF_REQUIRE(n_mc >= 2, "the lattice needs at least 2 points per axis");
  if (n_verts == 0) return 0;
  NUDF_REQUIRE(verts && normals, "null pointer");
  NUDF_REQUIRE((s1 == nullptr) == (s2 == nullptr), "give both probe values or neither");
  if (!s1) {
    NUDF_REQUIRE(probes, "null pointer");
    k_probes<<<grid_for(3 * n_verts), 256, 0, (cudaStream_t)stream>>>(verts, normals, n_verts, eps, probes);
  } else {
    NUDF_REQUIRE(new_verts && next_indices, "null pointer");
    const float voxel = (float)(2.0 / (double)(n_mc - 1));
    k_refine<<<grid_for(n_verts), 256, 0, (cudaStream_t)stream>>>(verts, normals, n_verts, eps, s1, s2, n_mc, voxel, new_verts,
                                                                 next_indices);
  }
  NUDF_LAUNCH_OK();
  return 0;
}

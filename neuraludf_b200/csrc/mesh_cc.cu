// Face labelling by connected components (neuraludf_b200/clean.py face_components, keep_largest,
// remove_small_components).  The input is the mesh's edge keys lo * V + hi (nudf_mp_faces' edge codes >> 1), sorted in
// torch, with the face each key came from; tests/proto/mesh_cc.py restates the result with scipy's connected_components.
//   adjacency     trimesh's face_adjacency: a key that occurs exactly twice joins the faces of its two slots when they
//                 differ.  A key used once (boundary) or three or more times (non-manifold fan) joins nothing, and a
//                 degenerate face (a, a, b), whose two (a, b) slots are its own, pairs only with itself and is dropped.
//   labels        an asynchronous union-find over the faces in parent[] = label[]: one launch hooks every pair, one launch
//                 compresses every face to its root; no host read between them.
// Invariant: parent[x] <= x for every x, with equality exactly at the roots.  It holds at the start (parent[x] = x); a hook
// CASes a root hi from hi to a strictly smaller root lo, and path halving CASes parent[x] from p to parent[p] <= p, so
// every write moves a pointer to an ancestor and no write raises it.  A node that stops being a root never becomes one
// again (the only write to a root is the hook's CAS), so trees only merge.  A pair (a, b) returns once find(a) ==
// find(b) or once its own CAS hooked one root under the other; a failed CAS means the root it read was hooked by another
// thread meanwhile, and the pair retries from the new roots.  So when the hooking launch ends, the trees are exactly the
// components, whatever the interleaving, and by the invariant each root is the smallest face of its tree: the labels are
// deterministic and equal the smallest face index of each component.
#include "../../include/nudf.h"
#include "common.cuh"

namespace nudf {
namespace cc {

typedef unsigned long long u64;

__device__ __forceinline__ int64_t ld(const int64_t* p) { return *(const volatile int64_t*)p; }

// the root of x, halving the path on the way (each CAS moves parent[y] from p to the grandparent of y)
__device__ __forceinline__ int64_t find(int64_t* par, int64_t x) {
  for (;;) {
    const int64_t p = ld(par + x);
    if (p == x) return x;
    const int64_t g = ld(par + p);
    if (g == p) return p;
    atomicCAS((u64*)(par + x), (u64)p, (u64)g);
    x = g;
  }
}

__global__ void k_init(int64_t* __restrict__ par, uint8_t* __restrict__ paired, int64_t nf) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nf; i += (int64_t)gridDim.x * blockDim.x) {
    par[i] = i;
    paired[i] = 0;
  }
}

// one thread per sorted key slot e: the pair starts at e when keys[e] == keys[e + 1] and neither neighbour repeats it
__global__ void k_hook(const int64_t* __restrict__ keys, const int64_t* __restrict__ key_face, int64_t nk, int64_t* par,
                       uint8_t* __restrict__ paired) {
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e + 1 < nk; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = keys[e];
    if (keys[e + 1] != k || (e > 0 && keys[e - 1] == k) || (e + 2 < nk && keys[e + 2] == k)) continue;
    const int64_t a = key_face[e], b = key_face[e + 1];
    if (a == b) continue;
    paired[a] = 1;
    paired[b] = 1;
    for (;;) {
      const int64_t ra = find(par, a), rb = find(par, b);
      if (ra == rb) break;
      const int64_t hi = max(ra, rb), lo = min(ra, rb);
      if (atomicCAS((u64*)(par + hi), (u64)hi, (u64)lo) == (u64)hi) break;
    }
  }
}

// after the hooking launch the roots are fixed: every face stores its root (halving CASes of other threads on par[x] can
// only fail once x has stored its root, since they expect a non-root value)
__global__ void k_compress(int64_t* par, int64_t nf) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nf; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = find(par, i);
    *(volatile int64_t*)(par + i) = r;
  }
}

}  // namespace cc
}  // namespace nudf

using namespace nudf;
using namespace nudf::cc;

int nudf_cc_label(const int64_t* keys, const int64_t* key_face, int64_t n_keys, int64_t n_faces, int64_t* label,
                  uint8_t* paired, void* stream) {
  NUDF_REQUIRE(n_keys >= 0 && n_faces >= 0, "negative size");
  if (n_faces == 0) return 0;
  NUDF_REQUIRE(label && paired && (n_keys == 0 || (keys && key_face)), "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  k_init<<<grid_for(n_faces), 256, 0, st>>>(label, paired, n_faces);
  NUDF_LAUNCH_OK();
  if (n_keys > 1) {
    k_hook<<<grid_for(n_keys), 256, 0, st>>>(keys, key_face, n_keys, label, paired);
    NUDF_LAUNCH_OK();
    k_compress<<<grid_for(n_faces), 256, 0, st>>>(label, n_faces);
    NUDF_LAUNCH_OK();
  }
  return 0;
}

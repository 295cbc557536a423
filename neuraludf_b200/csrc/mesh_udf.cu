// MeshUDF marching cubes on the device: the consumer of grid.py's dense UDF lattice + sparse near-surface normals.
// The reference meshes with a single-threaded Cython port of Lewiner's tables plus a breadth-first sign propagation
// (custom_mc/_marching_cubes_lewiner_cy.pyx:1115-1773).  Here every stage is data-parallel and order-free:
//   1. active cells   mean of the 8 corner udf < 1.05 voxel and max <= 1.74 voxel (the reference's thresholds, .pyx:1157-1158),
//                     summed in the reference's corner order so that the same cells pass;
//   2. pseudo-signs   per cell, every corner against the cell's reference corner r (largest udf, ties -> lowest corner):
//                     opposite sides when the normals are anti-parallel, unless they point away from each other along
//                     the corner-to-corner direction (the reference's edge vote, .pyx:1776-1806, generalised to diagonals);
//   3. polarity       face-adjacent active cells agree or disagree on their shared corners -> union-find with parity by
//                     min-root hooking (64-bit atomicMin on (root << 1 | parity): the winner does not depend on timing);
//                     a component takes the polarity that makes its root cell's corner 0 positive;
//   4. triangulation  no lookup table: the crossing segments of the 6 faces (ambiguous faces by the asymptotic decider,
//                     which is invariant under a global sign flip) are chained into loops; each loop is triangulated with
//                     no chord lying in a cube face (loop_triangles), so every edge of a closed surface has two triangles;
//   5. welding        vertices are keyed by lattice edge (3 * corner + axis) and placed at t = u_a / (u_a + u_b); the few
//                     loops that need a centre vertex key it after all edges (3 * n_points + 4 * cell + loop).
// Deviation from Lewiner: interior ambiguities (case 13 tunnels) are not resolved -- each loop is fanned on its own.
// Reads of df: stage 1 reads the 8 corners of each candidate cell; every later stage reads only the corners of active cells
// (k_signs, k_links and cell_loops read cell g's own corners, edge_point an edge of an active cell).  So, for the same
// candidates and normals, a lattice whose values equal the dense ones wherever those are <= max_t and are > max_t elsewhere
// (+inf included: max <= max_t fails) meshes exactly like the dense one -- what grid.udf_band's narrow band relies on.
// tests/proto/udf_mc.py restates every stage in NumPy with the same float32 operation order.
// Every MeshUDF stage reads df through a lattice reader A (df_access.cuh): DenseDf, the flat array, or BrickDf, the
// block-sparse band of grid.udf_band_sparse, as the nudf_lattice given to nudf_mc_* names.  The reader only replaces the
// load: both compute the same values from the same corner values.
// Threshold meshing (nudf_iso_*) runs stages 4-5 on v = fl32(f - level) instead of the pseudo-signed udf (the corner rules
// UdfCorners / IsoCorners), with its own active-cell test and fp64 vertices; tests/proto/iso_mc.py restates it.
#include <type_traits>

#include "../../include/nudf.h"
#include "common.cuh"
#include "compact.cuh"
#include "df_access.cuh"

namespace nudf {
namespace mc {

__constant__ int8_t kFaces[6][4] = {{0, 1, 3, 2}, {4, 6, 7, 5}, {0, 4, 5, 1}, {2, 3, 7, 6}, {0, 2, 6, 4}, {1, 5, 7, 3}};
__constant__ int8_t kLewinerOrder[8] = {0, 1, 3, 2, 4, 5, 7, 6};

struct Dims {
  int64_t n0, n1, n2;
  __device__ __forceinline__ int64_t coff(int c) const { return ((c >> 2) & 1) * n1 * n2 + ((c >> 1) & 1) * n2 + (c & 1); }
  __device__ __forceinline__ int64_t stride(int ax) const { return ax == 0 ? n1 * n2 : (ax == 1 ? n2 : 1); }
  __device__ __forceinline__ bool is_cell(int64_t g) const {
    const int64_t i = g / (n1 * n2), j = (g / n2) % n1, k = g % n2;
    return i < n0 - 1 && j < n1 - 1 && k < n2 - 1;
  }
  __device__ __forceinline__ int64_t coord(int64_t g, int ax) const {
    return ax == 0 ? g / (n1 * n2) : (ax == 1 ? (g / n2) % n1 : g % n2);
  }
};

// local edge id 0..11 = 4 * axis + rank of the lower corner among the 4 edges of that axis
__device__ __forceinline__ int edge_of(int a, int b) {
  const int lo = min(a, b), d = a ^ b;
  if (d == 4) return lo;
  if (d == 2) return 4 + ((lo & 1) | ((lo >> 2) << 1));
  return 8 + (lo >> 1);
}
__device__ __forceinline__ int edge_lo(int e) {
  const int r = e & 3;
  return e < 4 ? r : (e < 8 ? ((r & 1) | ((r >> 1) << 2)) : (r << 1));
}

__device__ __forceinline__ float dot3(const float* a, const float* b) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a[0], b[0]), __fmul_rn(a[1], b[1])), __fmul_rn(a[2], b[2]));
}

__device__ __forceinline__ int64_t find_sorted(const int64_t* __restrict__ a, int64_t n, int64_t key) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return (lo < n && a[lo] == key) ? lo : -1;
}

template <class A>
__global__ void k_active(A df, Dims D, const int64_t* __restrict__ cand, int64_t n, float avg_t,
                         float max_t, uint8_t* __restrict__ flag) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t g = cand ? cand[t] : t;
    uint8_t on = 0;
    if (D.is_cell(g)) {
      float s = df(g + D.coff(kLewinerOrder[0])), mx = s;
#pragma unroll
      for (int q = 1; q < 8; ++q) {
        const float v = df(g + D.coff(kLewinerOrder[q]));
        s = __fadd_rn(s, v);
        mx = fmaxf(mx, v);
      }
      on = (__fmul_rn(s, 0.125f) < avg_t) && (mx <= max_t);
    }
    flag[t] = on;
  }
}

template <class A>
__global__ void k_signs(A df, Dims D, const int64_t* __restrict__ cells, int64_t n,
                        const int64_t* __restrict__ idx, int64_t n_idx, const float* __restrict__ nrm,
                        uint8_t* __restrict__ mask) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t g = cells[t];
    float u[8], gv[8][3];
    int r = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const int64_t p = g + D.coff(c);
      u[c] = df(p);
      const int64_t row = idx ? find_sorted(idx, n_idx, p) : p;
#pragma unroll
      for (int k = 0; k < 3; ++k) gv[c][k] = row >= 0 ? nrm[row * 3 + k] : 0.f;
      if (u[c] > u[r]) r = c;
    }
    uint8_t m = 0;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      if (c == r) continue;
      const float d[3] = {(float)(((c >> 2) & 1) - ((r >> 2) & 1)), (float)(((c >> 1) & 1) - ((r >> 1) & 1)),
                          (float)((c & 1) - (r & 1))};
      const float pr = dot3(gv[r], d), pc = dot3(gv[c], d), dd = dot3(gv[r], gv[c]);
      const bool same = (pr < 0.f && pc > 0.f) || dd >= 0.f;
      if (!same) m |= (uint8_t)(1u << c);
    }
    mask[t] = m;
  }
}

template <class A>
__global__ void k_links(A df, Dims D, const int64_t* __restrict__ cells, int64_t n,
                        const uint8_t* __restrict__ mask, int64_t* __restrict__ links) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t g = cells[t];
    const int m = mask[t];
    for (int ax = 0; ax < 3; ++ax) {
      int64_t out = -1;
      const int64_t lim = ax == 0 ? D.n0 : (ax == 1 ? D.n1 : D.n2);
      const int64_t pos = D.coord(g, ax) + 1 < lim - 1 ? find_sorted(cells, n, g + D.stride(ax)) : -1;
      if (pos >= 0) {
        const int bit = 4 >> ax, mn = mask[pos];
        int agree = 0, disagree = 0;
        for (int c = 0; c < 8; ++c) {
          if (!(c & bit) || !(df(g + D.coff(c)) > 0.f)) continue;
          if (((m >> c) & 1) == ((mn >> (c ^ bit)) & 1)) ++agree; else ++disagree;
        }
        if ((agree == 0) != (disagree == 0)) out = 2 * pos + (disagree ? 1 : 0);
      }
      links[t * 3 + ax] = out;
    }
  }
}

// union-find with parity: parent[i] = (parent << 1) | (parity of i relative to parent)
__global__ void k_uf_init(int64_t* __restrict__ par, unsigned long long* __restrict__ hook, int64_t n) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    par[t] = t << 1;
    hook[t] = ~0ull;
  }
}

// pointer jumping; in place is safe: every value ever stored is a valid (ancestor, parity) pair of the same tree, and the
// converged state (root, parity along the unique tree path) does not depend on the interleaving
__global__ void k_uf_jump(int64_t* par, int64_t n, int32_t* changed) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = par[t], p = e >> 1;
    if (p == t) continue;
    const int64_t ep = *((volatile int64_t*)&par[p]), pp = ep >> 1;
    if (pp == p) continue;
    par[t] = (pp << 1) | ((e ^ ep) & 1);
    *changed = 1;
  }
}

__global__ void k_uf_hook(const int64_t* __restrict__ links, int64_t n, const int64_t* __restrict__ par,
                          unsigned long long* __restrict__ hook) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < 3 * n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t l = links[t];
    if (l < 0) continue;
    const int64_t ei = par[t / 3], ej = par[l >> 1];
    const int64_t ri = ei >> 1, rj = ej >> 1, pc = (ei ^ ej ^ l) & 1;
    if (rj < ri) atomicMin(&hook[ri], (unsigned long long)((rj << 1) | pc));
    else if (ri < rj) atomicMin(&hook[rj], (unsigned long long)((ri << 1) | pc));
  }
}

__global__ void k_uf_apply(unsigned long long* __restrict__ hook, int64_t* __restrict__ par, int64_t n, int32_t* changed) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const unsigned long long h = hook[t];
    if (h == ~0ull) continue;
    par[t] = (int64_t)h;
    hook[t] = ~0ull;
    *changed = 1;
  }
}

__global__ void k_uf_final(const int64_t* __restrict__ par, const uint8_t* __restrict__ mask_in, int64_t n,
                           uint8_t* __restrict__ mask_out) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t e = par[t];
    const int flip = (int)((e ^ mask_in[e >> 1]) & 1);
    mask_out[t] = flip ? (uint8_t)~mask_in[t] : mask_in[t];
  }
}

// Corner-value rules of the shared triangulation (cell_loops, loop_triangles): rule(D, t, g, v) writes the values v[8] of
// cell g = cells[t]; corner c is positive when v[c] > 0.  Faces are wound towards v > 0, or with kDescent towards v <= 0.
template <class A>
struct UdfCorners {             // MeshUDF: the udf with the cell's pseudo-sign
  A df;
  const uint8_t* __restrict__ mask;
  static constexpr bool kDescent = false;
  __device__ __forceinline__ void operator()(const Dims& D, int64_t t, int64_t g, float v[8]) const {
    const int m = mask[t];
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const float u = df(g + D.coff(c));
      v[c] = ((m >> c) & 1) ? -u : u;
    }
  }
};

template <class A>
struct IsoCorners {             // threshold meshing: v = fl32(f - level), faces wound from the > level side into the <= level side
  A df;
  float level;
  static constexpr bool kDescent = true;
  __device__ __forceinline__ void operator()(const Dims& D, int64_t, int64_t g, float v[8]) const {
#pragma unroll
    for (int c = 0; c < 8; ++c) v[c] = __fsub_rn(df(g + D.coff(c)), level);
  }
};

// the crossing loops of one cell with corner values v: local edge ids concatenated in loop[], lengths in len[]; returns the
// loop count (<= 4)
__device__ int cell_loops(const float v[8], int8_t loop[12], int8_t len[4]) {
  int p = 0;
#pragma unroll
  for (int c = 0; c < 8; ++c)
    if (v[c] > 0.f) p |= 1 << c;
  if (p == 0 || p == 0xFF) return 0;
  int8_t nxt[12];
#pragma unroll
  for (int e = 0; e < 12; ++e) nxt[e] = -1;
  for (int f = 0; f < 6; ++f) {
    int q[4], e[4], pq[4], ncross = 0;
    for (int s = 0; s < 4; ++s) { q[s] = kFaces[f][s]; pq[s] = (p >> q[s]) & 1; }
    for (int s = 0; s < 4; ++s) { e[s] = edge_of(q[s], q[(s + 1) & 3]); ncross += pq[s] != pq[(s + 1) & 3]; }
    if (ncross == 2) {
      int a = 0, b = 0;
      for (int s = 0; s < 4; ++s) {
        if (!pq[s] && pq[(s + 1) & 3]) a = e[s];
        if (pq[s] && !pq[(s + 1) & 3]) b = e[s];
      }
      nxt[a] = (int8_t)b;
    } else if (ncross == 4) {
      // asymptotic decider: sign of the bilinear saddle (ac - bd) / (a + c - b - d); exact ties join q0-q2
      const float det = __fsub_rn(__fmul_rn(v[q[0]], v[q[2]]), __fmul_rn(v[q[1]], v[q[3]]));
      const bool join_pos = det == 0.f ? (pq[0] == 1) : (pq[0] ? det > 0.f : det < 0.f);
      for (int s = 0; s < 4; ++s) {
        const bool cut = join_pos ? !pq[s] : pq[s];
        if (!cut) continue;
        const int e_in = e[(s + 3) & 3], e_out = e[s];
        if (pq[s]) nxt[e_in] = (int8_t)e_out; else nxt[e_out] = (int8_t)e_in;
      }
    }
  }
  int nl = 0, total = 0, seen = 0;
  for (int s = 0; s < 12; ++s) {
    if (nxt[s] < 0 || ((seen >> s) & 1)) continue;
    int n = 0, e = s;
    while (e >= 0 && !((seen >> e) & 1) && total + n < 12) { seen |= 1 << e; loop[total + n++] = (int8_t)e; e = nxt[e]; }
    len[nl++] = (int8_t)n;
    total += n;
  }
  return nl;
}

// bit f set when local edge e lies on cube face f (kFaces order: x=0, x=1, y=0, y=1, z=0, z=1)
__device__ __forceinline__ int edge_faces(int e) {
  const int lo = edge_lo(e), ax = e >> 2;
  int f = 0;
  for (int b = 0; b < 3; ++b)
    if (b != ax) f |= 1 << (2 * b + ((lo >> (2 - b)) & 1));
  return f;
}

constexpr int kCentre = 16;

// A loop from cell_loops starts at its smallest edge; its canonical order runs from there towards the smaller of the two
// neighbours.  Writes it to c[]; returns true when that is the reverse of the given order.
__device__ __forceinline__ bool canonical_loop(const int8_t* __restrict__ l, int n, int8_t* __restrict__ c) {
  const bool rev = n > 2 && l[n - 1] < l[1];
  c[0] = l[0];
  for (int i = 1; i < n; ++i) c[i] = rev ? l[n - i] : l[i];
  return rev;
}   // tri[] entry kCentre + l: the centre vertex of the cell's loop l

// Triangulation of one loop l[0..n) of loop `li`.  A chord whose two ends lie on one cube face would also be a chord or a
// segment of the neighbouring cell across that face (a non-manifold edge), so the triangulation with the fewest such
// chords is chosen by a dynamic programme over the polygon (cost[i][j] of loop[i..j], ties -> smallest apex k), emitted
// in pre-order.  When every triangulation needs one (reachable: some loops of 7+ edges through ambiguous faces), the
// loop is fanned around its own centre vertex instead, whose spokes no other cell shares.  Triangles are written in
// reversed loop order (loop order with `descent`); returns the count (n - 2, or n with the centre).  The programme runs
// on the loop in canonical order (canonical_loop) and the winding is flipped back, so a global sign flip (which reverses
// every loop) gives the same triangles with the opposite winding.
__device__ int loop_triangles(const int8_t* __restrict__ lin, int n, int li, int8_t (*tri)[3], bool descent) {
  int8_t l[12];
  const bool rev = canonical_loop(lin, n, l) != descent;
  const int a = rev ? 2 : 1, b = rev ? 1 : 2;     // winding slots
  int fm[12];
  int8_t cost[12][12], apex[12][12];
  for (int i = 0; i < n; ++i) {
    fm[i] = edge_faces(l[i]);
    for (int j = 0; j < n; ++j) cost[i][j] = 0;
  }
  auto bad = [&](int i, int j) { return (j - i > 1 && !(i == 0 && j == n - 1) && (fm[i] & fm[j])) ? 1 : 0; };
  for (int span = 2; span < n; ++span)
    for (int i = 0; i + span < n; ++i) {
      const int j = i + span;
      int best = 127, bk = i + 1;
      for (int k = i + 1; k < j; ++k) {
        const int c = cost[i][k] + cost[k][j] + bad(i, k) + bad(k, j);
        if (c < best) { best = c; bk = k; }
      }
      cost[i][j] = (int8_t)best;
      apex[i][j] = (int8_t)bk;
    }
  if (cost[0][n - 1] != 0) {
    for (int i = 0; i < n; ++i) {
      tri[i][0] = (int8_t)(kCentre + li); tri[i][a] = l[(i + 1) % n]; tri[i][b] = l[i];
    }
    return n;
  }
  int nt = 0, sp = 0;
  int8_t st[12][2];
  st[sp][0] = 0; st[sp][1] = (int8_t)(n - 1); ++sp;
  while (sp > 0) {
    --sp;
    const int i = st[sp][0], j = st[sp][1];
    if (j - i < 2) continue;
    const int k = apex[i][j];
    tri[nt][0] = l[i]; tri[nt][a] = l[j]; tri[nt][b] = l[k];
    ++nt;
    st[sp][0] = (int8_t)k; st[sp][1] = (int8_t)j; ++sp;
    st[sp][0] = (int8_t)i; st[sp][1] = (int8_t)k; ++sp;
  }
  return nt;
}

// triangles of one cell (<= 12) under the corner rule cv; entries are local edge ids or kCentre + loop
template <class C>
__device__ int cell_triangles(const C& cv, const Dims& D, int64_t t, int64_t g, int8_t tri[12][3]) {
  float v[8];
  cv(D, t, g, v);
  int8_t loop[12], len[4];
  const int nl = cell_loops(v, loop, len);
  int nt = 0, off = 0;
  for (int li = 0; li < nl; ++li) {
    nt += loop_triangles(loop + off, len[li], li, tri + nt, C::kDescent);
    off += len[li];
  }
  return nt;
}

template <class C>
__global__ void k_count(C cv, Dims D, const int64_t* __restrict__ cells, int64_t n, int32_t* __restrict__ counts) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    int8_t tri[12][3];
    counts[t] = cell_triangles(cv, D, t, cells[t], tri);
  }
}

// vertex keys: 3 * corner + axis for a lattice-edge point; 3 * n_points + 4 * t + l for the centre of loop l of cells[t]
template <class C>
__global__ void k_emit(C cv, Dims D, const int64_t* __restrict__ cells, int64_t n, const int64_t* __restrict__ offsets,
                       int64_t* __restrict__ keys) {
  const int64_t centre0 = 3 * D.n0 * D.n1 * D.n2;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    int8_t tri[12][3];
    const int64_t g = cells[t];
    const int nt = cell_triangles(cv, D, t, g, tri);
    int64_t* out = keys + 3 * offsets[t];
    for (int i = 0; i < nt; ++i)
      for (int k = 0; k < 3; ++k) {
        const int e = tri[i][k];
        out[3 * i + k] = e >= kCentre ? centre0 + 4 * t + (e - kCentre) : 3 * (g + D.coff(edge_lo(e))) + (e >> 2);
      }
  }
}

// the loop li of cells[c] in canonical order (the order its centre vertex sums its edge points in); returns its length
template <class C>
__device__ int centre_loop(const C& cv, const Dims& D, int64_t c, int64_t g, int li, int8_t cl[12]) {
  float v[8];
  cv(D, c, g, v);
  int8_t loop[12], len[4];
  cell_loops(v, loop, len);
  int off = 0;
  for (int i = 0; i < li; ++i) off += len[i];
  canonical_loop(loop + off, len[li], cl);
  return len[li];
}

// lattice-index coordinates of the point on the edge (lower corner gk, axis ax): t = u_a / (u_a + u_b)
template <class A>
__device__ __forceinline__ void edge_point(const A& df, const Dims& D, int64_t gk, int ax, float x[3]) {
  const float ua = df(gk), ub = df(gk + D.stride(ax));
  const float tt = __fdiv_rn(ua, __fadd_rn(ua, ub));
  for (int k = 0; k < 3; ++k) {
    const float c = (float)D.coord(gk, k);
    x[k] = k == ax ? __fadd_rn(c, tt) : c;
  }
}

template <class A>
__global__ void k_vertices(A df, Dims D, const int64_t* __restrict__ cells,
                           const uint8_t* __restrict__ mask, const int64_t* __restrict__ keys, int64_t n,
                           float* __restrict__ verts) {
  const int64_t centre0 = 3 * D.n0 * D.n1 * D.n2;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t key = keys[t];
    float x[3];
    if (key < centre0) {
      edge_point(df, D, key / 3, (int)(key % 3), x);
    } else {                   // centre of a loop: the mean of its edge points, summed in canonical loop order
      const int64_t c = (key - centre0) >> 2, g = cells[c];
      int8_t cl[12];
      const int len = centre_loop(UdfCorners<A>{df, mask}, D, c, g, (int)((key - centre0) & 3), cl);
      float s[3] = {0.f, 0.f, 0.f}, y[3];
      for (int i = 0; i < len; ++i) {
        const int e = cl[i];
        edge_point(df, D, g + D.coff(edge_lo(e)), e >> 2, y);
        for (int k = 0; k < 3; ++k) s[k] = __fadd_rn(s[k], y[k]);
      }
      for (int k = 0; k < 3; ++k) x[k] = __fdiv_rn(s[k], (float)len);
    }
    for (int k = 0; k < 3; ++k) verts[t * 3 + k] = x[k];
  }
}

// Threshold meshing of f at `level` (nudf_iso_*): the construction above on v = fl32(f - level), with no pseudo-signs and
// no polarity.  A cell is active when its corners take both sides (some v > 0, some v <= 0) and none is NaN.
__global__ void k_iso_active(const float* __restrict__ df, Dims D, float level, int64_t n, uint8_t* __restrict__ flag) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    uint8_t on = 0;
    if (D.is_cell(t)) {
      bool pos = false, neg = false, nan = false;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        const float v = __fsub_rn(df[t + D.coff(c)], level);
        pos |= v > 0.f;
        neg |= v <= 0.f;
        nan |= v != v;
      }
      on = pos && neg && !nan;
    }
    flag[t] = on;
  }
}

// Active cells without a scan of every cell (nudf_iso_cells_*): every active cell has a corner with v <= 0, which is
// finite and therefore stored, so visiting the storage positions of the lattice (S below) with v <= 0 and testing the up
// to 8 cells holding each finds them all.  A cell is emitted by its lowest corner with v <= 0 only (corners ascend with
// the flat index), so once.  The test is k_iso_active's on the same corner values, so the set is nonzero(nudf_iso_active)
// on any lattice whose reader gives those values -- +inf (unstored) and NaN corners included, with no Lipschitz condition.
// The positions are the items of compact.cuh's stable compaction (IsoCells below), so the cells come in position order;
// the caller sorts.
struct DenseSites {             // the flat array: position = flat index
  DenseDf df;
  int64_t n;
  __device__ __forceinline__ float at(int64_t p) const { return df.p[p]; }
  __device__ __forceinline__ bool point(const Dims& D, int64_t p, int64_t x[3]) const {
#pragma unroll
    for (int a = 0; a < 3; ++a) x[a] = D.coord(p, a);
    return true;
  }
  // w[(a + 1) * 9 + (b + 1) * 3 + c + 1] = the value at x + (a, b, c) for the offsets inside the lattice (others unread)
  __device__ __forceinline__ void around(const Dims& D, const int64_t x[3], const bool in[3][3], float w[27]) const {
    const int64_t g = (x[0] * D.n1 + x[1]) * D.n2 + x[2];
#pragma unroll
    for (int t = 0; t < 27; ++t)
      if (in[0][t / 9] && in[1][(t / 3) % 3] && in[2][t % 3])
        w[t] = df.p[g + (t / 9 - 1) * D.n1 * D.n2 + ((t / 3) % 3 - 1) * D.n2 + (t % 3 - 1)];
  }
};

struct BrickSites {             // the brick store: coarse positions, then brick slots (nudf_sb_flat's positions)
  BrickDf st;
  const int64_t* __restrict__ keys;
  int64_t n;
  __device__ __forceinline__ float at(int64_t p) const { return st.at(p); }
  // the lattice point stored at p; false for a brick slot beyond N - 1 or of a point held in coarse
  __device__ __forceinline__ bool point(const Dims&, int64_t p, int64_t x[3]) const {
    const int64_t m3 = st.mc * st.mc * st.mc, N = st.N;
    if (p < m3) {
      x[0] = min((p / (st.mc * st.mc)) * st.c, N - 1);
      x[1] = min(((p / st.mc) % st.mc) * st.c, N - 1);
      x[2] = min((p % st.mc) * st.c, N - 1);
      return true;
    }
    const int64_t q = p - m3, key = keys[q / kBrickPoints], l = q % kBrickPoints;
    x[0] = (key / (st.nbk * st.nbk)) * kBrick + l / (kBrick * kBrick);
    x[1] = ((key / st.nbk) % st.nbk) * kBrick + (l / kBrick) % kBrick;
    x[2] = (key % st.nbk) * kBrick + l % kBrick;
    return x[0] < N && x[1] < N && x[2] < N && !(st.coarse_of(x[0]) >= 0 && st.coarse_of(x[1]) >= 0 && st.coarse_of(x[2]) >= 0);
  }
  // as DenseSites::around, through BrickDf::position with the per-axis terms computed once
  __device__ __forceinline__ void around(const Dims&, const int64_t x[3], const bool in[3][3], float w[27]) const {
    int64_t co[3][3], bk[3][3], lo[3][3];
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int o = 0; o < 3; ++o) {
        const int64_t y = x[a] + o - 1;
        co[a][o] = in[a][o] ? st.coarse_of(y) : -1;
        bk[a][o] = y / kBrick;
        lo[a][o] = y % kBrick;
      }
#pragma unroll
    for (int t = 0; t < 27; ++t) {
      const int u = t / 9, v = (t / 3) % 3, z = t % 3;
      if (!(in[0][u] && in[1][v] && in[2][z])) continue;
      int64_t p;
      if (co[0][u] >= 0 && co[1][v] >= 0 && co[2][z] >= 0) {
        p = (co[0][u] * st.mc + co[1][v]) * st.mc + co[2][z];
      } else {
        const int32_t slot = st.dir[(bk[0][u] * st.nbk + bk[1][v]) * st.nbk + bk[2][z]];
        p = slot < 0 ? -1 : st.mc * st.mc * st.mc + (int64_t)slot * kBrickPoints + (lo[0][u] * kBrick + lo[1][v]) * kBrick + lo[2][z];
      }
      w[t] = st.at(p);
    }
  }
};

// counts the active cells position p owns (cells != NULL: writes them): the cells holding its lattice point of which it
// is the lowest corner with v <= 0, tested as k_iso_active tests them on the values around the point
template <class S>
__device__ __forceinline__ int iso_owned_cells(const S& sites, const Dims& D, float level, int64_t p,
                                               int64_t* __restrict__ cells) {
  if (p >= sites.n || !(__fsub_rn(sites.at(p), level) <= 0.f)) return 0;
  int64_t x[3];
  if (!sites.point(D, p, x)) return 0;
  const int64_t lim[3] = {D.n0, D.n1, D.n2};
  bool in[3][3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
#pragma unroll
    for (int o = 0; o < 3; ++o) in[a][o] = x[a] + o - 1 >= 0 && x[a] + o - 1 < lim[a];
  float w[27];
  sites.around(D, x, in, w);
  int n = 0;
#pragma unroll
  for (int q = 0; q < 8; ++q) {             // the cell whose corner q is the point: corner c at offset c - q per axis
    const int dq[3] = {(q >> 2) & 1, (q >> 1) & 1, q & 1};
    if (!(in[0][1 - dq[0]] && in[0][2 - dq[0]] && in[1][1 - dq[1]] && in[1][2 - dq[1]] && in[2][1 - dq[2]] &&
          in[2][2 - dq[2]]))
      continue;
    bool pos = false, neg = false, nan = false, lower = false;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const int t = (((c >> 2) & 1) - dq[0] + 1) * 9 + (((c >> 1) & 1) - dq[1] + 1) * 3 + ((c & 1) - dq[2] + 1);
      const float v = __fsub_rn(w[t], level);
      pos |= v > 0.f;
      neg |= v <= 0.f;
      nan |= v != v;
      lower |= c < q && v <= 0.f;
    }
    if (pos && neg && !nan && !lower) {
      if (cells) cells[n] = ((x[0] - dq[0]) * D.n1 + x[1] - dq[1]) * D.n2 + x[2] - dq[2];
      ++n;
    }
  }
  return n;
}

// the compaction op of the sites S: the emit pass computes a position's cells again, written in place (no Item holds them)
template <class S>
struct IsoCells {
  struct Item {};
  S sites;
  Dims D;
  float level;
  __device__ __forceinline__ int eval(int64_t p, Item&, bool) const {
    return iso_owned_cells(sites, D, level, p, (int64_t*)nullptr);
  }
  __device__ __forceinline__ void store(int64_t* __restrict__ cells, int64_t j, int64_t p, const Item&) const {
    iso_owned_cells(sites, D, level, p, cells + j);
  }
};

// fp64 lattice-index coordinates of the point on the edge (lower corner gk, axis ax): t = v_a / (v_a - v_b) of the fp32 v
template <class A>
__device__ __forceinline__ void iso_edge_point(const A& df, const Dims& D, float level, int64_t gk, int ax, double x[3]) {
  const double va = __fsub_rn(df(gk), level), vb = __fsub_rn(df(gk + D.stride(ax)), level);
  const double tt = __ddiv_rn(va, __dsub_rn(va, vb));
  for (int k = 0; k < 3; ++k) {
    const double c = (double)D.coord(gk, k);
    x[k] = k == ax ? __dadd_rn(c, tt) : c;
  }
}

template <class A>
__device__ __forceinline__ void iso_vertices(const A& df, const Dims& D, float level, const int64_t* __restrict__ cells,
                                             const int64_t* __restrict__ keys, int64_t n, double* __restrict__ verts) {
  const int64_t centre0 = 3 * D.n0 * D.n1 * D.n2;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t key = keys[t];
    double x[3];
    if (key < centre0) {
      iso_edge_point(df, D, level, key / 3, (int)(key % 3), x);
    } else {                   // centre of a loop: the mean of its edge points, summed in canonical loop order
      const int64_t c = (key - centre0) >> 2, g = cells[c];
      int8_t cl[12];
      const int len = centre_loop(IsoCorners<A>{df, level}, D, c, g, (int)((key - centre0) & 3), cl);
      double s[3] = {0.0, 0.0, 0.0}, y[3];
      for (int i = 0; i < len; ++i) {
        const int e = cl[i];
        iso_edge_point(df, D, level, g + D.coff(edge_lo(e)), e >> 2, y);
        for (int k = 0; k < 3; ++k) s[k] = __dadd_rn(s[k], y[k]);
      }
      for (int k = 0; k < 3; ++k) x[k] = __ddiv_rn(s[k], (double)len);
    }
    for (int k = 0; k < 3; ++k) verts[t * 3 + k] = x[k];
  }
}

template <class A>
__global__ void k_iso_vertices(A df, Dims D, float level, const int64_t* __restrict__ cells, const int64_t* __restrict__ keys,
                               int64_t n, double* __restrict__ verts) {
  iso_vertices(df, D, level, cells, keys, n, verts);
}

// the flat array as a restrict-qualified parameter: its loads take the read-only path, as before the reader template
__global__ void k_iso_vertices_dense(const float* __restrict__ df, Dims D, float level, const int64_t* __restrict__ cells,
                                     const int64_t* __restrict__ keys, int64_t n, double* __restrict__ verts) {
  iso_vertices(DenseDf{df}, D, level, cells, keys, n, verts);
}

static inline Dims dims(const nudf_lattice& l) { return Dims{l.n0, l.n1, l.n2}; }

}  // namespace mc
}  // namespace nudf

using namespace nudf;
using namespace nudf::mc;

int nudf_mc_active(const nudf_lattice* lat, const int64_t* cand, int64_t n_cand, float avg_t, float max_t, uint8_t* flags,
                   void* stream) {
  return with_lattice(lat, [&](auto df) {
    NUDF_REQUIRE(flags && n_cand >= 0 && (cand || lat->df || n_cand == 0), "null pointer or negative count");
    if (n_cand == 0) return 0;
    k_active<<<grid_for(n_cand), 256, 0, (cudaStream_t)stream>>>(df, dims(*lat), cand, n_cand, avg_t, max_t, flags);
    NUDF_LAUNCH_OK();
    return 0;
  });
}

int nudf_mc_cell_signs(const nudf_lattice* lat, const int64_t* cells, int64_t n_cells, const int64_t* idx, int64_t n_idx,
                       const float* normals, uint8_t* mask, void* stream) {
  return with_lattice(lat, [&](auto df) {
    NUDF_REQUIRE(cells && normals && mask && n_cells >= 0, "null pointer or negative count");
    if (n_cells == 0) return 0;
    k_signs<<<grid_for(n_cells), 128, 0, (cudaStream_t)stream>>>(df, dims(*lat), cells, n_cells, idx, n_idx, normals, mask);
    NUDF_LAUNCH_OK();
    return 0;
  });
}

int nudf_mc_links(const nudf_lattice* lat, const int64_t* cells, int64_t n_cells, const uint8_t* mask, int64_t* links,
                  void* stream) {
  return with_lattice(lat, [&](auto df) {
    NUDF_REQUIRE(cells && mask && links && n_cells >= 0, "null pointer or negative count");
    if (n_cells == 0) return 0;
    k_links<<<grid_for(n_cells), 256, 0, (cudaStream_t)stream>>>(df, dims(*lat), cells, n_cells, mask, links);
    NUDF_LAUNCH_OK();
    return 0;
  });
}

int nudf_mc_polarity(const int64_t* links, int64_t n_cells, const uint8_t* mask_in, int64_t* parent_ws, int64_t* hook_ws,
                     int32_t* flag_ws, uint8_t* mask_out, int32_t* stats, void* stream) {
  NUDF_REQUIRE(links && mask_in && parent_ws && hook_ws && flag_ws && mask_out && n_cells >= 0, "null pointer");
  if (stats) stats[0] = stats[1] = 0;
  if (n_cells == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  unsigned long long* hook = (unsigned long long*)hook_ws;
  const unsigned gr = grid_for(n_cells);
  k_uf_init<<<gr, 256, 0, st>>>(parent_ws, hook, n_cells);
  NUDF_LAUNCH_OK();
  // Termination: a round that hooks turns at least one root into a child of a smaller root and creates none, so there are
  // at most n_cells - 1 hooking rounds.  In practice a hooking round leaves only the roots that are local minima of their
  // root neighbourhood (cells are numbered by lattice index, so a surface sheet collapses onto few minima).  Measured
  // (stats[0] / stats[1], reported by tools/mesh_bench.py and tests/test_gpu_mesh.py): 1-2 hooking rounds and 9-19
  // pointer-jumping passes on the golden meshes and the C5 scene at 256^3 / 512^3, 4 rounds on a random field.  Each
  // pass costs one host read of flag_ws.
  int32_t changed = 0, rounds = 0, jumps = 0;
  for (;;) {
    do {
      NUDF_CUDA_OK(cudaMemsetAsync(flag_ws, 0, sizeof(int32_t), st));
      k_uf_jump<<<gr, 256, 0, st>>>(parent_ws, n_cells, flag_ws);
      NUDF_LAUNCH_OK();
      ++jumps;
      NUDF_CUDA_OK(cudaMemcpyAsync(&changed, flag_ws, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
      NUDF_CUDA_OK(cudaStreamSynchronize(st));
    } while (changed);
    NUDF_CUDA_OK(cudaMemsetAsync(flag_ws, 0, sizeof(int32_t), st));
    k_uf_hook<<<grid_for(3 * n_cells), 256, 0, st>>>(links, n_cells, parent_ws, hook);
    NUDF_LAUNCH_OK();
    k_uf_apply<<<gr, 256, 0, st>>>(hook, parent_ws, n_cells, flag_ws);
    NUDF_LAUNCH_OK();
    NUDF_CUDA_OK(cudaMemcpyAsync(&changed, flag_ws, sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    NUDF_CUDA_OK(cudaStreamSynchronize(st));
    if (!changed) break;
    ++rounds;
  }
  if (stats) { stats[0] = rounds; stats[1] = jumps; }
  k_uf_final<<<gr, 256, 0, st>>>(parent_ws, mask_in, n_cells, mask_out);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_mc_count(const nudf_lattice* lat, const int64_t* cells, int64_t n_cells, const uint8_t* mask, int32_t* counts,
                  void* stream) {
  return with_lattice(lat, [&](auto df) {
    NUDF_REQUIRE(cells && mask && counts && n_cells >= 0, "null pointer or negative count");
    if (n_cells == 0) return 0;
    k_count<<<grid_for(n_cells), 128, 0, (cudaStream_t)stream>>>(UdfCorners<decltype(df)>{df, mask}, dims(*lat), cells,
                                                                  n_cells, counts);
    NUDF_LAUNCH_OK();
    return 0;
  });
}

int nudf_mc_emit(const nudf_lattice* lat, const int64_t* cells, int64_t n_cells, const uint8_t* mask, const int64_t* offsets,
                 int64_t* keys, void* stream) {
  return with_lattice(lat, [&](auto df) {
    NUDF_REQUIRE(cells && mask && offsets && keys && n_cells >= 0, "null pointer or negative count");
    if (n_cells == 0) return 0;
    k_emit<<<grid_for(n_cells), 128, 0, (cudaStream_t)stream>>>(UdfCorners<decltype(df)>{df, mask}, dims(*lat), cells,
                                                                 n_cells, offsets, keys);
    NUDF_LAUNCH_OK();
    return 0;
  });
}

int nudf_mc_vertices(const nudf_lattice* lat, const int64_t* cells, int64_t n_cells, const uint8_t* mask, const int64_t* keys,
                     int64_t n_keys, float* verts, void* stream) {
  return with_lattice(lat, [&](auto df) {
    NUDF_REQUIRE(cells && mask && keys && verts && n_cells >= 0 && n_keys >= 0, "null pointer or negative count");
    if (n_keys == 0) return 0;
    k_vertices<<<grid_for(n_keys), 128, 0, (cudaStream_t)stream>>>(df, dims(*lat), cells, mask, keys, n_keys, verts);
    NUDF_LAUNCH_OK();
    return 0;
  });
}

#define ISO_LEVEL_OK() NUDF_REQUIRE(level == level && level - level == 0.f, "level must be finite")

// the threshold stages on a lattice descriptor
template <class F>
static int with_iso_lattice(const nudf_lattice* lat, float level, F&& launch) {
  ISO_LEVEL_OK();
  return with_lattice(lat, [&](auto df) { return launch(df, dims(*lat)); });
}

// every cell of a df lattice; the raw restrict pointer keeps k_iso_active's loads on the read-only path
int nudf_iso_active(const nudf_lattice* lat, float level, uint8_t* flags, void* stream) {
  return with_iso_lattice(lat, level, [&](auto, Dims D) {
    NUDF_REQUIRE(lat->df, "nudf_iso_active reads a df lattice only (nudf_iso_cells_* read a store)");
    NUDF_REQUIRE(flags, "null pointer");
    const int64_t n = D.n0 * D.n1 * D.n2;
    k_iso_active<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(lat->df, D, level, n, flags);
    NUDF_LAUNCH_OK();
    return 0;
  });
}

static int iso_cells(const nudf_lattice* lat, float level, int64_t n_seg, int32_t* counts, const int64_t* offsets,
                     int64_t* cells, void* stream) {
  return with_iso_lattice(lat, level, [&](auto df, Dims D) {
    NUDF_REQUIRE(offsets ? (cells != nullptr) : (counts != nullptr), "null pointer");
    int64_t n_pos = D.n0 * D.n1 * D.n2;
    if (lat->store) {
      NUDF_REQUIRE(lat->store->n_bricks == 0 || lat->store->keys, "null brick keys");
      n_pos = (int64_t)lat->store->mc * lat->store->mc * lat->store->mc + lat->store->n_bricks * kBrickPoints;
    }
    NUDF_REQUIRE(n_seg == cdiv(n_pos, kSeg), "n_seg must be ceil(storage positions / NUDF_COMPACT_SEG)");
    using Out = int64_t* __restrict__;
    if constexpr (std::is_same<decltype(df), DenseDf>::value)
      return seg_compact<Out>(IsoCells<DenseSites>{{df, n_pos}, D, level}, n_pos, counts, offsets, cells, stream);
    else
      return seg_compact<Out>(IsoCells<BrickSites>{{df, lat->store->keys, n_pos}, D, level}, n_pos, counts, offsets,
                              cells, stream);
  });
}

int nudf_iso_cells_count(const nudf_lattice* lat, float level, int64_t n_seg, int32_t* counts, void* stream) {
  return iso_cells(lat, level, n_seg, counts, nullptr, nullptr, stream);
}

int nudf_iso_cells_emit(const nudf_lattice* lat, float level, int64_t n_seg, const int64_t* offsets, int64_t* cells,
                        void* stream) {
  NUDF_REQUIRE(offsets, "null pointer");
  return iso_cells(lat, level, n_seg, nullptr, offsets, cells, stream);
}

int nudf_iso_count(const nudf_lattice* lat, float level, const int64_t* cells, int64_t n_cells, int32_t* counts,
                   void* stream) {
  return with_iso_lattice(lat, level, [&](auto df, Dims D) {
    NUDF_REQUIRE(cells && counts && n_cells >= 0, "null pointer or negative count");
    if (n_cells == 0) return 0;
    k_count<<<grid_for(n_cells), 128, 0, (cudaStream_t)stream>>>(IsoCorners<decltype(df)>{df, level}, D, cells, n_cells,
                                                                  counts);
    NUDF_LAUNCH_OK();
    return 0;
  });
}

int nudf_iso_emit(const nudf_lattice* lat, float level, const int64_t* cells, int64_t n_cells, const int64_t* offsets,
                  int64_t* keys, void* stream) {
  return with_iso_lattice(lat, level, [&](auto df, Dims D) {
    NUDF_REQUIRE(cells && offsets && keys && n_cells >= 0, "null pointer or negative count");
    if (n_cells == 0) return 0;
    k_emit<<<grid_for(n_cells), 128, 0, (cudaStream_t)stream>>>(IsoCorners<decltype(df)>{df, level}, D, cells, n_cells,
                                                                 offsets, keys);
    NUDF_LAUNCH_OK();
    return 0;
  });
}

int nudf_iso_vertices(const nudf_lattice* lat, float level, const int64_t* cells, int64_t n_cells, const int64_t* keys,
                      int64_t n_keys, double* verts, void* stream) {
  return with_iso_lattice(lat, level, [&](auto df, Dims D) {
    NUDF_REQUIRE(cells && keys && verts && n_cells >= 0 && n_keys >= 0, "null pointer or negative count");
    if (n_keys == 0) return 0;
    if constexpr (std::is_same<decltype(df), DenseDf>::value)
      k_iso_vertices_dense<<<grid_for(n_keys), 128, 0, (cudaStream_t)stream>>>(df.p, D, level, cells, keys, n_keys, verts);
    else
      k_iso_vertices<<<grid_for(n_keys), 128, 0, (cudaStream_t)stream>>>(df, D, level, cells, keys, n_keys, verts);
    NUDF_LAUNCH_OK();
    return 0;
  });
}

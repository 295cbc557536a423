// Readers of an N^3 udf lattice by flat index g = (i * N + j) * N + k, shared by the band block test (mesh_band.cu), the
// MeshUDF marching cubes (mesh_udf.cu) and the brick store's own kernels (mesh_sparse.cu).
//   DenseDf   the flat fp32 array (grid.udf_band, grid.udf_grid): df[g];
//   BrickDf   the block-sparse narrow band of grid.udf_band_sparse (nudf_brick_store in include/nudf.h): the points of the
//             stride-c lattice (per axis 0, c, 2 c, ... and N - 1) in a dense coarse array [mc^3], every other point in an
//             8^3 brick found through a dense directory over the ceil(N / 8)^3 bricks; a point whose brick has no slot
//             reads +inf, as an unevaluated point of the dense band does.
// with_lattice picks the reader a nudf_lattice descriptor names, so that every entry point taking one launches the same
// kernel instantiations for both forms.
#pragma once
#include <math.h>
#include <stdint.h>

#include "../../include/nudf.h"
#include "common.cuh"

namespace nudf {

struct DenseDf {
  const float* __restrict__ p;
  __device__ __forceinline__ float operator()(int64_t g) const { return p[g]; }
};

constexpr int kBrick = NUDF_BRICK;                  // lattice points per brick edge
constexpr int kBrickPoints = kBrick * kBrick * kBrick;

struct BrickDf {
  int64_t N;                        // lattice points per axis
  int64_t c;                        // stride of the coarse lattice
  int64_t mc;                       // coarse points per axis: ceil((N - 1) / c) + 1
  int64_t nbk;                      // bricks per axis: ceil(N / 8)
  const float* __restrict__ coarse;
  const int32_t* __restrict__ dir;
  const float* __restrict__ bricks;

  // coarse coordinate of lattice coordinate i, or -1 when i is not on the stride-c lattice
  __device__ __forceinline__ int64_t coarse_of(int64_t i) const { return i == N - 1 ? mc - 1 : (i % c == 0 ? i / c : -1); }
  // storage position: [0, mc^3) in the coarse array, mc^3 + slot * 512 + local in the bricks, -1 for a missing brick
  __device__ __forceinline__ int64_t position(int64_t i, int64_t j, int64_t k) const {
    const int64_t ci = coarse_of(i), cj = coarse_of(j), ck = coarse_of(k);
    if (ci >= 0 && cj >= 0 && ck >= 0) return (ci * mc + cj) * mc + ck;
    const int32_t slot = dir[((i / kBrick) * nbk + j / kBrick) * nbk + k / kBrick];
    if (slot < 0) return -1;
    return mc * mc * mc + (int64_t)slot * kBrickPoints + ((i % kBrick) * kBrick + j % kBrick) * kBrick + k % kBrick;
  }
  __device__ __forceinline__ float at(int64_t p) const {
    const int64_t m3 = mc * mc * mc;
    return p < 0 ? INFINITY : (p < m3 ? coarse[p] : bricks[p - m3]);
  }
  __device__ __forceinline__ float operator()(int64_t g) const {
    const int64_t nn = N * N;
    return at(position(g / nn, (g / N) % N, g % N));
  }
};

inline BrickDf brick_df(const nudf_brick_store& s) {
  return BrickDf{s.n, s.c, s.mc, s.nbk, s.coarse, s.dir, s.bricks};
}

// Checks the descriptor, then returns launch(DenseDf) or launch(BrickDf) for the lattice it names (-1: invalid).
template <class F>
inline int with_lattice(const nudf_lattice* lat, F&& launch) {
  NUDF_REQUIRE(lat, "null lattice");
  NUDF_REQUIRE(lat->n0 >= 2 && lat->n1 >= 2 && lat->n2 >= 2, "lattice dimensions must be at least 2");
  NUDF_REQUIRE(!lat->df != !lat->store, "exactly one of df and store must be set");
  if (lat->df) return launch(DenseDf{lat->df});
  const nudf_brick_store* st = lat->store;
  NUDF_REQUIRE(st->n >= 2 && st->coarse && st->dir && (st->bricks || st->n_bricks == 0), "null or invalid brick store");
  NUDF_REQUIRE(lat->n0 == st->n && lat->n1 == st->n && lat->n2 == st->n, "the lattice dimensions must be the store's n");
  return launch(brick_df(*st));
}

}  // namespace nudf

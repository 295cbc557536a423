// The block-sparse narrow band of grid.udf_band_sparse (layout: nudf_brick_store in include/nudf.h, reader: BrickDf in
// df_access.cuh): brick allocation from the kept blocks of the coarse stride, value stores and reads by flat lattice index,
// and the inverse map from storage positions to flat indices that the near-surface selection uses.
// tests/proto/udf_sparse.py restates the layout and the level chain in NumPy.
#include "../../include/nudf.h"
#include "common.cuh"
#include "df_access.cuh"

namespace nudf {
namespace sb {

// one thread per block of stride s: a kept block marks every brick that meets its closed box [a, min(a + s, N - 1)]^3
__global__ void k_mark(BrickDf st, int64_t s, int64_t nb, const uint8_t* __restrict__ flags, int32_t* __restrict__ marks) {
  const int64_t n = nb * nb * nb;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    if (!flags[t]) continue;
    const int64_t b[3] = {t / (nb * nb), (t / nb) % nb, t % nb};
    int64_t lo[3], hi[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      lo[a] = b[a] * s / kBrick;
      hi[a] = min(b[a] * s + s, st.N - 1) / kBrick;
    }
    for (int64_t x = lo[0]; x <= hi[0]; ++x)
      for (int64_t y = lo[1]; y <= hi[1]; ++y)
        for (int64_t z = lo[2]; z <= hi[2]; ++z) marks[(x * st.nbk + y) * st.nbk + z] = 1;
  }
}

__global__ void k_store(BrickDf st, float* __restrict__ coarse, float* __restrict__ bricks, const int64_t* __restrict__ idx,
                        const float* __restrict__ vals, int64_t n, int32_t* __restrict__ missing) {
  const int64_t m3 = st.mc * st.mc * st.mc, nn = st.N * st.N;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t g = idx[t];
    const int64_t p = st.position(g / nn, (g / st.N) % st.N, g % st.N);
    if (p < 0) *missing = 1;
    else if (p < m3) coarse[p] = vals[t];
    else bricks[p - m3] = vals[t];
  }
}

__global__ void k_gather(BrickDf st, const int64_t* __restrict__ idx, int64_t n, float* __restrict__ out) {
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x)
    out[t] = st(idx[t]);
}

__global__ void k_flat(BrickDf st, const int64_t* __restrict__ keys, const int64_t* __restrict__ pos, int64_t n,
                       int64_t* __restrict__ out) {
  const int64_t m3 = st.mc * st.mc * st.mc;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < n; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = pos[t];
    int64_t i, j, k;
    if (p < m3) {
      const int64_t ci = p / (st.mc * st.mc), cj = (p / st.mc) % st.mc, ck = p % st.mc;
      i = min(ci * st.c, st.N - 1);
      j = min(cj * st.c, st.N - 1);
      k = min(ck * st.c, st.N - 1);
    } else {
      const int64_t q = p - m3, key = keys[q / kBrickPoints], l = q % kBrickPoints;
      i = (key / (st.nbk * st.nbk)) * kBrick + l / (kBrick * kBrick);
      j = ((key / st.nbk) % st.nbk) * kBrick + (l / kBrick) % kBrick;
      k = (key % st.nbk) * kBrick + l % kBrick;
    }
    out[t] = (i * st.N + j) * st.N + k;
  }
}

}  // namespace sb
}  // namespace nudf

using namespace nudf;
using namespace nudf::sb;

#define SB_STORE_OK() NUDF_REQUIRE(st && st->n >= 2 && st->c >= 1 && st->coarse && st->dir && \
                                   (st->n_bricks == 0 || (st->bricks && st->keys)), "null or invalid brick store")

int nudf_sb_mark(const nudf_brick_store* st, int32_t s, const uint8_t* flags, int32_t* marks, void* stream) {
  SB_STORE_OK();
  NUDF_REQUIRE(flags && marks, "null pointer");
  NUDF_REQUIRE(s >= st->c && s % st->c == 0, "the stride must be a multiple of the store's coarse stride");
  const int64_t nb = cdiv(st->n - 1, s);
  k_mark<<<grid_for(nb * nb * nb), 256, 0, (cudaStream_t)stream>>>(brick_df(*st), s, nb, flags, marks);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_sb_store(const nudf_brick_store* st, const int64_t* idx, const float* vals, int64_t n, int32_t* missing, void* stream) {
  SB_STORE_OK();
  NUDF_REQUIRE(n >= 0 && missing && (n == 0 || (idx && vals)), "null pointer or negative count");
  if (n == 0) return 0;
  k_store<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(brick_df(*st), st->coarse, st->bricks, idx, vals, n, missing);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_sb_gather(const nudf_brick_store* st, const int64_t* idx, int64_t n, float* out, void* stream) {
  SB_STORE_OK();
  NUDF_REQUIRE(n >= 0 && (n == 0 || (idx && out)), "null pointer or negative count");
  if (n == 0) return 0;
  k_gather<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(brick_df(*st), idx, n, out);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_sb_flat(const nudf_brick_store* st, const int64_t* pos, int64_t n, int64_t* out, void* stream) {
  SB_STORE_OK();
  NUDF_REQUIRE(n >= 0 && (n == 0 || (pos && out)), "null pointer or negative count");
  if (n == 0) return 0;
  k_flat<<<grid_for(n), 256, 0, (cudaStream_t)stream>>>(brick_df(*st), st->keys, pos, n, out);
  NUDF_LAUNCH_OK();
  return 0;
}

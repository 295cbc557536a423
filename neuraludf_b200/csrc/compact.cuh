// Stable segmented compaction, shared by the point clouds' survivors (udf_cloud.cu), the visibility pairs
// (udf_paint.cu) and the active cells of threshold meshing (mesh_udf.cu).  The items [0, n) are taken in segments of
// NUDF_COMPACT_SEG, one thread per item and one block per segment, the blocks striding over the segments.  The count
// pass (offsets NULL) writes counts[seg], the outputs of the segment's items; the emit pass makes the same decisions
// again and writes those outputs from offsets[seg] (an exclusive scan of the counts, plus any base the caller adds), in
// item order.  Both passes run one instantiation, so they agree exactly on what each item makes.
//
// An Op provides
//   Item, what eval hands on to store;
//   int eval(int64_t i, Item& it, bool emit): the number of outputs of item i < n.  emit is true in the emit pass only,
//     the one place a side effect may happen;
//   void store(Out out, int64_t j, int64_t i, const Item& it): writes them to out from output j on.
// The output is a kernel parameter of its own, not an op member: as a restrict-qualified pointer it tells the compiler
// that the stores leave the op's inputs alone, so those are loaded through the read-only path.
#pragma once
#include "../../include/nudf.h"
#include "common.cuh"

namespace nudf {

constexpr int kSeg = NUDF_COMPACT_SEG;

template <class Op, class Out>
__global__ void __launch_bounds__(kSeg) k_seg_compact(Op op, int64_t n, int64_t n_seg, int32_t* __restrict__ counts,
                                                      const int64_t* __restrict__ offsets, Out out) {
  __shared__ int32_t warp_sum[kSeg / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int64_t seg = blockIdx.x; seg < n_seg; seg += gridDim.x) {   // every thread of the block takes both barriers
    const int64_t i = seg * kSeg + threadIdx.x;
    typename Op::Item it;
    const int c = i < n ? op.eval(i, it, offsets != nullptr) : 0;
    int incl = c;                           // inclusive scan over the block: warps, then the warp totals
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += y;
    }
    if (lane == 31) warp_sum[warp] = incl;
    __syncthreads();
    int before = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kSeg / 32; ++w) {
      before += w < warp ? warp_sum[w] : 0;
      total += warp_sum[w];
    }
    if (!offsets) {
      if (threadIdx.x == 0) counts[seg] = total;
    } else if (c) {
      op.store(out, offsets[seg] + before + incl - c, i, it);
    }
    __syncthreads();                        // warp_sum is reused by the next segment
  }
}

// the count pass (offsets NULL; counts[ceil(n / kSeg)]) or the emit pass of op over n items.  Out is given explicitly,
// so that a pointer output keeps its __restrict__ qualifier in the kernel.
template <class Out, class Op>
static inline int seg_compact(Op op, int64_t n, int32_t* counts, const int64_t* offsets, Out out, void* stream) {
  k_seg_compact<Op, Out><<<grid_for(n, kSeg), kSeg, 0, (cudaStream_t)stream>>>(op, n, cdiv(n, kSeg), counts, offsets,
                                                                             out);
  NUDF_LAUNCH_OK();
  return 0;
}

}  // namespace nudf

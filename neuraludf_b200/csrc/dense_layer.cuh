// One dense layer Y = X W^T (+ b) as the host code of the three networks sees it: its shape, where its fp32 weights and bias
// live, and the split-bf16 operand images (gemm_tc.cuh) it owns.  The planners, the fold / prepare job lists and the launches
// all read this record, so a layer's N, K, plane count and image offset are stated once: here.
#pragma once
#include "gemm_engine.cuh"

namespace nudf {

// The operand images a layer can own: of X W^T with 2 planes (tangent chain) and with 3 planes (forward passes), of dY W with
// 2 planes (gradient chains).  A network names the ones its launches read as bits 1 << IMG_*.
enum { IMG_NT2 = 0, IMG_NT3 = 1, IMG_NN2 = 2, IMG_KINDS = 3, IMG_ALL = (1 << IMG_KINDS) - 1 };

// The fold and prepare job lists take every layer of a network in one launch and are filled without a bounds check.  The
// colour network is the largest: two stacks of up to NUDF_MAX_LAYERS layers, each layer with at most two images (NT3, NN2).
// The UDF network needs at most 3 NUDF_MAX_LAYERS images, NeRF++ at most 2 (NUDF_MAX_LAYERS + 4).
static_assert(NUDF_MAX_JOBS >= 2 * NUDF_MAX_LAYERS, "FoldJobs must hold both stacks of the deepest colour network");
static_assert(sizeof(tc::PrepWJobs::j) / sizeof(tc::PrepWJob) >= 4 * NUDF_MAX_LAYERS,
              "PrepWJobs must hold every image of the deepest colour network");

struct DenseLayer {
  int n_out, n_in;
  int64_t ldw;                  // W is [n_out, ldw]
  int64_t w_off, b_off;         // weight-normed networks: offsets of W in the folded buffer and of the bias in the bias block
  int64_t img_off[IMG_KINDS];   // uint16 offsets into the image block; -1 = the layer has no such image
  const float* W;
  const float* bias;
  const uint16_t* img;          // the image block; null (exact-fp32 engine) sends every launch to the FFMA kernel
};

struct ImgShape { int N, K, transposed, planes; };
static inline ImgShape img_shape(const DenseLayer& L, int kind) {
  if (kind == IMG_NN2) return ImgShape{L.n_in, L.n_out, 1, 2};     // operand of dY W   (N = in,  K = out)
  return ImgShape{L.n_out, L.n_in, 0, kind == IMG_NT3 ? 3 : 2};    // operand of X W^T  (N = out, K = in)
}

// plan: the layer gets the images in `want` whose shape gemm_nt / gemm_nn run on the tensor cores (any other image would be
// rebuilt every optimiser step and read by no launch), packed from `off`; returns the offset after them
static inline int64_t plan_images(DenseLayer& L, int want, int64_t off) {
  for (int k = 0; k < IMG_KINDS; ++k) {
    const ImgShape s = img_shape(L, k);
    L.img_off[k] = -1;
    if ((want >> k & 1) && tc_shape_ok(s.N, s.K)) { L.img_off[k] = off; off += tc::image_elems(s.N, s.K, s.planes); }
  }
  return off;
}

// weight-normed networks keep one buffer: the folded fp32 weights of every layer, then the image block.  wfold may be null
// (size queries): such a plan is not launched from
static inline void bind_layers(DenseLayer* L, int n, const float* wfold, int64_t w_total) {
  for (int i = 0; i < n; ++i) {
    L[i].W = wfold != nullptr ? wfold + L[i].w_off : nullptr;
    L[i].img = wfold != nullptr ? reinterpret_cast<const uint16_t*>(wfold + w_total) : nullptr;
  }
}

// prepare: the jobs that build the layer's images of `kinds` from its fp32 weights, into the (writable) image block
static inline void add_prep_jobs(tc::PrepWJobs& pj, const DenseLayer& L, uint16_t* img, int kinds) {
  for (int k = 0; k < IMG_KINDS; ++k) {
    const ImgShape s = img_shape(L, k);
    if ((kinds >> k & 1) && L.img_off[k] >= 0)
      pj.j[pj.n++] = tc::PrepWJob{L.W, img + L.img_off[k], (int)L.ldw, s.N, s.K, s.transposed, s.planes};
  }
}

// weight norm: W = g v / |v| into the folded buffer, and its adjoint (dg, dv) from the folded gradient
static inline void add_fold_job(FoldJobs& jobs, const DenseLayer& L, const float* g, const float* v, float* wfold) {
  jobs.j[jobs.n++] = FoldJob{g, v, nullptr, nullptr, nullptr, wfold + L.w_off, L.n_out, L.n_in, (int)L.ldw};
}
static inline void add_unfold_job(FoldJobs& jobs, const DenseLayer& L, const float* g, const float* v, const float* dwfold,
                                  float* dg, float* dv) {
  jobs.j[jobs.n++] = FoldJob{g, v, dwfold + L.w_off, dg, dv, nullptr, L.n_out, L.n_in, (int)L.ldw};
}

// launch: Y = epi(X W^T) and dX = epi(dY W) against the layer's own image of the chain's plane count; without one (or with
// the chain masked off) the exact-fp32 FFMA kernel reads W itself
static inline const uint16_t* layer_img(const DenseLayer& L, int kind) {
  return L.img != nullptr && L.img_off[kind] >= 0 ? L.img + L.img_off[kind] : nullptr;
}
template <class Epi>
static inline int layer_nt(const DenseLayer& L, const float* X, int64_t ldx, int64_t P, const Epi& epi, int chain, cudaStream_t st) {
  const bool fwd = (chain & (TC_FWD | TC_RELU_FWD)) != 0;          // the forward passes take 3 planes (gemm_engine.cuh)
  return gemm_nt(X, ldx, L.W, L.ldw, P, L.n_out, L.n_in, epi, st, layer_img(L, fwd ? IMG_NT3 : IMG_NT2), chain, fwd ? 3 : 2);
}
template <class Epi>
static inline int layer_nn(const DenseLayer& L, const float* dY, int64_t ldy, int64_t P, const Epi& epi, int chain, cudaStream_t st) {
  return gemm_nn(dY, ldy, L.W, L.ldw, P, L.n_in, L.n_out, epi, st, layer_img(L, IMG_NN2), chain);
}

}  // namespace nudf

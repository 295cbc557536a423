// Engine dispatch: every dense contraction of the hot path goes through gemm_nt / gemm_nn / gemm_tn.
//   engine 0: exact-fp32 FFMA kernel (gemm_simt.cuh) -- always used for small / odd shapes;
//   engine 1: wgmma split-bf16 tensor-core kernels (gemm_tc.cuh) when the caller supplies the pre-split weight
//             image built at fold time (gemm_nt / gemm_nn) or for the weight-gradient contraction (gemm_tn).
// Which chains may use the tensor engine is a bit mask (NUDF_TC_MASK, see tc_mask()): the forward passes need fp32-grade
// accuracy (udf feeds exp(-25000 u) and sigmoid(400 u); ReLU gates), so they take three bf16 planes / six products, the
// gradient chains tolerate the 2-plane (3-product) split.
#pragma once
#include <stdlib.h>
#include "gemm_tc.cuh"

namespace nudf {

// TC_FWD: UDF value chain (hidden layers and feature rows on gemm_w<3>; the udf-head row stays an exact-fp32 dot product,
// udf_net.cu); TC_REV/TAN/BWD: UDF gradient, tangent and backward chains; TC_WGRAD:
// weight gradients; TC_COLOR / TC_NERF: BACKWARD data GEMMs of the ReLU networks (2 planes); TC_RELU_FWD: their forward passes,
// with 3 planes / 6 products (gemm_w<3>, per-K-slice accumulators summed in fp32): a 4e-6 perturbation of a pre-activation (the
// 2-plane split) flips ~60x more ReLU gates than the reference's own fp32 rounding does, which shows up as O(1/batch) jumps in
// the parameter gradients and fails test_color_network_vs_reference_and_grads; the 3-plane product (3.5e-7 per layer) passes.
enum TcChain { TC_FWD = 1, TC_REV = 2, TC_TAN = 4, TC_BWD = 8, TC_WGRAD = 16, TC_COLOR = 32, TC_NERF = 64, TC_RELU_FWD = 128 };

int get_engine();
int tc_mask();
static inline bool tc_on(int chain) { return get_engine() == 1 && (tc_mask() & chain) != 0; }
// the operand shapes B(N, K) the weights-resident tensor-core kernel takes; the planners (dense_layer.cuh) build images of these only
static inline bool tc_shape_ok(int N, int64_t K) { return K >= 32 && N >= 16; }

template <class Epi>
static inline int gemm_nt(const float* A, int64_t lda, const float* W, int64_t ldw, int64_t M, int N, int64_t K,
                          const Epi& epi, cudaStream_t st, const uint16_t* img = nullptr, int chain = 0, int planes = 2) {
  if (img != nullptr && tc_on(chain) && tc_shape_ok(N, K))
    return planes == 3 ? tc::gemm_w<3>(A, lda, M, N, (int)K, img, epi, st) : tc::gemm_w<2>(A, lda, M, N, (int)K, img, epi, st);
  return gemm_simt<true, true, Epi>(A, lda, W, ldw, M, N, K, epi, st, 1);
}
template <class Epi>
static inline int gemm_nn(const float* A, int64_t lda, const float* W, int64_t ldw, int64_t M, int N, int64_t K,
                          const Epi& epi, cudaStream_t st, const uint16_t* img = nullptr, int chain = 0) {
  if (img != nullptr && tc_on(chain) && tc_shape_ok(N, K))
    return tc::gemm_w<2>(A, lda, M, N, (int)K, img, epi, st);
  return gemm_simt<true, false, Epi>(A, lda, W, ldw, M, N, K, epi, st, 1);
}
// C[M x N] += A[K x M]^T B[K x N]   (contraction over points)
int colsum(const float* X, int64_t ldx, const float* w, float wscale, int64_t P, int N, float* out, cudaStream_t st);

// colsum_a (optional): colsum_a[m] += sum_k A[k, m] -- the bias gradient that goes with a weight gradient; fused into the
// tensor-engine kernel's operand staging, a separate reduction kernel on the FFMA path.  Each engine picks its own split
// over the points: tc::gemm_tn from the shape (tn_k_chunk), the FFMA kernel one split per SIMT_TN_POINTS points.
constexpr int64_t SIMT_TN_POINTS = 2048;
template <class Epi>
static inline int gemm_tn(const float* A, int64_t lda, const float* B, int64_t ldb, int M, int N, int64_t K,
                          const Epi& epi, cudaStream_t st, int chain = TC_WGRAD, float* colsum_a = nullptr) {
  if (tc_on(chain) && M >= 32 && N >= 32 && K >= 128) return tc::gemm_tn(A, lda, B, ldb, M, N, K, epi, st, colsum_a);
  if (int rc = gemm_simt<false, false, Epi>(A, lda, B, ldb, M, N, K, epi, st, (int)cdiv(K, SIMT_TN_POINTS))) return rc;
  if (colsum_a != nullptr) return colsum(A, lda, nullptr, 1.f, K, M, colsum_a, st);
  return 0;
}

}  // namespace nudf

// Stand-alone entry points of the tensor-core engine (unit-tested on the GPU against fp64 matmuls before it is trusted
// inside the network chains): weight-image preparation, one dense layer, one weight-gradient contraction.
#include "../../include/nudf.h"
#include "common.cuh"
#include "gemm_engine.cuh"

using namespace nudf;

extern "C" {

int64_t nudf_tc_image_elems(int32_t N, int32_t K, int32_t planes) { return tc::image_elems(N, K, planes == 3 ? 3 : 2); }

int nudf_tc_prepare_weights(const float* W, int64_t ldw, int32_t N, int32_t K, int32_t transposed, int32_t planes,
                            uint16_t* img, void* stream) {
  NUDF_REQUIRE(W && img, "null pointer");
  NUDF_REQUIRE((reinterpret_cast<uintptr_t>(img) & 15) == 0, "image must be 16-byte aligned");
  NUDF_REQUIRE(planes == 2 || planes == 3, "planes must be 2 or 3");
  return tc::prep_weights(W, ldw, N, K, transposed, planes, img, (cudaStream_t)stream);
}

int nudf_dense_forward_tc(const float* X, int64_t ldx, const uint16_t* img, int32_t planes, const float* bias, float* Y,
                          int64_t ldy, int64_t M, int32_t N, int32_t K, int32_t act, void* stream) {
  NUDF_REQUIRE(X && img && Y, "null pointer");
  NUDF_REQUIRE(act >= 0 && act <= 3, "bad act");
  EpiAct e{Y, ldy, bias, act, 1.0f};
  NUDF_REQUIRE(planes == 2 || planes == 3, "planes must be 2 or 3");
  if (planes == 3) return tc::gemm_w<3>(X, ldx, M, N, K, img, e, (cudaStream_t)stream);
  return tc::gemm_w<2>(X, ldx, M, N, K, img, e, (cudaStream_t)stream);
}

// dW[n_out, n_in] += dZ[P, n_out]^T X[P, n_in];  engine 0 = fp32 FFMA, 1 = tensor cores (wgmma)
int nudf_wgrad(const float* dZ, int64_t ldz, const float* X, int64_t ldx, int32_t n_out, int32_t n_in, int64_t P, float* dW,
               int64_t ldw, int32_t engine, void* stream) {
  NUDF_REQUIRE(dZ && X && dW, "null pointer");
  EpiAtomicAdd e{dW, ldw};
  // the same partition over the points as inside the networks' backward passes (gemm_engine.cuh)
  if (engine == 1) return tc::gemm_tn(dZ, ldz, X, ldx, n_out, n_in, P, e, (cudaStream_t)stream);
  return gemm_simt<false, false, EpiAtomicAdd>(dZ, ldz, X, ldx, n_out, n_in, P, e, (cudaStream_t)stream, (int)cdiv(P, SIMT_TN_POINTS));
}

}  // extern "C"

// Stand-alone entry points of the tensor-core engine (unit-tested on the GPU against fp64 matmuls before it is trusted
// inside the network chains): weight-image preparation, one dense layer, one weight-gradient contraction.
#include "../../include/nudf.h"
#include "common.cuh"
#include "ew_kernels.cuh"
#include "gemm_engine.cuh"

using namespace nudf;

namespace {
// A [rows x width] operand as the tensor-core kernels read it (tc::tma_operand_ok): the caller's, or a copy with stride
// round_up(width, 4) in a temporary taken on the stream and freed on it when this goes out of scope.  The kernels' tensor
// maps stop at the width, so the padding columns are never read and the result has the bits of an aligned operand.
struct TmaOperand {
  const float* p = nullptr;
  int64_t ld = 0;
  float* tmp = nullptr;
  cudaStream_t st;
  explicit TmaOperand(cudaStream_t s) : st(s) {}
  ~TmaOperand() { if (tmp != nullptr) cudaFreeAsync(tmp, st); }
  int init(const float* X, int64_t ldx, int64_t rows, int width) {
    p = X; ld = ldx;
    if (tc::tma_operand_ok(X, ldx) || rows <= 0) return 0;
    ld = round_up(width > 0 ? width : 1, 4);
    NUDF_CUDA_OK(cudaMallocAsync(reinterpret_cast<void**>(&tmp), sizeof(float) * rows * ld, st));
    p = tmp;
    if (width > 0) {
      ew_copy_cols_kernel<<<ew_blocks(rows * width, 256), 256, 0, st>>>(X, ldx, tmp, ld, 0, width, rows, 1.f);
      NUDF_LAUNCH_OK();
    }
    return 0;
  }
};
}  // namespace

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
  NUDF_REQUIRE(planes == 2 || planes == 3, "planes must be 2 or 3");
  EpiAct e{Y, ldy, bias, act, 1.0f};
  cudaStream_t st = (cudaStream_t)stream;
  TmaOperand x(st);
  if (int rc = x.init(X, ldx, M, K)) return rc;
  // K = 0 gives act(bias) on either plane count; the 2-plane kernel issues no copy then, the 3-plane kernel needs K > 0
  if (planes == 3 && K > 0) return tc::gemm_w<3>(x.p, x.ld, M, N, K, img, e, st);
  return tc::gemm_w<2>(x.p, x.ld, M, N, K, img, e, st);
}

// dW[n_out, n_in] += dZ[P, n_out]^T X[P, n_in];  engine 0 = fp32 FFMA, 1 = tensor cores (wgmma)
int nudf_wgrad(const float* dZ, int64_t ldz, const float* X, int64_t ldx, int32_t n_out, int32_t n_in, int64_t P, float* dW,
               int64_t ldw, int32_t engine, void* stream) {
  NUDF_REQUIRE(dZ && X && dW, "null pointer");
  EpiAtomicAdd e{dW, ldw};
  // the same partition over the points as inside the networks' backward passes (gemm_engine.cuh)
  if (engine == 1) {
    cudaStream_t st = (cudaStream_t)stream;
    TmaOperand z(st), x(st);
    if (int rc = z.init(dZ, ldz, P, n_out)) return rc;
    if (int rc = x.init(X, ldx, P, n_in)) return rc;
    return tc::gemm_tn(z.p, z.ld, x.p, x.ld, n_out, n_in, P, e, st);
  }
  return gemm_simt<false, false, EpiAtomicAdd>(dZ, ldz, X, ldx, n_out, n_in, P, e, (cudaStream_t)stream, (int)cdiv(P, SIMT_TN_POINTS));
}

}  // extern "C"

// UDFNetwork: forward value chain, exact input-gradient (reverse sweep), and the first+second order
// parameter gradients (tangent chain + backward chain + weight-gradient contractions).
// Reference semantics: models/fields.py:115-231 (forward :192-211, gradient :219-231); maths: SURVEY.md App. A and
// tests/proto/udf_pipeline.py (the torch prototype of exactly this sequence, checked against autograd).
#include "../../include/nudf.h"
#include "common.cuh"
#include "ew_kernels.cuh"
#include "dense_layer.cuh"
#include <string.h>

namespace nudf {

struct UdfPlan {
  int n_lin, d_in, L, d_pe, d_out, skip;
  float scale;
  // the n_lin layers, then the feature rows 1.. of the last one as an operand of their own: its udf-head row 0 stays an exact-fp32
  // dot product in the value chain (udf_head_kernel) and a rank-1 update in the backward chain (EpiBwdR1)
  DenseLayer layer[NUDF_MAX_LAYERS + 1];
  int64_t w_total, b_total, img_total;   // fp32 folded weights, biases, uint16 elements of the bf16 weight images
  int pe_ld, y_ld;
  int a_ld[NUDF_MAX_LAYERS];    // ld of A[l] (input of layer l), l >= 1
  int o_ld[NUDF_MAX_LAYERS];    // ld of D[l] / Q[l] (out_dim rounded)
  int max_ld;
};

// wfold (optional): the folded buffer the layers' weights and images are read from
static int make_plan(const nudf_udf_desc* d, UdfPlan* p, const float* wfold = nullptr) {
  NUDF_REQUIRE(d != nullptr, "null desc");
  NUDF_REQUIRE(d->n_lin >= 2 && d->n_lin <= NUDF_MAX_LAYERS, "n_lin out of range");
  NUDF_REQUIRE(d->d_in == 3, "d_in must be 3");
  NUDF_REQUIRE(d->multires >= 0 && d->multires <= 16, "multires out of range");
  p->n_lin = d->n_lin; p->d_in = d->d_in; p->L = d->multires; p->d_out = d->d_out; p->skip = d->skip_layer;
  p->scale = d->scale;
  p->d_pe = d->d_in * (1 + 2 * d->multires);
  NUDF_REQUIRE(p->skip < 0 || (p->skip >= 1 && p->skip <= p->n_lin - 1), "skip_layer out of range");
  int64_t off = 0, boff = 0;
  p->max_ld = 0;
  for (int l = 0; l < p->n_lin; ++l) {
    DenseLayer& L = p->layer[l];
    L.n_in = d->in_dim[l]; L.n_out = d->out_dim[l]; L.bias = d->bias[l];
    NUDF_REQUIRE(L.n_in > 0 && L.n_out > 0, "bad layer dims");
    L.ldw = round_up(L.n_in, 4);
    L.w_off = off; off += (int64_t)L.n_out * L.ldw;
    off = round_up(off, 4);
    L.b_off = boff; boff += L.n_out;
    p->a_ld[l] = (int)round_up(L.n_in, 8);        // the fused chains move 8-column octets: whole octets stay inside a tensor
    p->o_ld[l] = (int)round_up(L.n_out, 8);
    if (p->a_ld[l] > p->max_ld) p->max_ld = p->a_ld[l];
    if (p->o_ld[l] > p->max_ld) p->max_ld = p->o_ld[l];
  }
  p->w_total = off; p->b_total = boff;
  const int last = p->n_lin - 1;
  DenseLayer& F = p->layer[p->n_lin];
  F = p->layer[last];
  F.n_out = p->d_out - 1; F.w_off += F.ldw; F.b_off += 1;
  if (F.bias != nullptr) F.bias += 1;
  // hidden layers: value chain (3 planes), tangent chain, reverse / backward chains.  The tangent chain stops below the last layer,
  // whose whole-matrix dY W image serves the backward chain when the head is not split off; the feature rows serve the value
  // chain and the split backward (none when d_out == 1: plan_images drops the empty shape)
  int64_t ioff = 0;
  for (int l = 0; l < last; ++l) ioff = plan_images(p->layer[l], 1 << IMG_NT2 | 1 << IMG_NT3 | 1 << IMG_NN2, ioff);
  ioff = plan_images(p->layer[last], 1 << IMG_NN2, ioff);
  ioff = plan_images(F, 1 << IMG_NT3 | 1 << IMG_NN2, ioff);
  p->img_total = round_up(ioff, 8);
  bind_layers(p->layer, p->n_lin + 1, wfold, p->w_total);
  NUDF_REQUIRE(p->layer[0].n_in == p->d_pe, "in_dim[0] must equal the positional-encoding width");
  NUDF_REQUIRE(p->layer[last].n_out == p->d_out, "last layer width must equal d_out");
  for (int l = 1; l < p->n_lin; ++l) {
    int expect = p->layer[l - 1].n_out + (l == p->skip ? p->d_pe : 0);
    NUDF_REQUIRE(p->layer[l].n_in == expect, "layer dims are not chained consistently");
  }
  p->pe_ld = (int)round_up(p->d_pe, 8);
  p->y_ld = (int)round_up(p->d_out, 8);
  return 0;
}

// ---- context / scratch layout (all offsets in floats; every block starts 16B-aligned) -------------------------
struct UdfCtx {
  int64_t e0, a[NUDF_MAX_LAYERS], y, sgn, d[NUDF_MAX_LAYERS], gpe, ge, total;
};
static void ctx_layout(const UdfPlan& p, int64_t P, int with_grad, UdfCtx* c) {
  Bump b;
  c->e0 = b.take(P * p.pe_ld);
  for (int l = 1; l < p.n_lin; ++l) c->a[l] = b.take(P * p.a_ld[l]);
  c->y = b.take(P * p.y_ld);
  c->sgn = b.take(P);
  if (with_grad) {
    for (int l = 0; l < p.n_lin - 1; ++l) c->d[l] = b.take(P * p.o_ld[l]);
    c->gpe = b.take(P * p.pe_ld);
    c->ge = b.take(P * p.pe_ld);
  }
  c->total = b.off;
}
struct UdfScratch {
  int64_t edot, adot[2], q[NUDF_MAX_LAYERS], zlast, total;
};
static void scratch_layout(const UdfPlan& p, int64_t P, UdfScratch* s) {
  Bump b;
  s->edot = b.take(P * p.pe_ld);
  s->adot[0] = b.take(P * p.max_ld);
  s->adot[1] = b.take(P * p.max_ld);
  for (int l = 0; l < p.n_lin - 1; ++l) s->q[l] = b.take(P * p.o_ld[l]);
  s->zlast = b.take(P * p.y_ld);
  s->total = b.off;
}

// ---- element-wise kernels ---------------------------------------------------------------------------------------

// E0 = PE(x*scale) [P, pe_ld]; optionally also E0/sqrt2 into the skip columns of A[skip].
__global__ void pe_forward_kernel(const float* __restrict__ pts, int64_t P, int L, float scale, float* __restrict__ e0,
                                  int pe_ld, float* __restrict__ askip, int askip_ld, int askip_col) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  float x[3] = {pts[i * 3 + 0] * scale, pts[i * 3 + 1] * scale, pts[i * 3 + 2] * scale};
  float* e = e0 + i * pe_ld;
  float* a = askip ? askip + i * askip_ld + askip_col : nullptr;
  int d_pe = 3 * (1 + 2 * L);
#pragma unroll
  for (int c = 0; c < 3; ++c) { e[c] = x[c]; if (a) a[c] = x[c] * NUDF_SQRT1_2; }
  float f = 1.0f;
  for (int k = 0; k < L; ++k) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float s, co;
      sincosf(x[c] * f, &s, &co);
      e[3 + 6 * k + c] = s; e[3 + 6 * k + 3 + c] = co;
      if (a) { a[3 + 6 * k + c] = s * NUDF_SQRT1_2; a[3 + 6 * k + 3 + c] = co * NUDF_SQRT1_2; }
    }
    f *= 2.0f;
  }
  for (int c = d_pe; c < pe_ld; ++c) e[c] = 0.f;
}

// out = cat(|y0|/scale, y[1:]); sgn = sign(y0)
// y [P, y_ld] -> udf[row * ld_u] = |y0| / scale, feat[row * ld_f + j] = y[1 + j]  (the classic [P, 1 + F] tensor is udf = out,
// feat = out + 1, ld_u = ld_f = ld_out); sgn <- sign(y0)
__global__ void udf_finalize_kernel(const float* __restrict__ y, int y_ld, int d_out, int64_t P, float inv_scale,
                                    float* __restrict__ udf, int64_t ld_u, float* __restrict__ feat, int64_t ld_f, float* __restrict__ sgn) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t row = idx / d_out;
  int c = (int)(idx - row * d_out);
  if (row >= P) return;
  float v = y[row * y_ld + c];
  if (c == 0) {
    if (sgn) sgn[row] = (v > 0.f) ? 1.f : ((v < 0.f) ? -1.f : 0.f);
    if (udf) udf[row * ld_u] = fabsf(v) * inv_scale;
  } else if (feat) {
    feat[row * ld_f + c - 1] = v;
  }
}
// udf head: y[row * y_ld] = A[row, :K] . w0 + b0, exact fp32 (it feeds exp(-25000 u)); one warp per point, lane j sums
// k = j, j + 32, ... and a fixed butterfly adds the lanes, so a point gets the same bits in any batch and position
__global__ void udf_head_kernel(const float* __restrict__ A, int64_t lda, const float* __restrict__ w0, const float* __restrict__ b0,
                                int K, int64_t P, float* __restrict__ y, int y_ld) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= P) return;
  const float* a = A + row * lda;
  float s = 0.f;
#pragma unroll 8
  for (int k = lane; k < K; k += 32) s = fmaf(a[k], w0[k], s);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if (lane == 0) y[row * y_ld] = s + (b0 != nullptr ? b0[0] : 0.f);
}

__global__ void udf_value_only_kernel(const float* __restrict__ y, int y_ld, int64_t P, float inv_scale, float* __restrict__ udf) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < P) udf[i] = fabsf(y[i * y_ld]) * inv_scale;
}

// Reverse-sweep seed: G = (sgn/scale) W_last[0,:]  -> D[n_lin-2] (and Gpe when the last layer is the skip layer).
template <class Epi>
__global__ void rev_init_kernel(const float* __restrict__ sgn, const float* __restrict__ wlast_row0, int in_last,
                                float inv_scale, int64_t P, Epi epi) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int cols4 = (in_last + 3) / 4;
  int64_t row = idx / cols4;
  int c = (int)(idx - row * cols4) * 4;
  if (row >= P) return;
  float s = sgn[row] * inv_scale;
  float v[4];
  int nv = in_last - c < 4 ? in_last - c : 4;
#pragma unroll
  for (int j = 0; j < 4; ++j) v[j] = j < nv ? s * wlast_row0[c + j] : 0.f;
  epi(row, c, v, nv);
}

// grad_x = scale * J_e(x)^T Ge
__global__ void pe_vjp_kernel(const float* __restrict__ pts, const float* __restrict__ ge, int pe_ld, int64_t P, int L,
                              float scale, float* __restrict__ grad) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  float g[3 * (1 + 2 * 16)];
  const int d_pe_ = 3 * (1 + 2 * L);
  for (int c = 0; c < d_pe_; ++c) g[c] = ge[i * pe_ld + c];
  float f = 1.0f;
  float acc[3] = {g[0], g[1], g[2]};
  float x[3] = {pts[i * 3 + 0] * scale, pts[i * 3 + 1] * scale, pts[i * 3 + 2] * scale};
  for (int k = 0; k < L; ++k) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float s, co;
      sincosf(x[c] * f, &s, &co);
      acc[c] += f * (co * g[3 + 6 * k + c] - s * g[3 + 6 * k + 3 + c]);
    }
    f *= 2.0f;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) grad[i * 3 + c] = acc[c] * scale;
}

// Edot = scale * J_e(x) gbar  [P, pe_ld]
__global__ void pe_jvp_kernel(const float* __restrict__ pts, const float* __restrict__ gbar, int64_t P, int L, float scale,
                              float* __restrict__ edot, int pe_ld) {
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  float* e = edot + i * pe_ld;
  float x[3] = {pts[i * 3 + 0] * scale, pts[i * 3 + 1] * scale, pts[i * 3 + 2] * scale};
  float v[3] = {gbar[i * 3 + 0] * scale, gbar[i * 3 + 1] * scale, gbar[i * 3 + 2] * scale};
  int d_pe = 3 * (1 + 2 * L);
#pragma unroll
  for (int c = 0; c < 3; ++c) e[c] = v[c];
  float f = 1.0f;
  for (int k = 0; k < L; ++k) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float s, co;
      sincosf(x[c] * f, &s, &co);
      e[3 + 6 * k + c] = f * co * v[c];
      e[3 + 6 * k + 3 + c] = -f * s * v[c];
    }
    f *= 2.0f;
  }
  for (int c = d_pe; c < pe_ld; ++c) e[c] = 0.f;
}

// out[c] (+)= sum_rows w[row] * X[row, c]   (w may be null = 1).  grid: (col tiles of 32, row chunks).  With several row
// chunks each block stores its partial sum into part[chunk][c] and colsum() adds the chunks in order (same bits every run).
__global__ void weighted_colsum_kernel(const float* __restrict__ X, int64_t ldx, const float* __restrict__ w, float wscale,
                                       int64_t P, int N, int64_t rows_per_block, float* __restrict__ out, float* __restrict__ part) {
  int c = blockIdx.x * 32 + (threadIdx.x & 31);
  int ry = threadIdx.x >> 5;  // 0..7
  int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
  int64_t r1 = r0 + rows_per_block < P ? r0 + rows_per_block : P;
  float acc = 0.f;
  if (c < N)
    for (int64_t r = r0 + ry; r < r1; r += 8) acc += (w ? w[r] * wscale : 1.f) * X[r * ldx + c];
  __shared__ float red[8][33];
  red[ry][threadIdx.x & 31] = acc;
  __syncthreads();
  if (ry == 0 && c < N) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += red[k][threadIdx.x & 31];
    if (part != nullptr) part[(int64_t)blockIdx.y * N + c] = t;
    else out[c] += t;
  }
}

int colsum(const float* X, int64_t ldx, const float* w, float wscale, int64_t P, int N, float* out, cudaStream_t st) {
  if (P <= 0 || N <= 0) return 0;
  int64_t rpb = 512;
  while (cdiv(P, rpb) * N > SPLIT_WS_FLOATS) rpb *= 2;
  const int chunks = (int)cdiv(P, rpb);
  float* part = nullptr;
  if (chunks > 1 && (part = split_workspace(st)) == nullptr) return -2;
  dim3 grid((unsigned)cdiv(N, 32), (unsigned)chunks);
  weighted_colsum_kernel<<<grid, 256, 0, st>>>(X, ldx, w, wscale, P, N, rpb, out, part);
  NUDF_LAUNCH_OK();
  return part != nullptr ? vec_reduce(part, chunks, N, out, st) : 0;
}

// Zlast[:,0] = sgn * ob[:,0] / scale ; Zlast[:,1:] = ob[:,1:]
__global__ void zlast_kernel(const float* __restrict__ ub, int64_t ld_ub, const float* __restrict__ fb, int64_t ld_fb,
                             const float* __restrict__ sgn, float inv_scale, int d_out, int y_ld, int64_t P, float* __restrict__ z) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t row = idx / y_ld;
  int c = (int)(idx - row * y_ld);
  if (row >= P) return;
  float v = 0.f;
  if (c == 0) v = ub ? ub[row * ld_ub] * sgn[row] * inv_scale : 0.f;
  else if (c < d_out) v = fb ? fb[row * ld_fb + c - 1] : 0.f;
  z[row * y_ld + c] = v;
}

// Upstream gradient of the last layer, split: zf[:, j] = feat_bar[:, j] (features, ld = F) and z0 = sgn * udf_bar / scale (udf head);
// a null pointer stands for a zero gradient
__global__ void zlast_split_kernel(const float* __restrict__ ub, int64_t ld_ub, const float* __restrict__ fb, int64_t ld_fb,
                                   const float* __restrict__ sgn, float inv_scale, int F, int64_t P, float* __restrict__ zf,
                                   float* __restrict__ z0) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t row = idx / (F + 1);
  int c = (int)(idx - row * (F + 1));
  if (row >= P) return;
  if (c == 0) z0[row] = ub ? ub[row * ld_ub] * sgn[row] * inv_scale : 0.f;
  else zf[row * F + c - 1] = fb ? fb[row * ld_fb + c - 1] : 0.f;
}

static inline unsigned nblk(int64_t n, int t) { return (unsigned)cdiv(n, t); }

// ---- host orchestration -----------------------------------------------------------------------------------------

static int fold_all(const UdfPlan& p, const nudf_udf_desc* d, float* wfold, cudaStream_t st) {
  FoldJobs jobs;
  jobs.n = 0;
  for (int l = 0; l < p.n_lin; ++l) add_fold_job(jobs, p.layer[l], d->weight_g[l], d->weight_v[l], wfold);
  if (int rc = run_fold_jobs(jobs, false, st)) return rc;
  if (get_engine() != 1) return 0;
  // split-bf16 images of the tensor-core layer kernels (gemm_tc.cuh), all in one launch; the 3-plane ones only when the value
  // chain runs there
  tc::PrepWJobs pj;
  pj.n = 0;
  const int kinds = 1 << IMG_NT2 | 1 << IMG_NN2 | (tc_on(TC_FWD) ? 1 << IMG_NT3 : 0);
  for (int l = 0; l <= p.n_lin; ++l) add_prep_jobs(pj, p.layer[l], reinterpret_cast<uint16_t*>(wfold + p.w_total), kinds);
  return tc::prep_weights_jobs(pj, st);
}

// Y[:, 0] (udf head) and, with `features`, Y[:, 1:] of the last layer, with every layer's input saved in the context
static int value_chain(const UdfPlan& p, const float* pts, int64_t P, float* ctx, const UdfCtx& c, bool features, cudaStream_t st) {
  float* e0 = ctx + c.e0;
  float* askip = nullptr; int askip_ld = 0, askip_col = 0;
  if (p.skip >= 1) { askip = ctx + c.a[p.skip]; askip_ld = p.a_ld[p.skip]; askip_col = p.layer[p.skip - 1].n_out; }
  pe_forward_kernel<<<nblk(P, 128), 128, 0, st>>>(pts, P, p.L, p.scale, e0, p.pe_ld, askip, askip_ld, askip_col);
  NUDF_LAUNCH_OK();
  const int last = p.n_lin - 1;
  for (int l = 0; l < last; ++l) {
    const float* A = l == 0 ? e0 : ctx + c.a[l];
    int64_t lda = l == 0 ? p.pe_ld : p.a_ld[l];
    EpiAct epi{ctx + c.a[l + 1], p.a_ld[l + 1], p.layer[l].bias, ACT_SOFTPLUS100, (l + 1 == p.skip) ? NUDF_SQRT1_2 : 1.0f};
    if (int rc = layer_nt(p.layer[l], A, lda, P, epi, TC_FWD, st)) return rc;
  }
  const float* A = ctx + c.a[last];
  const DenseLayer& Ll = p.layer[last];
  udf_head_kernel<<<nblk(P * 32, 256), 256, 0, st>>>(A, p.a_ld[last], Ll.W, Ll.bias, Ll.n_in, P, ctx + c.y, p.y_ld);
  NUDF_LAUNCH_OK();
  if (features && p.d_out > 1) {
    const DenseLayer& Lf = p.layer[p.n_lin];
    EpiAct epi{ctx + c.y + 1, p.y_ld, Lf.bias, ACT_NONE, 1.0f};      // unaligned columns: st4 stores them one by one
    if (int rc = layer_nt(Lf, A, p.a_ld[last], P, epi, TC_FWD, st)) return rc;
  }
  return 0;
}

static int reverse_chain(const UdfPlan& p, const float* pts, int64_t P, float* ctx, const UdfCtx& c, float* grad, cudaStream_t st) {
  const int last = p.n_lin - 1;
  auto make_rev = [&](int l) {  // epilogue that turns G (wrt A[l]) into D[l-1]
    EpiRev e;
    e.n_main = p.layer[l - 1].n_out;
    e.post_scale = (l == p.skip) ? NUDF_SQRT1_2 : 1.0f;
    e.Anext = ctx + c.a[l]; e.lda = p.a_ld[l]; e.a_unscale = (l == p.skip) ? 1.41421356237309504880f : 1.0f;
    e.Dprev = ctx + c.d[l - 1]; e.ldd = p.o_ld[l - 1];
    e.Gpe = (l == p.skip) ? ctx + c.gpe : nullptr; e.ldg = p.pe_ld;
    return e;
  };
  {
    EpiRev e = make_rev(last);
    const int in_last = p.layer[last].n_in;
    int cols4 = (in_last + 3) / 4;
    rev_init_kernel<EpiRev><<<nblk(P * cols4, 256), 256, 0, st>>>(ctx + c.sgn, p.layer[last].W, in_last, 1.0f / p.scale, P, e);
    NUDF_LAUNCH_OK();
  }
  for (int l = last - 1; l >= 1; --l) {
    EpiRev e = make_rev(l);
    if (int rc = layer_nn(p.layer[l], ctx + c.d[l], p.o_ld[l], P, e, TC_REV, st)) return rc;
  }
  {
    EpiRevFinal e{ctx + c.ge, p.pe_ld, p.skip >= 1 ? ctx + c.gpe : nullptr, p.pe_ld};
    if (int rc = layer_nn(p.layer[0], ctx + c.d[0], p.o_ld[0], P, e, TC_REV, st)) return rc;
  }
  pe_vjp_kernel<<<nblk(P, 128), 128, 0, st>>>(pts, ctx + c.ge, p.pe_ld, P, p.L, p.scale, grad);
  NUDF_LAUNCH_OK();
  return 0;
}

}  // namespace nudf

using namespace nudf;

extern "C" {

int64_t nudf_udf_folded_floats(const nudf_udf_desc* d) {
  UdfPlan p;
  if (make_plan(d, &p)) return -1;
  return p.w_total + p.img_total / 2;   // fp32 folded weights, then the 16-bit weight images (2 per float)
}

int nudf_udf_fold_weights(const nudf_udf_desc* d, float* wfold, void* stream) {
  UdfPlan p;
  if (int rc = make_plan(d, &p, wfold)) return rc;
  NUDF_REQUIRE(wfold != nullptr, "null wfold");
  cudaStream_t st = (cudaStream_t)stream;
  return fold_all(p, d, wfold, st);
}

int64_t nudf_udf_ctx_floats(const nudf_udf_desc* d, int64_t P, int with_grad) {
  UdfPlan p;
  if (make_plan(d, &p)) return -1;
  UdfCtx c;
  ctx_layout(p, P, with_grad, &c);
  return c.total;
}

int64_t nudf_udf_scratch_floats(const nudf_udf_desc* d, int64_t P) {
  UdfPlan p;
  if (make_plan(d, &p)) return -1;
  UdfScratch s;
  scratch_layout(p, P, &s);
  return s.total;
}

static int udf_forward_impl(const nudf_udf_desc* d, const float* wfold, const float* pts, int64_t P, float* udf, int64_t ld_u, float* feat,
                            int64_t ld_f, float* grad, float* ctx, void* stream) {
  UdfPlan p;
  if (int rc = make_plan(d, &p, wfold)) return rc;
  if (P <= 0) return 0;
  NUDF_REQUIRE(wfold && pts && ctx, "null pointer");
  NUDF_REQUIRE(aligned16(ctx), "ctx must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  UdfCtx c;
  ctx_layout(p, P, grad != nullptr, &c);
  if (int rc = value_chain(p, pts, P, ctx, c, feat != nullptr, st)) return rc;
  udf_finalize_kernel<<<nblk(P * p.d_out, 256), 256, 0, st>>>(ctx + c.y, p.y_ld, p.d_out, P, 1.0f / p.scale, udf, ld_u, feat, ld_f,
                                                              ctx + c.sgn);
  NUDF_LAUNCH_OK();
  if (grad) return reverse_chain(p, pts, P, ctx, c, grad, st);
  return 0;
}

int nudf_udf_forward(const nudf_udf_desc* d, const float* wfold, const float* pts, int64_t P, float* out, int64_t ld_out,
                     float* grad, float* ctx, void* stream) {
  NUDF_REQUIRE(d != nullptr, "null descriptor");
  NUDF_REQUIRE(out == nullptr || ld_out >= d->d_out, "ld_out too small");
  return udf_forward_impl(d, wfold, pts, P, out, ld_out, out ? out + 1 : nullptr, ld_out, grad, ctx, stream);
}

int nudf_udf_forward_split(const nudf_udf_desc* d, const float* wfold, const float* pts, int64_t P, float* udf, float* feat,
                           int64_t ld_feat, float* grad, float* ctx, void* stream) {
  NUDF_REQUIRE(d != nullptr, "null descriptor");
  NUDF_REQUIRE(feat == nullptr || ld_feat >= d->d_out - 1, "ld_feat too small");
  return udf_forward_impl(d, wfold, pts, P, udf, 1, feat, ld_feat, grad, ctx, stream);
}

int nudf_udf_value(const nudf_udf_desc* d, const float* wfold, const float* pts, int64_t P, float* udf, float* work,
                   void* stream) {
  UdfPlan p;
  if (int rc = make_plan(d, &p, wfold)) return rc;
  if (P <= 0) return 0;
  NUDF_REQUIRE(wfold && pts && udf, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  NUDF_REQUIRE(work != nullptr, "null pointer (work)");
  NUDF_REQUIRE(aligned16(work), "work must be 16-byte aligned");
  UdfCtx c;
  ctx_layout(p, P, 0, &c);
  // value-only: of the last layer only row 0 (the udf head), through the same kernel as the full forward
  if (int rc = value_chain(p, pts, P, work, c, false, st)) return rc;
  udf_value_only_kernel<<<nblk(P, 256), 256, 0, st>>>(work + c.y, p.y_ld, P, 1.0f / p.scale, udf);
  NUDF_LAUNCH_OK();
  return 0;
}

static int udf_backward_impl(const nudf_udf_desc* d, const float* wfold, const float* pts, int64_t P, const float* ub, int64_t ld_ub,
                             const float* fb, int64_t ld_fb, const float* grad_bar, const float* ctx_c, float* scratch, float* dwfold,
                             float* dbias, void* stream);

int nudf_udf_backward(const nudf_udf_desc* d, const float* wfold, const float* pts, int64_t P, const float* out_bar,
                      int64_t ld_ob, const float* grad_bar, const float* ctx_c, float* scratch, float* dwfold,
                      float* dbias, void* stream) {
  return udf_backward_impl(d, wfold, pts, P, out_bar, ld_ob, out_bar ? out_bar + 1 : nullptr, ld_ob, grad_bar, ctx_c, scratch, dwfold, dbias,
                           stream);
}

int nudf_udf_backward_split(const nudf_udf_desc* d, const float* wfold, const float* pts, int64_t P, const float* udf_bar,
                            const float* feat_bar, int64_t ld_fb, const float* grad_bar, const float* ctx_c, float* scratch,
                            float* dwfold, float* dbias, void* stream) {
  return udf_backward_impl(d, wfold, pts, P, udf_bar, 1, feat_bar, ld_fb, grad_bar, ctx_c, scratch, dwfold, dbias, stream);
}

static int udf_backward_impl(const nudf_udf_desc* d, const float* wfold, const float* pts, int64_t P, const float* ub, int64_t ld_ub,
                             const float* fb, int64_t ld_fb, const float* grad_bar, const float* ctx_c, float* scratch, float* dwfold,
                             float* dbias, void* stream) {
  const bool out_bar = ub != nullptr || fb != nullptr;      // some upstream gradient of the value / feature outputs
  UdfPlan p;
  if (int rc = make_plan(d, &p, wfold)) return rc;
  NUDF_REQUIRE(wfold && dwfold && dbias, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  NUDF_CUDA_OK(cudaMemsetAsync(dwfold, 0, sizeof(float) * p.w_total, st));
  NUDF_CUDA_OK(cudaMemsetAsync(dbias, 0, sizeof(float) * p.b_total, st));
  if (P <= 0) return 0;
  NUDF_REQUIRE(pts && ctx_c && scratch, "null pointer");
  NUDF_REQUIRE(aligned16(ctx_c) && aligned16(scratch), "ctx and scratch must be 16-byte aligned");
  float* ctx = const_cast<float*>(ctx_c);  // read-only use
  UdfCtx c;
  ctx_layout(p, P, 1, &c);
  UdfScratch s;
  scratch_layout(p, P, &s);
  const int last = p.n_lin - 1;
  const DenseLayer& Ll = p.layer[last];

  // ---- tangent chain (second-order terms) ----
  if (grad_bar) {
    float* edot = scratch + s.edot;
    pe_jvp_kernel<<<nblk(P, 128), 128, 0, st>>>(pts, grad_bar, P, p.L, p.scale, edot, p.pe_ld);
    NUDF_LAUNCH_OK();
    const float* adot = edot;
    int64_t ld_adot = p.pe_ld;
    for (int l = 0; l < last; ++l) {
      const DenseLayer& L = p.layer[l];
      // dW_l += D_l^T Adot_l
      EpiAtomicAdd ew{dwfold + L.w_off, L.ldw};
      if (int rc = gemm_tn(ctx + c.d[l], p.o_ld[l], adot, ld_adot, L.n_out, L.n_in, P, ew, st)) return rc;
      float* nxt = scratch + s.adot[l & 1];
      int64_t ld_nxt = p.a_ld[l + 1];
      EpiTan et;
      et.Anext = ctx + c.a[l + 1]; et.lda = p.a_ld[l + 1];
      et.a_unscale = (l + 1 == p.skip) ? 1.41421356237309504880f : 1.0f;
      et.D = ctx + c.d[l]; et.ldd = p.o_ld[l];
      et.Q = scratch + s.q[l]; et.ldq = p.o_ld[l];
      et.AdotNext = nxt; et.ldn = ld_nxt; et.post_scale = (l + 1 == p.skip) ? NUDF_SQRT1_2 : 1.0f;
      if (int rc = layer_nt(L, adot, ld_adot, P, et, TC_TAN, st)) return rc;
      if (l + 1 == p.skip) {
        ew_copy_cols_kernel<<<nblk(P * p.d_pe, 256), 256, 0, st>>>(edot, p.pe_ld, nxt, ld_nxt, L.n_out, p.d_pe, P, NUDF_SQRT1_2);
        NUDF_LAUNCH_OK();
      }
      adot = nxt; ld_adot = ld_nxt;
    }
    // g_last = W_last^T d_last with d_last = (sgn/scale) e_0  =>  dW_last[0,:] += sum_p (sgn/scale) Adot_last
    if (int rc = colsum(adot, ld_adot, ctx + c.sgn, 1.0f / p.scale, P, Ll.n_in, dwfold + Ll.w_off, st)) return rc;
  }

  // ---- backward chain ----
  const bool has_q = grad_bar != nullptr;
  if (!has_q)
    for (int l = 0; l < last; ++l)
      NUDF_CUDA_OK(cudaMemsetAsync(scratch + s.q[l], 0, sizeof(float) * P * p.o_ld[l], st));
  float* zl = scratch + s.zlast;
  const int F = p.d_out - 1;
  // 257 = 1 udf-head row + 256 feature rows: the feature block is the K (at most 256) of a contraction on the weights-resident
  // tensor kernel, the head row a rank-1 update in its epilogue (and a weighted column sum for its weight gradient).
  const bool split_head = out_bar && tc_on(TC_BWD) && F >= 64 && (F % 4) == 0 && F <= 256;
  if (split_head) {
    const DenseLayer& Lf = p.layer[p.n_lin];
    float* zf = zl;
    float* z0 = zl + P * F;
    zlast_split_kernel<<<nblk(P * p.d_out, 256), 256, 0, st>>>(ub, ld_ub, fb, ld_fb, ctx + c.sgn, 1.0f / p.scale, F, P, zf, z0);
    NUDF_LAUNCH_OK();
    EpiAtomicAdd ew{dwfold + Lf.w_off, Lf.ldw};
    if (int rc = gemm_tn(zf, F, ctx + c.a[last], p.a_ld[last], F, Lf.n_in, P, ew, st, TC_WGRAD, dbias + Lf.b_off)) return rc;
    if (int rc = colsum(ctx + c.a[last], p.a_ld[last], z0, 1.0f, P, Ll.n_in, dwfold + Ll.w_off, st)) return rc;
    if (int rc = colsum(z0, 1, nullptr, 1.0f, P, 1, dbias + Ll.b_off, st)) return rc;
    EpiBwdR1 eb;
    eb.n_main = p.layer[last - 1].n_out; eb.post_scale = (last == p.skip) ? NUDF_SQRT1_2 : 1.0f;
    eb.Anext = ctx + c.a[last]; eb.lda = p.a_ld[last]; eb.a_unscale = (last == p.skip) ? 1.41421356237309504880f : 1.0f;
    eb.QZ = scratch + s.q[last - 1]; eb.ldq = p.o_ld[last - 1];
    eb.z0 = z0; eb.w0 = Ll.W;
    if (int rc = layer_nn(Lf, zf, F, P, eb, TC_BWD, st)) return rc;
  } else if (out_bar) {
    zlast_kernel<<<nblk(P * p.y_ld, 256), 256, 0, st>>>(ub, ld_ub, fb, ld_fb, ctx + c.sgn, 1.0f / p.scale, p.d_out, p.y_ld, P, zl);
    NUDF_LAUNCH_OK();
    EpiAtomicAdd ew{dwfold + Ll.w_off, Ll.ldw};
    if (int rc = gemm_tn(zl, p.y_ld, ctx + c.a[last], p.a_ld[last], Ll.n_out, Ll.n_in, P, ew, st, TC_WGRAD, dbias + Ll.b_off)) return rc;
    EpiBwd eb;
    eb.n_main = p.layer[last - 1].n_out; eb.post_scale = (last == p.skip) ? NUDF_SQRT1_2 : 1.0f;
    eb.Anext = ctx + c.a[last]; eb.lda = p.a_ld[last]; eb.a_unscale = (last == p.skip) ? 1.41421356237309504880f : 1.0f;
    eb.QZ = scratch + s.q[last - 1]; eb.ldq = p.o_ld[last - 1];
    if (int rc = layer_nn(Ll, zl, p.y_ld, P, eb, TC_BWD, st)) return rc;
  }
  for (int l = last - 1; l >= 0; --l) {
    const DenseLayer& L = p.layer[l];
    const float* zb = scratch + s.q[l];  // now holds Zbar_l
    const float* A = l == 0 ? ctx + c.e0 : ctx + c.a[l];
    int64_t lda = l == 0 ? p.pe_ld : p.a_ld[l];
    EpiAtomicAdd ew{dwfold + L.w_off, L.ldw};
    if (int rc = gemm_tn(zb, p.o_ld[l], A, lda, L.n_out, L.n_in, P, ew, st, TC_WGRAD, dbias + L.b_off)) return rc;
    if (l > 0) {
      EpiBwd eb;
      eb.n_main = p.layer[l - 1].n_out; eb.post_scale = (l == p.skip) ? NUDF_SQRT1_2 : 1.0f;
      eb.Anext = ctx + c.a[l]; eb.lda = p.a_ld[l]; eb.a_unscale = (l == p.skip) ? 1.41421356237309504880f : 1.0f;
      eb.QZ = scratch + s.q[l - 1]; eb.ldq = p.o_ld[l - 1];
      if (int rc = layer_nn(L, zb, p.o_ld[l], P, eb, TC_BWD, st)) return rc;
    }
  }
  return 0;
}

int nudf_udf_unfold_grads(const nudf_udf_desc* d, const float* dwfold, float* const* dg, float* const* dv, void* stream) {
  UdfPlan p;
  if (int rc = make_plan(d, &p)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  FoldJobs jobs;
  jobs.n = 0;
  for (int l = 0; l < p.n_lin; ++l) add_unfold_job(jobs, p.layer[l], d->weight_g[l], d->weight_v[l], dwfold, dg[l], dv[l]);
  return run_fold_jobs(jobs, true, st);
}

}  // extern "C"

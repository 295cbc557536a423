// ResidualRenderingNetwork ('no_normal', models/fields.py:400-495) and the NeRF++ background network
// (models/fields.py:541-628): ReLU MLPs built from the dense-layer engine (gemm_engine.cuh) with fused
// bias / activation epilogues and hand-written backward passes.
#include "../../include/nudf.h"
#include "common.cuh"
#include "ew_kernels.cuh"
#include "dense_layer.cuh"

namespace nudf {

// =================================================================================================================
// shared pieces
// =================================================================================================================

// C[row, c] = acc routed by column range: used for d(main-stack input) = [d PE(view) | d color_base | d x_hidden]
struct EpiColorMainIn {
  int c_cb, c_hid, n_total;            // column where color_base starts, where x_hidden starts, total width
  float* dcb; int64_t ld_dcb;          // [P, d_out]  gradient wrt color_base coming through the main stack
  const float* xhid; int64_t ld_xhid;  // post-ReLU x_hidden (mask)
  float* dzb; int64_t ld_dzb;          // [P, H]      masked gradient wrt the base stack's layer n_lin-2 pre-activation
  struct Aux { float h[4]; };
  __device__ __forceinline__ void load(int64_t row, int col, int nv, Aux& x) const {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int c = col + j;
      x.h[j] = (j < nv && c >= c_hid && c < n_total) ? xhid[row * ld_xhid + (c - c_hid)] : 0.f;
    }
  }
  __device__ __forceinline__ void apply(int64_t row, int col, const float acc[4], int nv, const Aux& x) const {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (j >= nv) break;
      int c = col + j;
      if (c < c_cb) continue;
      if (c < c_hid) dcb[row * ld_dcb + (c - c_cb)] = acc[j];
      else if (c < n_total) dzb[row * ld_dzb + (c - c_hid)] = (x.h[j] > 0.f) ? acc[j] : 0.f;
    }
  }
  NUDF_EPI_CALL
};

// dY = bar * s (1 - s) for the first n_sig columns (sigmoid heads), bar elsewhere; optional extra additive term
__global__ void sigmoid_head_bwd_kernel(const float* __restrict__ bar, int ld_bar, const float* __restrict__ extra,
                                        int ld_extra, const float* __restrict__ s, int ld_s, int n_sig,
                                        const float* __restrict__ bar2, int ld_bar2, int n2, int64_t P,
                                        float* __restrict__ dy, int ld_dy) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t row = idx / ld_dy;
  int c = (int)(idx - row * ld_dy);
  if (row >= P) return;
  float v = 0.f;
  if (c < n_sig) {
    float b = bar ? bar[row * ld_bar + c] : 0.f;
    if (extra) b += extra[row * ld_extra + c];
    float sv = s[row * ld_s + c];
    v = b * sv * (1.0f - sv);
  } else if (c < n_sig + n2) {
    v = bar2 ? bar2[row * ld_bar2 + (c - n_sig)] : 0.f;
  }
  dy[row * ld_dy + c] = v;
}

// color = sigmoid(ym[:, :3]); blend = ym[:, 3:]
__global__ void color_head_kernel(const float* __restrict__ ym, int ld_ym, int d_out, int n_blend, int64_t P,
                                  float* __restrict__ color, float* __restrict__ cs, int ld_cs, float* __restrict__ blend) {
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int w = d_out + n_blend;
  int64_t row = idx / w;
  int c = (int)(idx - row * w);
  if (row >= P) return;
  float v = ym[row * ld_ym + c];
  if (c < d_out) {
    float s = sigmoidf_(v);
    if (color) color[row * d_out + c] = s;
    cs[row * ld_cs + c] = s;
  } else if (blend) {
    blend[row * n_blend + (c - d_out)] = v;
  }
}

__global__ void pack_pts_feat_kernel(const float* __restrict__ pts, const float* __restrict__ feat, int64_t ld_feat, int F,
                                     int64_t P, float* __restrict__ xb, int ld_xb) {
  // one thread = 4 consecutive columns of one row (ld_xb % 4 == 0: one 16-byte store; the reads of the odd-width feature
  // tensor stay scalar but consecutive across the warp)
  const int q4 = ld_xb >> 2;
  int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  int64_t row = idx / q4;
  int c = (int)(idx - row * q4) * 4;
  if (row >= P) return;
  float v[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int cj = c + j;
    v[j] = cj < 3 ? pts[row * 3 + cj] : (cj < 3 + F ? feat[row * ld_feat + (cj - 3)] : 0.f);
  }
  *reinterpret_cast<float4*>(xb + row * ld_xb + c) = make_float4(v[0], v[1], v[2], v[3]);
}

// Forward of a narrow head (N <= 16 outputs, K <= 128: colour_base, the colour / blending-logit head): Y[p, n] = act(<X[p, :], W[n, :]> + b[n]).
// One warp per point, lanes along K (coalesced 128-byte reads of X, which may be an unaligned column window of a wider tensor); the
// weights live in registers.  Streams X once (HBM-bound) instead of padding 3..13 output columns to a 128-wide GEMM tile.
template <int MAXN>
__global__ void __launch_bounds__(256) dense_small_forward_kernel(const float* __restrict__ X, int64_t ldx, const float* __restrict__ W, int64_t ldw,
                                                                 const float* __restrict__ bias, int N, int K, int act, float post_scale,
                                                                 float* __restrict__ C, int64_t ldc, int64_t P) {
  const int lane = threadIdx.x & 31;
  const int64_t gwarp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  float w[MAXN][4];
#pragma unroll
  for (int n = 0; n < MAXN; ++n)
#pragma unroll
    for (int i = 0; i < 4; ++i) w[n][i] = (n < N && lane + 32 * i < K) ? W[(int64_t)n * ldw + lane + 32 * i] : 0.f;
  const float b = (bias != nullptr && lane < N) ? bias[lane] : 0.f;
  constexpr int R = 4;                                     // points per warp iteration: 16 independent loads in flight per lane
  for (int64_t row0 = gwarp * R; row0 < P; row0 += nwarps * R) {
    float x[R][4];
#pragma unroll
    for (int r = 0; r < R; ++r)
#pragma unroll
      for (int i = 0; i < 4; ++i) x[r][i] = (row0 + r < P && lane + 32 * i < K) ? X[(row0 + r) * ldx + lane + 32 * i] : 0.f;
    float mine[R];
#pragma unroll
    for (int r = 0; r < R; ++r) mine[r] = 0.f;
#pragma unroll
    for (int n = 0; n < MAXN; ++n) {
      if (n < N) {
        float t[R];
#pragma unroll
        for (int r = 0; r < R; ++r) t[r] = x[r][0] * w[n][0] + x[r][1] * w[n][1] + x[r][2] * w[n][2] + x[r][3] * w[n][3];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
          for (int r = 0; r < R; ++r) t[r] += __shfl_xor_sync(0xffffffffu, t[r], o);
#pragma unroll
        for (int r = 0; r < R; ++r)
          if (lane == n) mine[r] = t[r];
      }
    }
    if (lane < N) {
#pragma unroll
      for (int r = 0; r < R; ++r) {
        if (row0 + r < P) {
          float t = mine[r] + b;
          if (act == ACT_RELU) t = fmaxf(t, 0.f);
          else if (act == ACT_SOFTPLUS100) t = softplus100(t);
          else if (act == ACT_SIGMOID) t = sigmoidf_(t);
          C[(row0 + r) * ldc + lane] = t * post_scale;
        }
      }
    }
  }
}
static inline int dense_small_forward(const float* X, int64_t ldx, const float* W, int64_t ldw, int64_t P, int N, int K, const EpiAct& e,
                                      cudaStream_t st) {
  int blocks = (int)cdiv(P, 8 * 16);                         // ~16 points per warp
  if (blocks > tc::sm_count() * 8) blocks = tc::sm_count() * 8;
  if (blocks < 1) blocks = 1;
  dense_small_forward_kernel<16><<<blocks, 256, 0, st>>>(X, ldx, W, ldw, e.bias, N, K, e.act, e.post_scale, e.C, e.ldc, P);
  NUDF_LAUNCH_OK();
  return 0;
}

// Weight gradient of a narrow head (n_out <= 16: colour / density heads): dW[m, n] += sum_p dZ[p, m] X[p, n], db[m] += sum_p dZ[p, m].
// Streams X once (HBM-bound) instead of padding the 3..13 output rows to a 128-wide GEMM tile.  CTA = 128 input columns x 4
// point lanes over a point chunk; the lanes' partial sums meet in shared memory and each CTA stores its chunk's partial dW
// (and db) into the split-K workspace, summed over the chunks in order afterwards (same bits every run).
template <int MAXM>
__global__ void __launch_bounds__(512)
wgrad_small_kernel(const float* __restrict__ dZ, int64_t ldz, const float* __restrict__ X, int64_t ldx, int n_out, int n_in, int64_t P,
                   int64_t chunk, float* __restrict__ part_w, float* __restrict__ part_b) {
  const int tx = threadIdx.x & 127, ty = threadIdx.x >> 7;
  const int n = blockIdx.x * 128 + tx;
  const int64_t p0 = (int64_t)blockIdx.y * chunk;
  const int64_t p1 = p0 + chunk < P ? p0 + chunk : P;
  float acc[MAXM];
#pragma unroll
  for (int m = 0; m < MAXM; ++m) acc[m] = 0.f;
  float bs = 0.f;
  __shared__ float sdz[64][MAXM];
  __shared__ float red[3][MAXM][128];
  for (int64_t pb = p0; pb < p1; pb += 64) {
    __syncthreads();
    for (int i = threadIdx.x; i < 64 * MAXM; i += blockDim.x) {
      int r = i / MAXM, m = i - r * MAXM;
      sdz[r][m] = (pb + r < p1 && m < n_out) ? dZ[(pb + r) * ldz + m] : 0.f;
    }
    __syncthreads();
    const int cnt = (int)((p1 - pb) < 64 ? (p1 - pb) : 64);
#pragma unroll 4
    for (int r = ty; r < cnt; r += 4) {
      const float x = n < n_in ? X[(pb + r) * ldx + n] : 0.f;
#pragma unroll
      for (int m = 0; m < MAXM; ++m) acc[m] = fmaf(sdz[r][m], x, acc[m]);
    }
    if (threadIdx.x < MAXM)
      for (int r = 0; r < cnt; ++r) bs += sdz[r][threadIdx.x];
  }
  if (ty > 0) {
#pragma unroll
    for (int m = 0; m < MAXM; ++m) red[ty - 1][m][tx] = acc[m];
  }
  __syncthreads();
  if (ty == 0 && n < n_in) {
#pragma unroll
    for (int m = 0; m < MAXM; ++m)
      if (m < n_out) part_w[((int64_t)blockIdx.y * n_out + m) * n_in + n] = acc[m] + red[0][m][tx] + red[1][m][tx] + red[2][m][tx];
  }
  if (blockIdx.x == 0 && threadIdx.x < n_out) part_b[(int64_t)blockIdx.y * n_out + threadIdx.x] = bs;
}

// dW += dZ^T X, db += column sums of dZ, for the layer's shape (dW has the layer's leading dimension)
static int wgrad(const DenseLayer& L, const float* dZ, int64_t ldz, const float* X, int64_t ldx, int64_t P, float* dW, float* db,
                 cudaStream_t st) {
  const int n_out = L.n_out, n_in = L.n_in;
  if (n_out <= 16 && P > 0) {
    int64_t chunk = 256;
    while (cdiv(P, chunk) * (int64_t)n_out * (n_in + 1) > SPLIT_WS_FLOATS) chunk *= 2;
    const int chunks = (int)cdiv(P, chunk);
    float* ws = split_workspace(st);
    if (ws == nullptr) return -2;
    float* part_b = ws + (int64_t)chunks * n_out * n_in;
    dim3 grid((unsigned)cdiv(n_in, 128), (unsigned)chunks);
    wgrad_small_kernel<16><<<grid, 512, 0, st>>>(dZ, ldz, X, ldx, n_out, n_in, P, chunk, ws, part_b);
    NUDF_LAUNCH_OK();
    if (int rc = splitk_reduce(ws, chunks, n_out, n_in, EpiAtomicAdd{dW, L.ldw}, st)) return rc;
    return db != nullptr ? vec_reduce(part_b, chunks, n_out, db, st) : 0;
  }
  EpiAtomicAdd ew{dW, L.ldw};
  return gemm_tn(dZ, ldz, X, ldx, n_out, n_in, P, ew, st, TC_WGRAD, db);
}

// =================================================================================================================
// colour network
// =================================================================================================================
enum { BASE = 0, MAIN = 1 };
struct ColorPlan {
  int n_lin, F, H, d_out, n_blend, Lv, d_view;
  DenseLayer stack[2][NUDF_MAX_LAYERS];        // [BASE] and [MAIN], n_lin layers each
  int64_t w_total, b_total, img_total;
  int ld_xb, ld_xm, ld_ym, ld_h, c_cb, c_hid;   // ld_h: row stride of the hidden activations and their gradients
};

// wfold (optional): the folded buffer the layers' weights and images are read from
static int color_plan(const nudf_color_desc* d, ColorPlan* p, const float* wfold = nullptr) {
  NUDF_REQUIRE(d != nullptr, "null desc");
  NUDF_REQUIRE(d->n_lin >= 3 && d->n_lin <= NUDF_MAX_LAYERS, "n_lin out of range");
  p->n_lin = d->n_lin; p->F = d->d_feature; p->H = d->d_hidden; p->d_out = d->d_out; p->n_blend = d->n_blend;
  p->Lv = d->multires_view;
  p->d_view = 3 * (1 + 2 * p->Lv);
  NUDF_REQUIRE(p->d_out >= 1 && p->d_out <= 4, "d_out must be <= 4");
  const float* const* bias[2] = {d->base_b, d->main_b};
  int64_t off = 0, boff = 0, ioff = 0;
  for (int s = 0; s < 2; ++s)                  // folded weights and biases: the base stack's layers, then the main stack's
    for (int l = 0; l < p->n_lin; ++l) {
      DenseLayer& L = p->stack[s][l];
      L.n_in = l > 0 ? p->H : (s == BASE ? 3 + p->F : p->d_view + p->d_out + p->H);
      L.n_out = l < p->n_lin - 1 ? p->H : (s == BASE ? p->d_out : p->d_out + p->n_blend);
      L.bias = bias[s][l];
      L.ldw = round_up(L.n_in, 4);
      L.w_off = off; off = round_up(off + (int64_t)L.n_out * L.ldw, 4);
      L.b_off = boff; boff += L.n_out;
      ioff = plan_images(L, 1 << IMG_NT3 | 1 << IMG_NN2, ioff);    // forward images: 3 planes (6 products)
    }
  p->w_total = off; p->b_total = boff;
  p->img_total = round_up(ioff, 8);
  bind_layers(p->stack[BASE], p->n_lin, wfold, p->w_total);
  bind_layers(p->stack[MAIN], p->n_lin, wfold, p->w_total);
  p->ld_xb = (int)round_up(3 + p->F, 4);
  p->ld_xm = (int)round_up(p->stack[MAIN][0].n_in, 4);
  p->ld_ym = (int)round_up(p->d_out + p->n_blend, 4);
  p->ld_h = (int)round_up(p->H, 4);
  p->c_cb = p->d_view; p->c_hid = p->d_view + p->d_out;
  return 0;
}

struct ColorCtx { int64_t xb, hb[NUDF_MAX_LAYERS], xm, hm[NUDF_MAX_LAYERS], ym, cs, total; };
static void color_ctx_layout(const ColorPlan& p, int64_t P, ColorCtx* c) {
  Bump b;
  c->xb = b.take(P * p.ld_xb);
  for (int l = 1; l <= p.n_lin - 2; ++l) c->hb[l] = b.take(P * p.ld_h);   // outputs of base layers 0..n_lin-3
  c->xm = b.take(P * p.ld_xm);
  for (int l = 1; l <= p.n_lin - 1; ++l) c->hm[l] = b.take(P * p.ld_h);   // outputs of main layers 0..n_lin-2
  c->ym = b.take(P * p.ld_ym);
  c->cs = b.take(P * 4);
  c->total = b.off;
}
struct ColorScratch { int64_t buf[2], dym, dyb, dcbx, total; };
static void color_scratch_layout(const ColorPlan& p, int64_t P, ColorScratch* s) {
  Bump b;
  s->buf[0] = b.take(P * p.ld_h); s->buf[1] = b.take(P * p.ld_h);
  s->dym = b.take(P * p.ld_ym); s->dyb = b.take(P * 4); s->dcbx = b.take(P * 4);
  s->total = b.off;
}

// forward of one colour-network layer: the narrow heads (dense_small_forward_kernel) stream X once, the others are a layer GEMM
static int color_layer_forward(const DenseLayer& L, const float* X, int64_t ldx, int64_t P, const EpiAct& e, cudaStream_t st) {
  if (L.n_out <= 16 && L.n_in <= 128) return dense_small_forward(X, ldx, L.W, L.ldw, P, L.n_out, L.n_in, e, st);
  return layer_nt(L, X, ldx, P, e, TC_RELU_FWD, st);
}

}  // namespace nudf

using namespace nudf;

extern "C" {

// One dense layer Y = act(X W^T + b): the primitive every network above is built from, exported for the tests and the
// micro-benchmarks under tools/ and for callers that want a single fused layer.
int nudf_dense_forward(const float* X, int64_t ldx, const float* W, int64_t ldw, const float* bias, float* Y, int64_t ldy,
                       int64_t M, int32_t N, int32_t K, int32_t act, void* stream) {
  NUDF_REQUIRE(X && W && Y, "null pointer");
  NUDF_REQUIRE(act >= 0 && act <= 3, "act must be 0 (none), 1 (relu), 2 (softplus beta=100), 3 (sigmoid)");
  NUDF_REQUIRE(ldx >= K && ldw >= K && ldy >= N, "leading dimension too small");
  EpiAct e{Y, ldy, bias, act, 1.0f};
  return gemm_nt(X, ldx, W, ldw, M, N, K, e, (cudaStream_t)stream);
}

int64_t nudf_color_folded_floats(const nudf_color_desc* d) {
  ColorPlan p;
  if (color_plan(d, &p)) return -1;
  return p.w_total + p.img_total / 2;
}

int nudf_color_fold_weights(const nudf_color_desc* d, float* wfold, void* stream) {
  ColorPlan p;
  if (int rc = color_plan(d, &p, wfold)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const float* const* g[2] = {d->base_g, d->main_g};
  const float* const* v[2] = {d->base_v, d->main_v};
  FoldJobs jobs;                                        // all layers of both stacks: one launch
  jobs.n = 0;
  for (int s = 0; s < 2; ++s)
    for (int l = 0; l < p.n_lin; ++l) add_fold_job(jobs, p.stack[s][l], g[s][l], v[s][l], wfold);
  if (int rc = run_fold_jobs(jobs, false, st)) return rc;
  if (get_engine() != 1) return 0;
  tc::PrepWJobs pj;
  pj.n = 0;
  for (int s = 0; s < 2; ++s)
    for (int l = 0; l < p.n_lin; ++l) add_prep_jobs(pj, p.stack[s][l], reinterpret_cast<uint16_t*>(wfold + p.w_total), IMG_ALL);
  return tc::prep_weights_jobs(pj, st);
}

int64_t nudf_color_ctx_floats(const nudf_color_desc* d, int64_t P) {
  ColorPlan p;
  if (color_plan(d, &p)) return -1;
  ColorCtx c;
  color_ctx_layout(p, P, &c);
  return c.total;
}
int64_t nudf_color_scratch_floats(const nudf_color_desc* d, int64_t P) {
  ColorPlan p;
  if (color_plan(d, &p)) return -1;
  ColorScratch s;
  color_scratch_layout(p, P, &s);
  return s.total;
}

int nudf_color_forward(const nudf_color_desc* d, const float* wfold, const float* pts, const float* dirs,
                       int32_t samples_per_ray, const float* feat, int64_t ld_feat, int64_t P, float* color_base,
                       float* color, float* blend, float* ctx, void* stream) {
  ColorPlan p;
  if (int rc = color_plan(d, &p, wfold)) return rc;
  if (P <= 0) return 0;
  NUDF_REQUIRE(wfold && pts && dirs && feat && ctx, "null pointer");
  NUDF_REQUIRE(aligned16(ctx), "ctx must be 16-byte aligned");
  NUDF_REQUIRE(ld_feat >= p.F, "ld_feat too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int spr = samples_per_ray > 0 ? samples_per_ray : 1;
  ColorCtx c;
  color_ctx_layout(p, P, &c);
  float* xb = ctx + c.xb;
  float* xm = ctx + c.xm;
  pack_pts_feat_kernel<<<ew_blocks(P * (p.ld_xb / 4), 256), 256, 0, st>>>(pts, feat, ld_feat, p.F, P, xb, p.ld_xb);
  NUDF_LAUNCH_OK();
  ew_pe_kernel<<<ew_blocks(P, 128), 128, 0, st>>>(dirs, 3, p.Lv, spr, P, xm, p.ld_xm, 0, nullptr, 0, 0);
  NUDF_LAUNCH_OK();
  const int nl = p.n_lin;
  // base stack
  for (int l = 0; l < nl; ++l) {
    const float* X = l == 0 ? xb : (l == nl - 1 ? xm + p.c_hid : ctx + c.hb[l]);
    int64_t ldx = l == 0 ? p.ld_xb : (l == nl - 1 ? p.ld_xm : p.ld_h);
    EpiAct e;
    e.bias = p.stack[BASE][l].bias; e.post_scale = 1.0f;
    if (l < nl - 2) { e.C = ctx + c.hb[l + 1]; e.ldc = p.ld_h; e.act = ACT_RELU; }
    else if (l == nl - 2) { e.C = xm + p.c_hid; e.ldc = p.ld_xm; e.act = ACT_RELU; }      // x_hidden (fields.py:472-473)
    else { e.C = xm + p.c_cb; e.ldc = p.ld_xm; e.act = ACT_SIGMOID; }                      // color_base (:475-476)
    if (int rc = color_layer_forward(p.stack[BASE][l], X, ldx, P, e, st)) return rc;
  }
  if (color_base) {
    ew_copy_cols_kernel<<<ew_blocks(P * p.d_out, 256), 256, 0, st>>>(xm + p.c_cb, p.ld_xm, color_base, p.d_out, 0, p.d_out, P, 1.f);
    NUDF_LAUNCH_OK();
  }
  // main stack
  for (int l = 0; l < nl; ++l) {
    const float* X = l == 0 ? xm : ctx + c.hm[l];
    int64_t ldx = l == 0 ? p.ld_xm : p.ld_h;
    EpiAct e;
    e.bias = p.stack[MAIN][l].bias; e.post_scale = 1.0f;
    if (l < nl - 1) { e.C = ctx + c.hm[l + 1]; e.ldc = p.ld_h; e.act = ACT_RELU; }
    else { e.C = ctx + c.ym; e.ldc = p.ld_ym; e.act = ACT_NONE; }
    if (int rc = color_layer_forward(p.stack[MAIN][l], X, ldx, P, e, st)) return rc;
  }
  color_head_kernel<<<ew_blocks(P * (p.d_out + p.n_blend), 256), 256, 0, st>>>(ctx + c.ym, p.ld_ym, p.d_out, p.n_blend, P,
                                                                              color, ctx + c.cs, 4, blend);
  NUDF_LAUNCH_OK();
  return 0;
}

int nudf_color_backward(const nudf_color_desc* d, const float* wfold, int64_t P, const float* cb_bar, const float* c_bar,
                        const float* blend_bar, const float* ctx_c, float* scratch, float* dfeat, int64_t ld_df,
                        float* dwfold, float* dbias, void* stream) {
  ColorPlan p;
  if (int rc = color_plan(d, &p, wfold)) return rc;
  NUDF_REQUIRE(wfold && ctx_c && scratch && dwfold && dbias, "null pointer");
  NUDF_REQUIRE(aligned16(ctx_c) && aligned16(scratch), "ctx and scratch must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  NUDF_CUDA_OK(cudaMemsetAsync(dwfold, 0, sizeof(float) * p.w_total, st));
  NUDF_CUDA_OK(cudaMemsetAsync(dbias, 0, sizeof(float) * p.b_total, st));
  if (P <= 0) return 0;
  float* ctx = const_cast<float*>(ctx_c);
  ColorCtx c;
  color_ctx_layout(p, P, &c);
  ColorScratch s;
  color_scratch_layout(p, P, &s);
  const int nl = p.n_lin;
  float* xm = ctx + c.xm;
  float* dym = scratch + s.dym;
  sigmoid_head_bwd_kernel<<<ew_blocks(P * p.ld_ym, 256), 256, 0, st>>>(c_bar, p.d_out, nullptr, 0, ctx + c.cs, 4, p.d_out,
                                                                      blend_bar, p.n_blend, p.n_blend, P, dym, p.ld_ym);
  NUDF_LAUNCH_OK();
  // ---- main stack, top down ----
  const float* dz = dym; int64_t ldz = p.ld_ym;
  int flip = 0;
  for (int l = nl - 1; l >= 0; --l) {
    const DenseLayer& L = p.stack[MAIN][l];
    const float* X = l == 0 ? xm : ctx + c.hm[l];
    int64_t ldx = l == 0 ? p.ld_xm : p.ld_h;
    if (int rc = wgrad(L, dz, ldz, X, ldx, P, dwfold + L.w_off, dbias + L.b_off, st)) return rc;
    float* out = scratch + s.buf[flip];
    if (l >= 1) {
      EpiReluBwd e{0, p.H, ctx + c.hm[l], p.ld_h, out, p.ld_h, 0};
      if (int rc = layer_nn(L, dz, ldz, P, e, TC_COLOR, st)) return rc;
    } else {
      EpiColorMainIn e{p.c_cb, p.c_hid, L.n_in, scratch + s.dcbx, 4, xm + p.c_hid, p.ld_xm, out, p.ld_h};
      if (int rc = layer_nn(L, dz, ldz, P, e, TC_COLOR, st)) return rc;
    }
    dz = out; ldz = p.ld_h; flip ^= 1;
  }
  // dz now = masked d(pre-activation of base layer nl-2) coming through the main stack, living in buf[flip^1]
  float* dzb = const_cast<float*>(dz);
  float* dyb = scratch + s.dyb;
  sigmoid_head_bwd_kernel<<<ew_blocks(P * 4, 256), 256, 0, st>>>(cb_bar, p.d_out, scratch + s.dcbx, 4, xm + p.c_cb, p.ld_xm,
                                                                p.d_out, nullptr, 0, 0, P, dyb, 4);
  NUDF_LAUNCH_OK();
  // ---- base stack ----
  {
    const DenseLayer& L = p.stack[BASE][nl - 1];       // colour_base head: K = d_out <= 4, no image, the FFMA kernel
    if (int rc = wgrad(L, dyb, 4, xm + p.c_hid, p.ld_xm, P, dwfold + L.w_off, dbias + L.b_off, st)) return rc;
    EpiReluBwd e{0, p.H, xm + p.c_hid, p.ld_xm, dzb, p.ld_h, 1};
    if (int rc = layer_nn(L, dyb, 4, P, e, TC_COLOR, st)) return rc;
  }
  dz = dzb; ldz = p.ld_h;
  for (int l = nl - 2; l >= 0; --l) {
    const DenseLayer& L = p.stack[BASE][l];
    const float* X = l == 0 ? ctx + c.xb : ctx + c.hb[l];
    int64_t ldx = l == 0 ? p.ld_xb : p.ld_h;
    if (int rc = wgrad(L, dz, ldz, X, ldx, P, dwfold + L.w_off, dbias + L.b_off, st)) return rc;
    if (l >= 1) {
      float* out = scratch + s.buf[flip];
      EpiReluBwd e{0, p.H, ctx + c.hb[l], p.ld_h, out, p.ld_h, 0};
      if (int rc = layer_nn(L, dz, ldz, P, e, TC_COLOR, st)) return rc;
      dz = out; flip ^= 1;
    } else if (dfeat) {
      EpiReluBwd e{3, 3 + p.F, nullptr, 0, dfeat, ld_df, 0};
      if (int rc = layer_nn(L, dz, ldz, P, e, TC_COLOR, st)) return rc;
    }
  }
  return 0;
}

int nudf_color_unfold_grads(const nudf_color_desc* d, const float* dwfold, float* const* dg_base, float* const* dv_base,
                            float* const* dg_main, float* const* dv_main, void* stream) {
  ColorPlan p;
  if (int rc = color_plan(d, &p)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const float* const* g[2] = {d->base_g, d->main_g};
  const float* const* v[2] = {d->base_v, d->main_v};
  float* const* dg[2] = {dg_base, dg_main};
  float* const* dv[2] = {dv_base, dv_main};
  FoldJobs jobs;
  jobs.n = 0;
  for (int s = 0; s < 2; ++s)
    for (int l = 0; l < p.n_lin; ++l) add_unfold_job(jobs, p.stack[s][l], g[s][l], v[s][l], dwfold, dg[s][l], dv[s][l]);
  return run_fold_jobs(jobs, true, st);
}

// =================================================================================================================
// NeRF++ background network
// =================================================================================================================
}  // extern "C"

namespace nudf {
enum { VIEWS = 0, FEATURE = 1, ALPHA = 2, RGB = 3 };
struct NerfPlan {
  int D, W, d_in, L, Lv, skip, ch, chv, ld_f, ld_x5;
  int ld_w, ld_v;   // row strides of the W-wide hidden activations (and gradients) and of the W / 2-wide views layer
  // the D pts layers, then [D + VIEWS .. D + RGB]: the order of nudf_nerf_backward's dparams (weight, bias) pairs
  DenseLayer layer[NUDF_MAX_LAYERS + 4];
  int64_t img_total;
};
// wimg (optional): the image block of nudf_nerf_prepare; null = exact-fp32 engine
static int nerf_plan(const nudf_nerf_desc* d, NerfPlan* p, const float* wimg = nullptr) {
  NUDF_REQUIRE(d != nullptr, "null desc");
  NUDF_REQUIRE(d->D >= 2 && d->D <= NUDF_MAX_LAYERS, "D out of range");
  p->D = d->D; p->W = d->W; p->d_in = d->d_in; p->L = d->multires; p->Lv = d->multires_view; p->skip = d->skip;
  NUDF_REQUIRE(p->skip < p->D - 1, "skip on the last layer is not supported");
  NUDF_REQUIRE(p->d_in >= 1 && p->d_in <= 4, "d_in out of range");
  p->ch = p->d_in * (1 + 2 * p->L);
  p->chv = 3 * (1 + 2 * p->Lv);
  p->ld_f = (int)round_up(p->W + p->chv, 4);
  p->ld_x5 = (int)round_up(p->W + p->ch, 4);
  p->ld_w = (int)round_up(p->W, 4);
  p->ld_v = (int)round_up(p->W / 2, 4);
  int64_t io = 0;
  auto set = [&](int i, const float* W, const float* b, int n_out, int n_in, int want) {
    DenseLayer& L = p->layer[i];
    L.W = W; L.bias = b; L.n_out = n_out; L.n_in = n_in;
    L.ldw = n_in; L.w_off = L.b_off = 0;                    // plain nn.Linear parameters, read in place
    L.img = reinterpret_cast<const uint16_t*>(wimg);
    io = plan_images(L, want, io);
  };
  // forward images with 3 planes (6 products); the backward pass ends at the first layer's weight gradient: no dY W image there.
  // The alpha and rgb heads (1 and 3 outputs) are no tensor-core shape: they own no image and run on the FFMA kernel.
  const int both = 1 << IMG_NT3 | 1 << IMG_NN2;
  for (int i = 0; i < p->D; ++i)
    set(i, d->pts_w[i], d->pts_b[i], p->W, i == 0 ? p->ch : (i - 1 == p->skip ? p->W + p->ch : p->W), i == 0 ? 1 << IMG_NT3 : both);
  set(p->D + VIEWS, d->views_w, d->views_b, p->W / 2, p->W + p->chv, both);
  set(p->D + FEATURE, d->feature_w, d->feature_b, p->W, p->W, both);
  set(p->D + ALPHA, d->alpha_w, d->alpha_b, 1, p->W, both);
  set(p->D + RGB, d->rgb_w, d->rgb_b, 3, p->W / 2, both);
  p->img_total = round_up(io, 8);
  return 0;
}
struct NerfCtx { int64_t e, h[NUDF_MAX_LAYERS], f, hv, total; };
// h[i] = post-ReLU output of pts layer i; for i == skip it lives inside the concatenated buffer at column ch.
static void nerf_ctx_layout(const NerfPlan& p, int64_t P, NerfCtx* c) {
  Bump b;
  c->e = b.take(P * round_up(p.ch, 4));
  for (int i = 0; i < p.D; ++i) c->h[i] = b.take(P * (i == p.skip ? p.ld_x5 : p.ld_w));
  c->f = b.take(P * p.ld_f);
  c->hv = b.take(P * p.ld_v);
  c->total = b.off;
}
struct NerfScratch { int64_t buf[2], dzv, total; };
static void nerf_scratch_layout(const NerfPlan& p, int64_t P, NerfScratch* s) {
  Bump b;
  s->buf[0] = b.take(P * p.ld_w); s->buf[1] = b.take(P * p.ld_w);
  s->dzv = b.take(P * p.ld_v);
  s->total = b.off;
}
// layer-i output location
static inline float* nerf_h(const NerfPlan& p, float* ctx, const NerfCtx& c, int i, int64_t* ld) {
  if (i == p.skip) { *ld = p.ld_x5; return ctx + c.h[i] + p.ch; }
  *ld = p.ld_w; return ctx + c.h[i];
}
// layer-i input location
static inline const float* nerf_x(const NerfPlan& p, float* ctx, const NerfCtx& c, int i, int64_t* ld) {
  if (i == 0) { *ld = round_up(p.ch, 4); return ctx + c.e; }
  if (i - 1 == p.skip) { *ld = p.ld_x5; return ctx + c.h[i - 1]; }
  *ld = p.ld_w; return ctx + c.h[i - 1];
}
}  // namespace nudf

extern "C" {

int64_t nudf_nerf_image_floats(const nudf_nerf_desc* d) {
  NerfPlan p;
  if (nerf_plan(d, &p)) return -1;
  return p.img_total / 2;
}

int nudf_nerf_prepare(const nudf_nerf_desc* d, float* wimg, void* stream) {
  NerfPlan p;
  if (int rc = nerf_plan(d, &p, wimg)) return rc;
  NUDF_REQUIRE(wimg != nullptr, "null wimg");
  cudaStream_t st = (cudaStream_t)stream;
  tc::PrepWJobs pj;                                        // all images in one launch
  pj.n = 0;
  for (int i = 0; i < p.D + 4; ++i) add_prep_jobs(pj, p.layer[i], reinterpret_cast<uint16_t*>(wimg), IMG_ALL);
  return tc::prep_weights_jobs(pj, st);
}

int64_t nudf_nerf_ctx_floats(const nudf_nerf_desc* d, int64_t P) {
  NerfPlan p;
  if (nerf_plan(d, &p)) return -1;
  NerfCtx c;
  nerf_ctx_layout(p, P, &c);
  return c.total;
}
int64_t nudf_nerf_scratch_floats(const nudf_nerf_desc* d, int64_t P) {
  NerfPlan p;
  if (nerf_plan(d, &p)) return -1;
  NerfScratch s;
  nerf_scratch_layout(p, P, &s);
  return s.total;
}

int nudf_nerf_forward(const nudf_nerf_desc* d, const float* wimg, const float* pts, const float* dirs, int32_t samples_per_ray,
                      int64_t P, float* sigma, float* rgb, float* ctx, void* stream) {
  NerfPlan p;
  if (int rc = nerf_plan(d, &p, wimg)) return rc;
  if (P <= 0) return 0;
  NUDF_REQUIRE(pts && dirs && sigma && rgb && ctx, "null pointer");
  NUDF_REQUIRE(aligned16(ctx), "ctx must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int spr = samples_per_ray > 0 ? samples_per_ray : 1;
  NerfCtx c;
  nerf_ctx_layout(p, P, &c);
  const int ld_e = (int)round_up(p.ch, 4);
  float* x5 = (p.skip >= 0) ? ctx + c.h[p.skip] : nullptr;
  ew_pe_kernel<<<ew_blocks(P, 128), 128, 0, st>>>(pts, p.d_in, p.L, 1, P, ctx + c.e, ld_e, 0, x5, p.ld_x5, 0);
  NUDF_LAUNCH_OK();
  ew_pe_kernel<<<ew_blocks(P, 128), 128, 0, st>>>(dirs, 3, p.Lv, spr, P, ctx + c.f, p.ld_f, p.W, nullptr, 0, 0);
  NUDF_LAUNCH_OK();
  for (int i = 0; i < p.D; ++i) {
    int64_t ldx, ldh;
    const float* X = nerf_x(p, ctx, c, i, &ldx);
    float* Hh = nerf_h(p, ctx, c, i, &ldh);
    EpiAct e{Hh, ldh, p.layer[i].bias, ACT_RELU, 1.0f};
    if (int rc = layer_nt(p.layer[i], X, ldx, P, e, TC_RELU_FWD, st)) return rc;
  }
  const DenseLayer* head = p.layer + p.D;
  int64_t ldl;
  const float* Hl = nerf_h(p, ctx, c, p.D - 1, &ldl);
  {
    EpiAct e{sigma, 1, head[ALPHA].bias, ACT_NONE, 1.0f};
    if (int rc = layer_nt(head[ALPHA], Hl, ldl, P, e, TC_RELU_FWD, st)) return rc;
  }
  {
    EpiAct e{ctx + c.f, p.ld_f, head[FEATURE].bias, ACT_NONE, 1.0f};
    if (int rc = layer_nt(head[FEATURE], Hl, ldl, P, e, TC_RELU_FWD, st)) return rc;
  }
  {
    EpiAct e{ctx + c.hv, p.ld_v, head[VIEWS].bias, ACT_RELU, 1.0f};
    if (int rc = layer_nt(head[VIEWS], ctx + c.f, p.ld_f, P, e, TC_RELU_FWD, st)) return rc;
  }
  {
    EpiAct e{rgb, 3, head[RGB].bias, ACT_NONE, 1.0f};
    if (int rc = layer_nt(head[RGB], ctx + c.hv, p.ld_v, P, e, TC_RELU_FWD, st)) return rc;
  }
  return 0;
}

int nudf_nerf_backward(const nudf_nerf_desc* d, const float* wimg, int64_t P, const float* sigma_bar, const float* rgb_bar,
                       const float* ctx_c, float* scratch, float* const* dparams, void* stream) {
  NerfPlan p;
  if (int rc = nerf_plan(d, &p, wimg)) return rc;
  NUDF_REQUIRE(sigma_bar && rgb_bar && ctx_c && scratch && dparams, "null pointer");
  NUDF_REQUIRE(aligned16(ctx_c) && aligned16(scratch), "ctx and scratch must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int D = p.D, W = p.W, W2 = p.W / 2, ld_w = p.ld_w, ld_v = p.ld_v;
  for (int i = 0; i < D + 4; ++i) {                        // dparams[2 i], [2 i + 1] = weight and bias gradient of layer i
    NUDF_CUDA_OK(cudaMemsetAsync(dparams[2 * i], 0, sizeof(float) * p.layer[i].n_out * p.layer[i].n_in, st));
    NUDF_CUDA_OK(cudaMemsetAsync(dparams[2 * i + 1], 0, sizeof(float) * p.layer[i].n_out, st));
  }
  if (P <= 0) return 0;
  float* ctx = const_cast<float*>(ctx_c);
  NerfCtx c;
  nerf_ctx_layout(p, P, &c);
  NerfScratch s;
  nerf_scratch_layout(p, P, &s);
  const DenseLayer* head = p.layer + D;
  float* const* dhead = dparams + 2 * D;
  // rgb head
  if (int rc = wgrad(head[RGB], rgb_bar, 3, ctx + c.hv, ld_v, P, dhead[2 * RGB], dhead[2 * RGB + 1], st)) return rc;
  float* dzv = scratch + s.dzv;
  {
    EpiReluBwd e{0, W2, ctx + c.hv, ld_v, dzv, ld_v, 0};
    if (int rc = layer_nn(head[RGB], rgb_bar, 3, P, e, TC_NERF, st)) return rc;
  }
  // views layer
  if (int rc = wgrad(head[VIEWS], dzv, ld_v, ctx + c.f, p.ld_f, P, dhead[2 * VIEWS], dhead[2 * VIEWS + 1], st)) return rc;
  float* dfeat = scratch + s.buf[0];
  {
    EpiReluBwd e{0, W, nullptr, 0, dfeat, ld_w, 0};
    if (int rc = layer_nn(head[VIEWS], dzv, ld_v, P, e, TC_NERF, st)) return rc;
  }
  // feature + alpha heads -> dZ of the last pts layer
  int64_t ldl;
  const float* Hl = nerf_h(p, ctx, c, D - 1, &ldl);
  if (int rc = wgrad(head[FEATURE], dfeat, ld_w, Hl, ldl, P, dhead[2 * FEATURE], dhead[2 * FEATURE + 1], st)) return rc;
  if (int rc = wgrad(head[ALPHA], sigma_bar, 1, Hl, ldl, P, dhead[2 * ALPHA], dhead[2 * ALPHA + 1], st)) return rc;
  float* dz = scratch + s.buf[1];
  {
    EpiReluBwd e0{0, W, nullptr, 0, dz, ld_w, 0};
    if (int rc = layer_nn(head[ALPHA], sigma_bar, 1, P, e0, TC_NERF, st)) return rc;
    EpiReluBwd e1{0, W, Hl, ldl, dz, ld_w, 1};
    if (int rc = layer_nn(head[FEATURE], dfeat, ld_w, P, e1, TC_NERF, st)) return rc;
  }
  int flip = 0;  // dz lives in buf[1]; next output goes to buf[0]
  for (int i = D - 1; i >= 0; --i) {
    int64_t ldx;
    const float* X = nerf_x(p, ctx, c, i, &ldx);
    if (int rc = wgrad(p.layer[i], dz, ld_w, X, ldx, P, dparams[2 * i], dparams[2 * i + 1], st)) return rc;
    if (i == 0) break;
    float* out = scratch + s.buf[flip];
    int64_t ldh;
    const float* Hprev = nerf_h(p, ctx, c, i - 1, &ldh);
    int col_lo = (i - 1 == p.skip) ? p.ch : 0;
    EpiReluBwd e{col_lo, col_lo + W, Hprev, ldh, out, ld_w, 0};
    if (int rc = layer_nn(p.layer[i], dz, ld_w, P, e, TC_NERF, st)) return rc;
    dz = out; flip ^= 1;
  }
  return 0;
}

}  // extern "C"

/* nudf.h -- C ABI of libnudf.so, the H100 (sm_90a) implementation of NeuralUDF's volume-rendering hot path.
 *
 * The reference (xxlong0/NeuralUDF) is pure PyTorch and has NO plugin / FFI layer (SURVEY.md section 0, fact 5);
 * its "boundary" for this path is the Python surface `exp_runner_blending.py:15-19` imports.  This header is the
 * C-ABI a drop-in replacement binds instead (INTEGRATION.md shows the ctypes stub): every entry point below cites
 * the reference interface it replaces.  Conventions:
 *   - all pointers are DEVICE pointers into caller-owned (torch) storages unless marked "host";
 *   - fp32, row-major, explicit leading dimensions (ld, in floats);
 *   - the library never allocates device memory: callers size workspaces with the *_floats() queries;
 *   - every call enqueues on `stream` (a cudaStream_t passed as void*) and returns immediately;
 *   - return value: 0 ok, -1 invalid argument, -2 CUDA error; nudf_last_error() has the text (thread-local).
 */
#ifndef NUDF_H_
#define NUDF_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NUDF_MAX_LAYERS 16
#define NUDF_ABI_VERSION 5
/* bits of the device-side status word (nudf_render_out.status, `status` of the sampling entry points): set by the kernels,
 * never cleared by the library; the caller reads it at a host synchronisation point of its choice */
#define NUDF_STATUS_NONFINITE_SAMPLES 1   /* sample_pdf / up_sample produced a non-finite sample position (:97-101, 265-269) */
#define NUDF_STATUS_NONFINITE_RENDER 2    /* compositing produced a non-finite per-ray result (:543-544) */

int nudf_abi_version(void);
const char* nudf_last_error(void);
/* GEMM engine for the wide (K,N in {128,256}) layers: 0 = exact-fp32 FFMA, 1 = wgmma split-bf16 tensor cores (default 1
 * when built with the tensor path).  Small / odd-shaped contractions always use the FFMA engine. */
int nudf_set_engine(int engine);
int nudf_get_engine(void);
/* Which contraction chains may use the tensor engine (bit mask; default 255 = all; the UDF value chain and the colour /
 * NeRF++ forward use three bf16 planes, the udf-head row stays exact fp32): 1 UDF forward value, 2 reverse sweep (grad_x udf), 4 tangent,
 * 8 backward, 16 weight gradients, 32 colour-network backward, 64 NeRF++ backward, 128 colour / NeRF++ forward. */
int nudf_set_tc_mask(int mask);
int nudf_get_tc_mask(void);
int nudf_default_tc_mask(void);   /* the mask the library ships (what bench.py times and the parity suite pins) */
/* --- tensor engine building blocks (unit-tested on their own) ---
 * weight image: bf16 hi/lo split of B(n,k) in UMMA shared-memory order; `transposed` selects B(n,k) = W[k*ldw+n]. */
/* planes: 2 = hi/lo (3 products, ~4e-6 vs fp64), 3 = hi/mid/lo (6 products, fp32-grade; used by the value chain) */
int64_t nudf_tc_image_elems(int32_t N, int32_t K, int32_t planes);
int nudf_tc_prepare_weights(const float* W, int64_t ldw, int32_t N, int32_t K, int32_t transposed, int32_t planes,
                            uint16_t* img, void* stream);
int nudf_dense_forward_tc(const float* X, int64_t ldx, const uint16_t* img, int32_t planes, const float* bias, float* Y,
                          int64_t ldy, int64_t M, int32_t N, int32_t K, int32_t act, void* stream);
/* dW[n_out, n_in] += dZ[P, n_out]^T X[P, n_in]  (engine 0: fp32 FFMA, 1: tensor cores) */
int nudf_wgrad(const float* dZ, int64_t ldz, const float* X, int64_t ldx, int32_t n_out, int32_t n_in, int64_t P,
               float* dW, int64_t ldw, int32_t engine, void* stream);

/* number of CUDA kernels this library has launched in this process (bench.py reports it as gpu_launches) */
int64_t nudf_launch_count(void);
/* Per-kernel-family device times for the benchmark's roofline table: while enabled, the library brackets its launches with
 * cudaEvent pairs on the launching stream.  nudf_read_launch_timing synchronises, writes the summed milliseconds and the
 * launch counts per family (host arrays of nudf_launch_family_count() entries; order: fused UDF value chain (not built), tensor-core
 * reverse-sweep / tangent / backward / other layers, tensor-core weight gradients, fp32 FFMA GEMMs, ray kernels, element-wise,
 * fused tangent + backward chains (not built))
 * and clears the record. */
int nudf_launch_family_count(void);
int nudf_set_launch_timing(int on);
int nudf_read_launch_timing(float* ms_per_family, int32_t* launches_per_family);
/* One fused dense layer Y[M,N] = act(X[M,K] W[N,K]^T + bias), act: 0 none, 1 relu, 2 softplus(beta=100), 3 sigmoid.
 * The building block of every network below (an nn.Linear + activation of the reference, e.g. fields.py:205-208). */
int nudf_dense_forward(const float* X, int64_t ldx, const float* W, int64_t ldw, const float* bias, float* Y, int64_t ldy,
                       int64_t M, int32_t N, int32_t K, int32_t act, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * UDFNetwork  (reference: models/fields.py:115-231; forward :192-211, gradient :219-231)
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct nudf_udf_desc {
  int32_t n_lin;      /* number of linear layers = n_layers + 1                                   */
  int32_t d_in;       /* 3                                                                        */
  int32_t multires;   /* positional-encoding octaves L (models/embedder.py:39-51)                 */
  int32_t d_out;      /* 257 = 1 (udf) + feature width                                            */
  int32_t skip_layer; /* layer whose input is cat(h, PE)/sqrt(2) (fields.py:202-203), -1 if none  */
  float scale;        /* fields.py:193                                                            */
  int32_t in_dim[NUDF_MAX_LAYERS];
  int32_t out_dim[NUDF_MAX_LAYERS];
  const float* weight_g[NUDF_MAX_LAYERS]; /* [out,1]  legacy weight_norm g  (lin{l}.weight_g)     */
  const float* weight_v[NUDF_MAX_LAYERS]; /* [out,in] legacy weight_norm v  (lin{l}.weight_v)     */
  const float* bias[NUDF_MAX_LAYERS];     /* [out]                          (lin{l}.bias)         */
} nudf_udf_desc;

/* floats needed for the folded weights W_l = g_l v_l/||v_l|| (rows padded to a multiple of 4 floats) */
int64_t nudf_udf_folded_floats(const nudf_udf_desc* d);
/* folds weight-norm once per optimiser step (replaces torch._weight_norm inside every nn.Linear call) */
int nudf_udf_fold_weights(const nudf_udf_desc* d, float* wfold, void* stream);
/* floats of the activation context saved by forward for `P` points (with_grad: also the reverse-sweep tensors).
 * The ctx, scratch and work buffers of every network below need 16-byte-aligned bases: the layouts keep each block's
 * rows in whole 16-byte units from there, as the tensor-core kernels read them through 2-D tensor maps. */
int64_t nudf_udf_ctx_floats(const nudf_udf_desc* d, int64_t P, int with_grad);
/* floats of the scratch needed by backward */
int64_t nudf_udf_scratch_floats(const nudf_udf_desc* d, int64_t P);
/* out[P, ld_out] <- cat(|y0|/scale, y[1:])   (UDFNetwork.forward, fields.py:192-211)
 * grad[P,3]     <- d udf / d x exactly, by a reverse sweep (UDFNetwork.gradient, fields.py:219-231); may be NULL.
 * ctx           <- saved activations (required; sized by nudf_udf_ctx_floats(d, P, grad != NULL)). */
int nudf_udf_forward(const nudf_udf_desc* d, const float* wfold, const float* pts, int64_t P, float* out,
                     int64_t ld_out, float* grad, float* ctx, void* stream);
/* Value only (no context kept): udf[P] <- |y0|/scale.  Used by importance sampling and grid queries
 * (udf_renderer_blending.py:731-733, 282-284; extract_mesh.py:60-73). `work` needs nudf_udf_ctx_floats(d,P,0). */
int nudf_udf_value(const nudf_udf_desc* d, const float* wfold, const float* pts, int64_t P, float* udf, float* work,
                   void* stream);
/* Parameter gradients for  L = <out_bar, out> + <grad_bar, grad>  (first- and second-order terms; the latter is
 * what autograd's double backward through create_graph=True computes in the reference).  out_bar [P, ld_ob] and
 * grad_bar [P,3] may each be NULL (= zero).  dwfold (same layout as wfold) and dbias (sum of out_dim floats) are
 * OVERWRITTEN.  ctx must come from nudf_udf_forward with grad != NULL on the same points. */
int nudf_udf_backward(const nudf_udf_desc* d, const float* wfold, const float* pts, int64_t P, const float* out_bar,
                      int64_t ld_ob, const float* grad_bar, const float* ctx, float* scratch, float* dwfold,
                      float* dbias, void* stream);
/* The same pair with the value and the feature part as SEPARATE tensors (udf [P], feat [P, ld_feat]; udf_bar [P], feat_bar
 * [P, ld_fb], each may be NULL = zero): what render_core consumes (udf_renderer_blending.py:364-366 slices udf_nn_output[:, :1]
 * and [:, 1:]) without an odd-width [P, 257] tensor in between and without re-assembling its gradient. */
int nudf_udf_forward_split(const nudf_udf_desc* d, const float* wfold, const float* pts, int64_t P, float* udf, float* feat,
                           int64_t ld_feat, float* grad, float* ctx, void* stream);
int nudf_udf_backward_split(const nudf_udf_desc* d, const float* wfold, const float* pts, int64_t P, const float* udf_bar,
                            const float* feat_bar, int64_t ld_fb, const float* grad_bar, const float* ctx, float* scratch,
                            float* dwfold, float* dbias, void* stream);
/* weight-norm backward: dwfold -> (dg[l] [out,1], dv[l] [out,in]) for every layer (overwrites) */
int nudf_udf_unfold_grads(const nudf_udf_desc* d, const float* dwfold, float* const* dg, float* const* dv, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * ResidualRenderingNetwork, mode 'no_normal'  (reference: models/fields.py:400-495)
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct nudf_color_desc {
  int32_t n_lin;        /* n_layers + 1 (5) */
  int32_t d_feature;    /* 256 */
  int32_t d_hidden;     /* 128 */
  int32_t d_out;        /* 3   */
  int32_t n_blend;      /* blending_cand_views (10) */
  int32_t multires_view;/* 4   */
  const float* base_g[NUDF_MAX_LAYERS]; const float* base_v[NUDF_MAX_LAYERS]; const float* base_b[NUDF_MAX_LAYERS];
  const float* main_g[NUDF_MAX_LAYERS]; const float* main_v[NUDF_MAX_LAYERS]; const float* main_b[NUDF_MAX_LAYERS];
} nudf_color_desc;

int64_t nudf_color_folded_floats(const nudf_color_desc* d);
int nudf_color_fold_weights(const nudf_color_desc* d, float* wfold, void* stream);
/* ctx and scratch: 16-byte-aligned bases */
int64_t nudf_color_ctx_floats(const nudf_color_desc* d, int64_t P);
int64_t nudf_color_scratch_floats(const nudf_color_desc* d, int64_t P);
/* color_base[P,3], color[P,3], blend[P,n_blend] <- forward(points, view_dirs, feature_vectors) (fields.py:452-495).
 * dirs is [P,3] when samples_per_ray <= 1; otherwise it is [P / samples_per_ray, 3] and row p uses
 * dirs[p / samples_per_ray] (the reference materialises that expansion of rays_d, udf_renderer_blending.py:359-362). */
int nudf_color_forward(const nudf_color_desc* d, const float* wfold, const float* pts, const float* dirs,
                       int32_t samples_per_ray, const float* feat, int64_t ld_feat, int64_t P, float* color_base,
                       float* color, float* blend, float* ctx, void* stream);
/* grads wrt parameters (dwfold/dbias overwritten) and wrt feature_vectors (dfeat [P, ld_df] overwritten).
 * cb_bar/c_bar [P,3], blend_bar [P,n_blend]; any may be NULL (= zero). */
int nudf_color_backward(const nudf_color_desc* d, const float* wfold, int64_t P, const float* cb_bar,
                        const float* c_bar, const float* blend_bar, const float* ctx, float* scratch, float* dfeat,
                        int64_t ld_df, float* dwfold, float* dbias, void* stream);
int nudf_color_unfold_grads(const nudf_color_desc* d, const float* dwfold, float* const* dg_base, float* const* dv_base,
                            float* const* dg_main, float* const* dv_main, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * NeRF++ background network  (reference: models/fields.py:541-628, use_viewdirs=True)
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct nudf_nerf_desc {
  int32_t D;             /* 8   */
  int32_t W;             /* 256 */
  int32_t d_in;          /* 4   */
  int32_t multires;      /* 10  */
  int32_t multires_view; /* 4   */
  int32_t skip;          /* skips[0] = 4: output of layer `skip` is concatenated as cat(PE, h) */
  const float* pts_w[NUDF_MAX_LAYERS]; const float* pts_b[NUDF_MAX_LAYERS];
  const float* views_w; const float* views_b;
  const float* feature_w; const float* feature_b;
  const float* alpha_w; const float* alpha_b;
  const float* rgb_w; const float* rgb_b;
} nudf_nerf_desc;

/* tensor-engine weight images of the NeRF layers (floats); build with nudf_nerf_prepare once per optimiser step and pass
 * to forward/backward (NULL = exact-fp32 engine) */
int64_t nudf_nerf_image_floats(const nudf_nerf_desc* d);
int nudf_nerf_prepare(const nudf_nerf_desc* d, float* wimg, void* stream);
/* ctx and scratch: 16-byte-aligned bases */
int64_t nudf_nerf_ctx_floats(const nudf_nerf_desc* d, int64_t P);
int64_t nudf_nerf_scratch_floats(const nudf_nerf_desc* d, int64_t P);
/* sigma[P], rgb[P,3] <- NeRF.forward(pts4, view_dirs) (fields.py:599-628; no sigmoid on rgb) */
int nudf_nerf_forward(const nudf_nerf_desc* d, const float* wimg, const float* pts, const float* dirs,
                      int32_t samples_per_ray, int64_t P, float* sigma, float* rgb, float* ctx, void* stream);
/* parameter gradients; dparams[] order: pts_w[0], pts_b[0], ..., views_w, views_b, feature_w, feature_b, alpha_w,
 * alpha_b, rgb_w, rgb_b  (each overwritten, same shape as the parameter). */
int nudf_nerf_backward(const nudf_nerf_desc* d, const float* wimg, int64_t P, const float* sigma_bar,
                       const float* rgb_bar, const float* ctx, float* scratch, float* const* dparams, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * render_core ray kernels  (reference: models/udf_renderer_blending.py:327-584)
 * ------------------------------------------------------------------------------------------------------------ */
typedef struct nudf_render_cfg {
  int32_t n_rays;           /* N */
  int32_t n_samples;        /* S  (columns of z_vals entering render_core) */
  int32_t n_outside;        /* O  (0 when no NeRF++ background is composited) */
  float sample_dist;        /* last-interval length, :353 */
  float cos_anneal_ratio;   /* :296-297; used only when has_cos_anneal != 0 */
  int32_t has_cos_anneal;
  float flip_saturation;    /* :409 */
  float sparse_scale_factor;/* :553 */
  int32_t use_norm_grad_for_cosine; /* :380-383 */
  int32_t has_background_rgb; float background_rgb[3]; /* :527-528 */
} nudf_render_cfg;

/* pts[N*S,3], mid_z[N,S], dists[N,S] <- rays and z_vals (:352-362) */
int nudf_ray_points(const float* rays_o, const float* rays_d, const float* z_vals, int32_t n_rays, int32_t n_samples,
                    float sample_dist, float* pts, float* mid_z, float* dists, void* stream);

/* per-sample / per-ray output pointers of the compositing pass; any per-sample pointer may be NULL */
typedef struct nudf_render_out {
  float* color_base; float* color; float* depth; float* normals;  /* [N,3] [N,3] [N,1] [N,3] */
  float* weights;                                                 /* [N,S+O] */
  float* weight_sum; float* weight_sum_fg_bg;                     /* [N,1] */
  float* ray_sums;  /* [N,5]: sum relax*(|g|-1)^2, sum relax, sum near*(|g|-1)^2, sum near, sum exp(-k udf) */
  float* gradient_mag; float* true_cos; float* vis_prob; float* alpha; float* alpha_plus; float* alpha_minus;
  float* alpha_occ; float* raw_occ; float* inside_sphere;        /* [N,S] each */
  float* gradients_flip;                                         /* [N,S,3] */
  int32_t* status;  /* DEVICE int or NULL: NUDF_STATUS_NONFINITE_RENDER is OR-ed in when a ray's colour / depth / weight sum /
                     * regulariser sums are not finite (the reference traps this with pdb, :543-544) */
} nudf_render_out;

/* alpha compositing with the visibility-weighted UDF density (:364-553 minus the networks).
 * heads: DEVICE float[3] = (inv_s, beta, gamma) after the clips of :373-377 (kept on the device so that a training
 * step needs no host synchronisation).
 * udf [N*S] (stride ld_udf floats between samples), grads [N*S,3], sampled colours [N*S,3] x2,
 * bg_alpha [N,S+O] / bg_color [N,S+O,3] from render_core_outside (only columns >= S are read), may be NULL. */
int nudf_render_composite_forward(const nudf_render_cfg* cfg, const float* heads, const float* rays_d, const float* pts,
                                  const float* mid_z, const float* dists, const float* udf, int64_t ld_udf,
                                  const float* grads, const float* sampled_color_base, const float* sampled_color,
                                  const float* bg_alpha, const float* bg_color, const nudf_render_out* out,
                                  void* stream);

/* per-ray outputs of the forward-only view renderer; each may be NULL.  They may point into a larger image at the chunk's
 * first ray, so that a whole view is written in place. */
typedef struct nudf_view_out {
  float* color;        /* [N,3]  as nudf_render_composite_forward's `color` (same bits) */
  float* color_pixel;  /* [N,3]  pixel-blend composite (needs c_pix) */
  float* depth;        /* [N,1]  as nudf_render_composite_forward's `depth` (same bits) */
  float* normal;       /* [N,3]  rot @ sum_i gradients_flip_i * weights_i * inside_sphere_i over the S foreground samples */
  float* weight_sum;   /* [N,1]  foreground weight sum */
} nudf_view_out;

/* Forward-only compositing of whole views (the image outputs of exp_runner_blending.py's validate(), :621-682): the alpha,
 * visibility scan and weights of nudf_render_composite_forward (the same device code), no per-sample outputs, no state for
 * a backward pass.  Inputs as nudf_render_composite_forward, without sampled_color_base, plus
 *   c_pix  [N*S,3] per-sample pixel-blend colour (nudf_blend_forward's c_pix) or NULL.  When n_outside > 0 the blend
 *          colour of a sample outside the unit sphere is replaced by bg_color of its own column (:503-507), so bg_color
 *          must then hold all S+O columns;
 *   rot    HOST row-major 3x3 applied to the normal (the inverse of the view's pose rotation, :681). */
int nudf_render_view_forward(const nudf_render_cfg* cfg, const float* heads, const float* rays_d, const float* pts,
                             const float* mid_z, const float* dists, const float* udf, int64_t ld_udf, const float* grads,
                             const float* sampled_color, const float* c_pix, const float* bg_alpha, const float* bg_color,
                             const float* rot, const nudf_view_out* out, void* stream);

typedef struct nudf_render_bar {   /* upstream gradients, any may be NULL */
  const float* color_base; const float* color; const float* depth;       /* [N,3] [N,3] [N,1] */
  const float* weight_sum; const float* weight_sum_fg_bg;                 /* [N,1] */
  const float* weights;  /* [N,S+O] d loss / d weights (pixel / patch blending composites are formed from `weights`) */
  const float* ray_sums; /* [N,5] d loss / d ray_sums (columns 1 and 3, the detached mask counts, are ignored) */
} nudf_render_bar;

/* Backward of the compositing pass.  Outputs (overwritten): udf_bar [N*S], grads_bar [N*S,3], scb_bar/sc_bar
 * [N*S,3], bg_alpha_bar [N,S+O] / bg_color_bar [N,S+O,3] (may be NULL), scalar_bar[N,3] = per-ray partial
 * d/d(inv_s, beta, gamma) (caller sums over rays). */
int nudf_render_composite_backward(const nudf_render_cfg* cfg, const float* heads, const float* rays_d, const float* pts,
                                   const float* mid_z, const float* dists, const float* udf, int64_t ld_udf,
                                   const float* grads, const float* sampled_color_base, const float* sampled_color,
                                   const float* bg_alpha, const float* bg_color, const nudf_render_bar* bar,
                                   float* udf_bar, float* grads_bar, float* scb_bar,
                                   float* sc_bar, float* bg_alpha_bar, float* bg_color_bar, float* scalar_bar,
                                   void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * hierarchical sampling  (reference: models/udf_renderer_blending.py:66-104, 197-290, 723-755, 834-866)
 * ------------------------------------------------------------------------------------------------------------ */
/* One up-sampling round: new_z[N,m] (and optionally the searchsorted indices inds[N,m], int64) from z[N,n], udf[N,n].
 * mode 0 = up_sample_unbias (:197-272), 1 = up_sample_no_occ_aware (:834-866).  Scans are accumulated in fp64 and
 * rounded to fp32 per element, like torch's CPU cumsum/cumprod, so that indices are reproducible.
 * u_lin: DEVICE float[m] = torch.linspace(0.5/m, 1-0.5/m, m) (:76), supplied by the caller so that its rounding is
 * exactly torch's.  status: DEVICE int or NULL, see NUDF_STATUS_NONFINITE_SAMPLES. */
int nudf_up_sample(int32_t mode, const float* rays_o, const float* rays_d, const float* z, const float* udf,
                   int32_t n_rays, int32_t n, int32_t m, float sample_dist, float inv_s, float beta, float gamma,
                   const float* u_lin, float* new_z, int64_t* inds, int32_t* status, void* stream);
/* sample_pdf(det=True) alone (:66-104): bins [N,n], weights [N,n-1] -> samples [N,m], inds [N,m] */
int nudf_sample_pdf(const float* bins, const float* weights, int32_t n_rays, int32_t n, int32_t m, const float* u_lin,
                    float* samples, int64_t* inds, int32_t* status, void* stream);
/* cat_z_vals merge (:274-290): z_out[N,n+m] sorted union, udf_out gathered likewise (udf/new_udf/udf_out may be
 * NULL for the `last` round).  new_pts[N*m,3] <- o + d*new_z (points to evaluate before the merge), optional. */
int nudf_merge_z(const float* z, const float* new_z, const float* udf, const float* new_udf, int32_t n_rays, int32_t n,
                 int32_t m, float* z_out, float* udf_out, void* stream);
int nudf_points_on_rays(const float* rays_o, const float* rays_d, const float* z, int32_t n_rays, int32_t n,
                        float* pts, void* stream);
/* NeRF++ inverted-sphere inputs and alpha (:161-184): pts4[N*n,4], then alpha = 1-exp(-relu(sigma) dists) */
int nudf_outside_points(const float* rays_o, const float* rays_d, const float* z, int32_t n_rays, int32_t n,
                        int32_t col0, float sample_dist, float* pts4, float* dists, void* stream);

/* --- pixel / patch blending of the fine-tuning stage (replaces patch_projector.pixel_warp / patch_warp +
 * fields.color_blend, models/patch_projector.py:21-166, models/projector_utils.py:8-85, models/fields.py:498-537, as used by
 * render_core, models/udf_renderer_blending.py:431-480).  One call fuses, for every sample point, the projection into each
 * source view, the bilinear gathers (pixel colour and homography-warped patch) and the masked-softmax fusion over views.
 *   pts    [P,3]  sample points (P = n_rays * n_samples, ray-major)
 *   proj   [V,12] row-major 3x4 matrices K[:3,:3] @ w2c[:3,:] of the source views
 *   hom    [V,P,9] row-major plane-induced homographies query pixel -> source pixel, or NULL (pixel blending only)
 *   px     [n_rays,2] pixel coordinates of each ray in the query image (patch centre)
 *   imgs   [V,3,H,W] source images;  logits [P, ld_logits]: blending logits, the first V columns are used
 *   c_pix  [P,3] blended pixel colour;  c_pat [P,(2h+1)^2,3] blended patch colours;  m_pat [P] 1 if any view sees the
 *   whole patch.  Backward: gradients w.r.t. the logits only ([P,V]); everything else is a constant of the graph.
 *   Limits: 1 <= n_views <= 32, 0 <= h_patch <= 5 (patches of at most 11 x 11 = 121 pixels); otherwise -1 and
 *   nudf_last_error(), nothing is launched. */
typedef struct {
  int32_t n_rays, n_samples, n_views, height, width, h_patch;
} nudf_blend_cfg;
int nudf_blend_forward(const nudf_blend_cfg* cfg, const float* pts, const float* proj, const float* hom, const float* px,
                       const float* imgs, const float* logits, int64_t ld_logits, float* c_pix, float* c_pat, float* m_pat,
                       void* stream);
int nudf_blend_backward(const nudf_blend_cfg* cfg, const float* pts, const float* proj, const float* hom, const float* px,
                        const float* imgs, const float* logits, int64_t ld_logits, const float* g_pix, const float* g_pat,
                        float* g_logits, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * ray generation on the device (replaces the per-step tensor algebra of the reference's data loader)
 * ------------------------------------------------------------------------------------------------------------ */
/* gen_random_rays_patches_at (dataset/dataset.py:228-294) without the patch crop: for n pixels (px, py: DEVICE int64, drawn by
 * the caller with torch.randint like the reference) of one image:
 *   rays[n,10] = (origin, unit direction in world space, rgb gathered from image[H,W,3], mask[H,W,3] > 0)
 *   ndc_uv[n,2] = 2 px/(W-1) - 1, 2 py/(H-1) - 1 (may be NULL);  near/far[n] = near_far_from_sphere (:329-335; may be NULL)
 * intrinsics_inv: DEVICE row-major 3x3 (top-left block of intrinsics_all_inv[idx], compact), pose: DEVICE row-major 4x4 c2w. */
int nudf_gen_rays(const float* intrinsics_inv, const float* pose, const int64_t* px, const int64_t* py, int32_t n,
                  const float* image, const float* mask, int32_t H, int32_t W, float* rays, float* ndc_uv, float* near,
                  float* far, void* stream);
/* gen_rays_at (dataset/dataset.py:151-164): rays of the [Hl, Wl] = [H // level, W // level] grid of pixel centres
 * linspace(0, W-1, Wl) x linspace(0, H-1, Hl); rays_o / rays_d [Hl, Wl, 3] (already transposed to image order). */
int nudf_gen_rays_grid(const float* intrinsics_inv, const float* pose, int32_t W, int32_t H, int32_t Wl, int32_t Hl, float* rays_o,
                       float* rays_d, float* near, float* far, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * MeshUDF marching cubes (replaces custom_mc's udf_mc_lewiner; neuraludf_b200/mesh.py drives the stages)
 * ------------------------------------------------------------------------------------------------------------
 * The lattice [n0, n1, n2] (axis 0 slowest) is named by a nudf_lattice.  Cells are named by the flat index of their lower
 * corner; every cell list is sorted ascending.  Normals are unit vectors towards the surface: dense [n0*n1*n2, 3]
 * (idx = NULL) or the sparse rows of the sorted flat indices idx[n_idx] (grid.near_surface_cells); a corner without a row
 * counts as the zero vector.  All buffers are caller-provided; nothing is allocated. */
/* The lattice a MeshUDF or narrow-band kernel reads, flat index (i n1 + j) n2 + k (the descriptor is host memory, the
 * pointers DEVICE): the fp32 array df, or the block-sparse band `store` (nudf_brick_store below; n0 = n1 = n2 = store->n).
 * Exactly one of df and store is set; every dimension is >= 2. */
typedef struct nudf_lattice {
  int32_t n0, n1, n2;
  const float* df;
  const struct nudf_brick_store* store;
} nudf_lattice;
/* flags[t] = 1 when cell cand[t] is active: mean corner udf < avg_t and max <= max_t.  cand = NULL (a df lattice only):
 * cell t of the whole lattice */
int nudf_mc_active(const nudf_lattice* lat, const int64_t* cand, int64_t n_cand, float avg_t, float max_t, uint8_t* flags,
                   void* stream);
/* mask[t] bit c = corner c of cells[t] on the other pseudo-side than the cell's largest-udf corner (c = 4 a0 + 2 a1 + a2) */
int nudf_mc_cell_signs(const nudf_lattice* lat, const int64_t* cells, int64_t n_cells, const int64_t* idx, int64_t n_idx,
                       const float* normals, uint8_t* mask, void* stream);
/* links[t*3+axis] = 2 * (position of the + axis neighbour in cells) + (1 when the shared corners with udf > 0 all disagree,
 * 0 when they all agree), or -1 (no active neighbour, mixed or no evidence) */
int nudf_mc_links(const nudf_lattice* lat, const int64_t* cells, int64_t n_cells, const uint8_t* mask, int64_t* links,
                  void* stream);
/* one polarity per linked component (deterministic union-find with parity; the root cell's corner 0 ends positive):
 * mask_out = mask_in, complemented where the cell flips.  Workspace: parent_ws, hook_ws [n_cells] int64, flag_ws [1] int32.
 * Synchronises the stream (one host read of flag_ws per pass).  stats (HOST int32[2], may be NULL): hooking rounds,
 * pointer-jumping passes.  At most n_cells - 1 hooking rounds; a handful in practice. */
int nudf_mc_polarity(const int64_t* links, int64_t n_cells, const uint8_t* mask_in, int64_t* parent_ws, int64_t* hook_ws,
                     int32_t* flag_ws, uint8_t* mask_out, int32_t* stats, void* stream);
/* triangles per cell (<= 12): each crossing loop is triangulated with no chord lying in a cube face (every edge of a
 * closed surface is shared by exactly two triangles); a loop that admits no such triangulation is fanned around a centre
 * vertex of its own */
int nudf_mc_count(const nudf_lattice* lat, const int64_t* cells, int64_t n_cells, const uint8_t* mask, int32_t* counts,
                  void* stream);
/* keys[3 * (offsets[t] + i) + k] = key of vertex k of triangle i of cells[t]: 3 * corner + axis for a lattice-edge point,
 * 3 * n0 * n1 * n2 + 4 * t + l for the centre vertex of the cell's loop l; offsets = exclusive scan of the counts */
int nudf_mc_emit(const nudf_lattice* lat, const int64_t* cells, int64_t n_cells, const uint8_t* mask, const int64_t* offsets,
                 int64_t* keys, void* stream);
/* verts[n_keys, 3]: lattice-index coordinates of the vertices of the keys: edge points at t = u_a / (u_a + u_b) from the
 * lower corner, loop centres at the mean of their edge points (cells / mask: those given to nudf_mc_emit) */
int nudf_mc_vertices(const nudf_lattice* lat, const int64_t* cells, int64_t n_cells, const uint8_t* mask, const int64_t* keys,
                     int64_t n_keys, float* verts, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Threshold marching cubes (replaces PyMCubes' marching_cubes in the runner's validate_mesh; neuraludf_b200/mesh.py's
 * iso_marching_cubes_index drives the stages).  The MeshUDF construction above on the corner values v = fl32(f - level)
 * (corner positive when v > 0), with no pseudo-signs and no polarity; the lattice is read in place, never shifted.
 * df: DEVICE fp32 lattice [n0, n1, n2]; level must be finite.  Faces are wound so that their normals (right-hand rule)
 * point from the > level side into the <= level side.  All buffers are caller-provided; nothing is allocated.
 * ------------------------------------------------------------------------------------------------------------ */
/* flags[g] (g < n0 * n1 * n2) = 1 when the cell with lower corner g has a corner with v > 0, one with v <= 0 and none NaN */
int nudf_iso_active(const float* df, int32_t n0, int32_t n1, int32_t n2, float level, uint8_t* flags, void* stream);
/* triangles per cell (<= 12), as nudf_mc_count */
int nudf_iso_count(const float* df, int32_t n0, int32_t n1, int32_t n2, float level, const int64_t* cells, int64_t n_cells,
                   int32_t* counts, void* stream);
/* vertex keys of the triangles, as nudf_mc_emit: 3 * corner + axis, then 3 * n0 * n1 * n2 + 4 * t + l for loop centres */
int nudf_iso_emit(const float* df, int32_t n0, int32_t n1, int32_t n2, float level, const int64_t* cells, int64_t n_cells,
                  const int64_t* offsets, int64_t* keys, void* stream);
/* verts[n_keys, 3] fp64 lattice-index coordinates: edge points at t = v_a / (v_a - v_b) from the lower corner (fp64 from the
 * fp32 v, no contraction), loop centres at the mean of their loop's edge points summed in loop order */
int nudf_iso_vertices(const float* df, int32_t n0, int32_t n1, int32_t n2, float level, const int64_t* cells, int64_t n_cells,
                      const int64_t* keys, int64_t n_keys, double* verts, void* stream);
/* The same stages on a nudf_lattice (the flat array or a brick store; the nudf_iso_* above are their df form, the same
 * kernels).  The active cells without a scan of every cell: the storage positions (df: the flat indices; a store: coarse,
 * then the brick slots, as nudf_sb_flat numbers them) are taken in n_seg = ceil(positions / NUDF_ISO_SEG) segments.  Each
 * position holding a lattice point with v <= 0 emits the active cells (as nudf_iso_active defines them) of which it is the
 * lowest corner with v <= 0: counts[seg] = the segment's cells; cells[offsets[seg] ...] = them, in position order
 * (offsets = exclusive scan of the counts).  Sorted, they are nonzero(nudf_iso_active) of the lattice's values, with no
 * condition on the field: every active cell has a corner with v <= 0, which is finite and so stored. */
#define NUDF_ISO_SEG 256
int nudf_iso_lat_cells_count(const nudf_lattice* lat, float level, int64_t n_seg, int32_t* counts, void* stream);
int nudf_iso_lat_cells_emit(const nudf_lattice* lat, float level, int64_t n_seg, const int64_t* offsets, int64_t* cells,
                            void* stream);
int nudf_iso_lat_count(const nudf_lattice* lat, float level, const int64_t* cells, int64_t n_cells, int32_t* counts,
                       void* stream);
int nudf_iso_lat_emit(const nudf_lattice* lat, float level, const int64_t* cells, int64_t n_cells, const int64_t* offsets,
                      int64_t* keys, void* stream);
int nudf_iso_lat_vertices(const nudf_lattice* lat, float level, const int64_t* cells, int64_t n_cells, const int64_t* keys,
                          int64_t n_keys, double* verts, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Point-cloud evaluation (the DTU / DeepFashion3D Chamfer protocols; neuraludf_b200/evaluate.py drives the stages)
 * ------------------------------------------------------------------------------------------------------------
 * Points are DEVICE fp64 [n, 3]; all buffers are caller-provided, nothing is allocated.  Host arrays are marked HOST. */
/* counts[f] = samples of triangle f of the scripts' surface sampling (0 when area2 == 0) */
int nudf_pc_sample_count(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, double density,
                         int64_t* counts, void* stream);
/* points[offsets[f] + s] = sample s of triangle f (row-major over i, j); offsets = exclusive scan of the counts */
int nudf_pc_sample_emit(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, double density,
                        const int64_t* offsets, double* points, void* stream);
/* keys[t] = (cx * dims[1] + cy) * dims[2] + cz, c = floor((p - lo) / cell) clamped to [0, dims - 1] (lo, dims: HOST [3]) */
int nudf_pc_cell_keys(const double* points, int64_t n, const double* lo, double cell, const int64_t* dims, int64_t* keys,
                      void* stream);
/* radius graph over n points of rank 0..n-1 sorted by cell: sorted_points[s] = point of rank order[s], sorted_keys[s] its key;
 * cells[n_cells] the distinct keys ascending, cell_start[n_cells + 1] their first sorted positions.  Neighbours of rank v:
 * ranks u < v with (dx^2 + dy^2) + dz^2 <= radius * radius; cell must be > radius (adjacent cells only are scanned).
 * counts[v] = their number; nbr[offsets[v] ...] = their ranks (offsets [n + 1]: exclusive scan of the counts) */
int nudf_pc_radius_count(const double* sorted_points, const int64_t* order, const int64_t* sorted_keys, int64_t n,
                         const int64_t* cells, const int64_t* cell_start, int64_t n_cells, const double* lo, double cell,
                         const int64_t* dims, double radius, int32_t* counts, void* stream);
int nudf_pc_radius_emit(const double* sorted_points, const int64_t* order, const int64_t* sorted_keys, int64_t n,
                        const int64_t* cells, const int64_t* cell_start, int64_t n_cells, const double* lo, double cell,
                        const int64_t* dims, double radius, const int64_t* offsets, int32_t* nbr, void* stream);
/* the scripts' greedy downsampling: state[v] = 1 (kept) / 2 (dropped) -- the lexicographically-first maximal independent set
 * in rank order, in parallel rounds.  Workspace flag_ws [1] int32.  Synchronises the stream (one host read per round).
 * rounds (HOST int32, may be NULL): the number of rounds */
int nudf_pc_greedy_mis(const int64_t* offsets, const int32_t* nbr, int64_t n, uint8_t* state, int32_t* flag_ws,
                       int32_t* rounds, void* stream);
/* codes[t] = 63-bit Morton code of floor((p - lo) * scale) clamped to [0, 2^21 - 1] per axis (lo: HOST [3]) */
int nudf_pc_morton(const double* points, int64_t n, const double* lo, double scale, int64_t* codes, void* stream);
/* AABBs of the implicit complete binary tree over 32-point leaves of the sorted targets: boxes [2 n_leaves - 1, 6]
 * (lo xyz, hi xyz; node i has children 2i+1, 2i+2; leaf l is node n_leaves - 1 + l); n_leaves a power of two >= n / 32 */
int nudf_pc_bvh_build(const double* sorted_targets, int64_t n, int64_t n_leaves, double* boxes, void* stream);
/* dist[q] = exact nearest distance sqrt((dx^2 + dy^2) + dz^2) from queries[q] to the targets when it is < max_dist, else +inf
 * (max_dist = +inf: unbounded).  query_order (may be NULL) = the processing order of the queries (Morton order for coherence) */
int nudf_pc_nearest(const double* queries, int64_t n_queries, const int64_t* query_order, const double* sorted_targets,
                    int64_t n_targets, const double* boxes, int64_t n_leaves, double max_dist, double* dist, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * DTU mesh cleaning by masks and visual hull (evaluation/clean_dtu_mesh.py; neuraludf_b200/clean.py drives the stages)
 * ------------------------------------------------------------------------------------------------------------
 * Caller-provided buffers only; host arrays are marked HOST. */
/* packed[v, y, w] bit b = (D(v, y, 32 w + b) > 128), or < 128 when below != 0, for columns < width (other bits 0), where
 * D = the grayscale dilation of masks [n_views, height, width] uint8 by the element whose row i covers columns
 * [row_lo[i], row_hi[i]) (HOST [kh]; empty when row_hi <= row_lo): D(y, x) = max of masks(y + i - anchor_y, x + j - anchor_x)
 * over the element, pixels outside the image not contributing.  packed: [n_views, height, ceil(width / 32)] uint32.
 * kh, kw <= 255. */
int nudf_cl_dilate(const uint8_t* masks, int32_t n_views, int32_t height, int32_t width, const int32_t* row_lo,
                   const int32_t* row_hi, int32_t kh, int32_t kw, int32_t anchor_x, int32_t anchor_y, int32_t below,
                   uint32_t* packed, void* stream);
/* counts[t] = number of views v (mats: DEVICE fp64 [n_views, 3, 4], n_views <= 512) in which points[t] projects to
 * u = rint(s0 / s2) + 1, v = rint(s1 / s2) + 1 (s = ((m0 x + m1 y) + m2 z) + m3 per row, fp64, half to even) with
 * border <= u <= width - border, border <= v <= height - border and the packed mask, padded by a ring of ones, set at (v, u) */
int nudf_cl_vote(const double* points, int64_t n, const double* mats, int32_t n_views, const uint32_t* packed,
                 int32_t height, int32_t width, int32_t border, int32_t* counts, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Narrow-band lattice evaluation, coarse to fine (neuraludf_b200/grid.py udf_band drives the levels)
 * ------------------------------------------------------------------------------------------------------------
 * The N^3 lattice, flat index (i * N + j) * N + k.  The stride-s lattice holds the coordinates 0, s, 2 s, ... and N - 1 per
 * axis; a block of stride s is the box [a, min(a + s, N - 1)] per axis (a a multiple of s below N - 1),
 * nb = ceil((N - 1) / s) per axis, numbered (bx * nb + by) * nb + bz.  The coordinates and the block test's spacing rule
 * are named by a nudf_band_coords.  Caller-provided buffers only. */
/* The band lattice's coordinates (host memory).  Cube (ax[0..2] NULL): [-1,1]^3, point i at fl(fl(i * fl32(voxel)) - 1)
 * per axis, as grid.lattice_points makes them.  Table (ax[0..2] all set): three DEVICE fp32 tables [N] (any box; grid.iso_band
 * passes the torch.linspace tables of the dense threshold sweep), point (i, j, k) at (ax[0][i], ax[1][j], ax[2][k]);
 * h[a] >= 0 the largest step of table a, pad >= 0 (the block test's only). */
typedef struct nudf_band_coords {
  double voxel;
  const float* ax[3];
  double h[3];
  double pad;
} nudf_band_coords;
/* idx / pts [m^3] (m = ceil((N - 1) / s) + 1): the stride-s lattice in (x, y, z) lexicographic order */
int nudf_nb_sublattice(int32_t n, int32_t s, const nudf_band_coords* co, int64_t* idx, float* pts, void* stream);
/* flags[nb^3] (may be NULL) = 1 for the kept blocks of stride s on the cubic lattice `lat` (N = n0 = n1 = n2): candidates
 * (every block when parent_flags is NULL, else the blocks inside a kept block of stride parent_s) with a NaN corner or
 * min(corner df) - lipschitz r < tau in fp64, r = half the box diagonal.  Cube: r in voxels, with slack
 * (r + 1e-6 relative + 1e-6, tau + 1e-6 relative) against rounding; edge slopes |du| / (e_a voxel).  Table (a df lattice
 * only): r from the block's table-coordinate box (fp64, |ax[hi] - ax[lo]| per axis), enlarged by 1e-6 relative plus pad,
 * and tau used as given (the caller's slack included); edge slopes |du| / (e_a h_a).  Candidates' corners must have been
 * evaluated.  max_slope (DEVICE uint32[1], fp32 bits, zeroed by the caller) is raised to the largest |du| / (edge length)
 * over the candidates' box edges with finite ends */
int nudf_nb_block_test(const nudf_lattice* lat, int32_t s, const uint8_t* parent_flags, int32_t parent_s,
                       const nudf_band_coords* co, double lipschitz, double tau, uint8_t* flags, uint32_t* max_slope,
                       void* stream);
/* nudf_nb_block_test on any lattice with either coordinate form: the table form on a brick store too
 * (grid.iso_band_sparse), the same test on the same corner values */
int nudf_nb_lat_block_test(const nudf_lattice* lat, int32_t s, const uint8_t* parent_flags, int32_t parent_s,
                           const nudf_band_coords* co, double lipschitz, double tau, uint8_t* flags, uint32_t* max_slope,
                           void* stream);
/* counts[i] = the points block kept[i] of stride s emits: the stride-t lattice (t divides s) in its closed box, less the
 * stride-s lattice, less the points that a lower-numbered kept block (flags) also holds.  kept: ascending block numbers */
int nudf_nb_count(const uint8_t* flags, int32_t n, int32_t s, int32_t t, const int64_t* kept, int64_t n_kept,
                  int32_t* counts, void* stream);
/* idx / pts[offsets[i] ...] = those points of block kept[i] in (x, y, z) lexicographic order; offsets = exclusive scan */
int nudf_nb_emit(const uint8_t* flags, int32_t n, int32_t s, int32_t t, const int64_t* kept, int64_t n_kept,
                 const int64_t* offsets, const nudf_band_coords* co, int64_t* idx, float* pts, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Block-sparse narrow band (neuraludf_b200/grid.py udf_band_sparse drives the levels, mesh.py udf_mesh_sparse meshes it)
 * ------------------------------------------------------------------------------------------------------------
 * The N^3 lattice of the nudf_nb_* entry points held without an N^3 array (a nudf_lattice with `store` set).  The points of the stride-c lattice (0, c, 2 c,
 * ... and N - 1 per axis; mc = ceil((N - 1) / c) + 1) live in the dense array coarse[mc^3], point (i, j, k) at
 * (ci * mc + cj) * mc + ck with ci = i / c, or mc - 1 for i = N - 1.  Every other point lives in a brick of NUDF_BRICK^3
 * points: brick (i / 8, j / 8, k / 8), numbered (bx * nbk + by) * nbk + bz (nbk = ceil(N / 8)), has slot dir[brick] (-1:
 * none), and the point is bricks[slot * 512 + ((i % 8) * 8 + j % 8) * 8 + k % 8].  keys[slot] is the brick number of
 * each slot, ascending.  A point of a brick without a slot reads +inf, as do the slots of the stride-c points inside
 * bricks (they are read from coarse).  Storage positions (nudf_sb_flat): [0, mc^3) for coarse, mc^3 + slot * 512 + local
 * for the bricks.  All pointers DEVICE; the descriptor itself is host memory. */
#define NUDF_BRICK 8
typedef struct nudf_brick_store {
  int32_t n, c, mc, nbk;
  int64_t n_bricks;
  float* coarse;          /* [mc^3] */
  int32_t* dir;           /* [nbk^3] */
  float* bricks;          /* [n_bricks * 512] */
  const int64_t* keys;    /* [n_bricks] */
} nudf_brick_store;
/* marks[b] = 1 (marks: [nbk^3], zeroed by the caller) for every brick b that meets the closed box of a kept block of
 * stride s (flags [ceil((N - 1) / s)^3], nudf_nb_block_test's); s must be a multiple of the store's c */
int nudf_sb_mark(const nudf_brick_store* st, int32_t s, const uint8_t* flags, int32_t* marks, void* stream);
/* writes vals[t] to lattice point idx[t] (flat); -1 when a point is neither on the stride-c lattice nor in a brick with a
 * slot (nothing is written then) */
int nudf_sb_store(const nudf_brick_store* st, const int64_t* idx, const float* vals, int64_t n, int32_t* missing, void* stream);
/* out[t] = the value of lattice point idx[t] (flat) */
int nudf_sb_gather(const nudf_brick_store* st, const int64_t* idx, int64_t n, float* out, void* stream);
/* out[t] = the flat lattice index of storage position pos[t] */
int nudf_sb_flat(const nudf_brick_store* st, const int64_t* pos, int64_t n, int64_t* out, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Mesh post-processing (neuraludf_b200/mesh_post.py drives the steps; sorting, unique and compaction in torch)
 * ------------------------------------------------------------------------------------------------------------
 * verts: fp64 [V,3]; faces and edges: int64 rows.  All fp64 arithmetic is correctly rounded per operation with no
 * contraction.  Caller-provided buffers only. */
/* per face i: out_faces[i] = remap[faces[i]] (faces[i] when remap is NULL), sorted_faces[i] = its ascending triple,
 * edge_codes[3 i + k] = (lo * V + hi) * 2 + (1 when the face runs hi -> lo) of its edge (k, k + 1 mod 3), and
 * nondegenerate[i] = 1 when |a|, |b|, |a x b| / |a| and |a x b| / |b| all exceed 1e-8 (a = v1 - v0, b = v2 - v0, in the
 * remapped vertices).  V < 2^30 */
int nudf_mp_faces(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, const int64_t* remap,
                  int64_t* out_faces, int64_t* sorted_faces, int64_t* edge_codes, uint8_t* nondegenerate, void* stream);
/* boundary edges [B,2] (u < v, ascending) with the CSR (rowptr [V+1], cols ascending per row) of boundary neighbours:
 * counts[i] = the faces edge i emits: 1 or 2 when it is the smallest edge of a boundary component that is a simple cycle of 3
 * or 4 vertices, else 0 */
int nudf_mp_hole_count(const int64_t* edges, int64_t n_edges, const int64_t* rowptr, const int64_t* cols, int64_t n_verts,
                       int32_t* counts, void* stream);
/* faces[offsets[i] ...] = those faces (offsets = exclusive scan of counts): they traverse edge i against its direction in its
 * face (dirs[i] = 1: the face runs v -> u); a quad is split along its shorter diagonal (squared fp64 length), a tie along the
 * diagonal through the smallest vertex */
int nudf_mp_hole_emit(const double* verts, const int64_t* edges, const uint8_t* dirs, int64_t n_edges, const int64_t* rowptr,
                      const int64_t* cols, int64_t n_verts, const int64_t* offsets, int64_t* faces, void* stream);
/* one Jacobi step of border smoothing: for each vertex b in border, verts_out[b] = v + lambda (s / count - v), v =
 * verts_in[b], s = its CSR neighbours' verts_in summed in ascending order.  Other rows of verts_out are not written */
int nudf_mp_smooth_step(const double* verts_in, double* verts_out, const int64_t* border, int64_t n_border,
                        const int64_t* rowptr, const int64_t* cols, double lambda, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Gradient branch of get_mesh_udf_fast (neuraludf_b200/extract_mesh.py drives the steps; the CSR sort in torch)
 * ------------------------------------------------------------------------------------------------------------
 * Every fp64 / fp32 operation is correctly rounded on its own, no contraction (acos aside). */
/* normals[V,3] fp32 <- the angle-weighted vertex normals of the fp64 mesh (verts [V,3], faces [F,3]): per face the unit
 * normal of (v1 - v0) x (v2 - v0) times the angle at each corner (face_terms: workspace of 9 F doubles), summed per vertex
 * over incidences [3F] = corner * F + face in the CSR order of rowptr [V+1] (the caller sorts them by (vertex, corner,
 * face)), divided by max(|sum|, 1e-300) and rounded to fp32.  A vertex without faces gets 0.  Two launches. */
int nudf_mg_vertex_normals(const double* verts, int64_t n_verts, const int64_t* faces, int64_t n_faces, const int64_t* rowptr,
                           const int64_t* incidences, double* face_terms, float* normals, void* stream);
/* fp32 verts / normals [V,3].  s1 == s2 == NULL: probes [2V,3] <- verts + eps n, then verts - eps n.  Otherwise (s1, s2 [V]:
 * the udf at those probes): new_verts [V,3] <- (v - (eps s1) n) + (eps s2) n, and next_indices [7V] <- the flat index of
 * trunc((x + 1) / fl32(2 / (n_mc - 1))) per axis and its six neighbours clamped to [0, n_mc - 1] along one axis (+x, +y,
 * +z, -x, -y, -z), block-major; a NaN or out-of-range quotient gives INT64_MIN, the index arithmetic wraps.  One launch. */
int nudf_mg_refine(const float* verts, const float* normals, int64_t n_verts, float eps, const float* s1, const float* s2,
                   int32_t n_mc, float* probes, float* new_verts, int64_t* next_indices, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Connected components of a mesh's faces (neuraludf_b200/clean.py face_components; sizes and selection in torch)
 * ------------------------------------------------------------------------------------------------------------ */
/* keys [n_keys] ascending: edge keys lo * V + hi (nudf_mp_faces' edge codes >> 1); key_face[e] in [0, n_faces): the face
 * of key slot e.  A key occurring exactly twice, from two different faces, joins those faces (trimesh face_adjacency).
 * label[F] <- the smallest face index of each face's component; paired[F] <- 1 when the face is in at least one such pair.
 * Three launches (init, hook, compress), no host synchronisation; the labels do not depend on scheduling. */
int nudf_cc_label(const int64_t* keys, const int64_t* key_face, int64_t n_keys, int64_t n_faces, int64_t* label,
                  uint8_t* paired, void* stream);

/* ------------------------------------------------------------------------------------------------------------
 * Colour loss of the training step (replaces loss/loss.py ColorLoss with loss/patch_metric.py; neuraludf_b200/loss.py)
 * ------------------------------------------------------------------------------------------------------------
 * fp32, row-major, contiguous.  N rays, P = (2 h_patch + 1)^2 patch pixels (row-major, the patch's x fastest). */
#define NUDF_PATCH_L1 0
#define NUDF_PATCH_SSD 1
#define NUDF_PATCH_SSIM 2
#define NUDF_PATCH_NCC 3
/* floats of the workspace both calls take (the forward writes it, the backward reads it); ws must be 8-byte aligned */
#define NUDF_COLOR_LOSS_WS_FLOATS(n_rays) (4 * (int64_t)(n_rays) + 8)
typedef struct nudf_color_loss_args {
  int32_t n_rays;            /* N, 1 .. 16384 */
  int32_t h_patch;           /* 1 .. 15 */
  int32_t patch_type;        /* NUDF_PATCH_* */
  float weights[4];          /* color_base, color, color_pixel, color_patch weights (loss.py:119-123) */
  const float* color_base;   /* [N,3] each; NULL: the term is absent */
  const float* color;
  const float* color_pixel;
  const float* gt_color;     /* [N,3] */
  const float* pixel_mask;   /* [N] or NULL: denominator sum(mask) + 1e-4 of color_base / color, else the mean over N * 3 */
  const float* patch_colors; /* [N,P,3]; NULL: no patch term */
  const float* gt_patch_colors; /* [N,P,3] */
  const uint8_t* patch_mask; /* [N] 0/1 or NULL: denominator count + 1e-4 of color_pixel, and the patch term's mask (required
                              * with it) */
  const float* window;       /* [P] Gaussian window of patch_metric.create_window (ssim / ncc) */
} nudf_color_loss_args;
/* losses[5] <- loss, color_base_loss, color_loss, color_pixel_loss, color_patch_loss (absent terms 0); kept[N] (with a patch
 * term) <- 1 for the masked rays left after excluding the first int(0.3f * count(mask)) rays of the descending order of
 * error * mask (NaN largest, equal keys in ray order; loss.py:78-84).  Two launches, no host synchronisation. */
int nudf_color_loss_forward(const nudf_color_loss_args* args, float* losses, uint8_t* kept, float* ws, void* stream);
/* d_* (same shapes as the predictions; NULL: not written) <- gradients of  sum_i losses_bar[i] * losses[i].  losses_bar:
 * HOST array of 5 DEVICE pointers to one float each, NULL = zero.  kept and ws: as the forward left them. */
int nudf_color_loss_backward(const nudf_color_loss_args* args, const float* const* losses_bar, const uint8_t* kept,
                             const float* ws, float* d_color_base, float* d_color, float* d_color_pixel, float* d_patch_colors,
                             void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NUDF_H_ */

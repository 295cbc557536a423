"""ctypes binding of libnudf.so (the C-ABI declared in include/nudf.h).

There is NO fallback: if the library is missing or a call fails, a RuntimeError is raised.  The library is built
in-tree by `python -m neuraludf_b200.build` (nvcc, sm_90a) and travels to the GPU box with the repository.
"""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("NUDF_LIB_PATH", os.path.join(HERE, "libnudf.so"))   # override: A/B builds of the library
MAX_LAYERS = 16

c_float_p = ctypes.POINTER(ctypes.c_float)
c_i64_p = ctypes.POINTER(ctypes.c_int64)
c_void_p = ctypes.c_void_p
FP_ARR = c_void_p * MAX_LAYERS


class UdfDesc(ctypes.Structure):
    _fields_ = [("n_lin", ctypes.c_int32), ("d_in", ctypes.c_int32), ("multires", ctypes.c_int32),
                ("d_out", ctypes.c_int32), ("skip_layer", ctypes.c_int32), ("scale", ctypes.c_float),
                ("in_dim", ctypes.c_int32 * MAX_LAYERS), ("out_dim", ctypes.c_int32 * MAX_LAYERS),
                ("weight_g", FP_ARR), ("weight_v", FP_ARR), ("bias", FP_ARR)]


class ColorDesc(ctypes.Structure):
    _fields_ = [("n_lin", ctypes.c_int32), ("d_feature", ctypes.c_int32), ("d_hidden", ctypes.c_int32),
                ("d_out", ctypes.c_int32), ("n_blend", ctypes.c_int32), ("multires_view", ctypes.c_int32),
                ("base_g", FP_ARR), ("base_v", FP_ARR), ("base_b", FP_ARR),
                ("main_g", FP_ARR), ("main_v", FP_ARR), ("main_b", FP_ARR)]


class NerfDesc(ctypes.Structure):
    _fields_ = [("D", ctypes.c_int32), ("W", ctypes.c_int32), ("d_in", ctypes.c_int32), ("multires", ctypes.c_int32),
                ("multires_view", ctypes.c_int32), ("skip", ctypes.c_int32),
                ("pts_w", FP_ARR), ("pts_b", FP_ARR),
                ("views_w", c_void_p), ("views_b", c_void_p), ("feature_w", c_void_p), ("feature_b", c_void_p),
                ("alpha_w", c_void_p), ("alpha_b", c_void_p), ("rgb_w", c_void_p), ("rgb_b", c_void_p)]


class RenderCfg(ctypes.Structure):
    _fields_ = [("n_rays", ctypes.c_int32), ("n_samples", ctypes.c_int32), ("n_outside", ctypes.c_int32),
                ("sample_dist", ctypes.c_float), ("cos_anneal_ratio", ctypes.c_float),
                ("has_cos_anneal", ctypes.c_int32), ("flip_saturation", ctypes.c_float),
                ("sparse_scale_factor", ctypes.c_float), ("use_norm_grad_for_cosine", ctypes.c_int32),
                ("has_background_rgb", ctypes.c_int32), ("background_rgb", ctypes.c_float * 3),
                ("alpha_rule", ctypes.c_int32)]


RENDER_OUT_FIELDS = ["color_base", "color", "depth", "normals", "weights", "weight_sum", "weight_sum_fg_bg",
                     "ray_sums", "gradient_mag", "true_cos", "vis_prob", "alpha", "alpha_plus", "alpha_minus",
                     "alpha_occ", "raw_occ", "inside_sphere", "gradients_flip", "status"]
STATUS_NONFINITE_SAMPLES, STATUS_NONFINITE_RENDER = 1, 2


class RenderOut(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in RENDER_OUT_FIELDS]


VIEW_OUT_FIELDS = ["color", "color_pixel", "depth", "normal", "weight_sum"]


class ViewOut(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in VIEW_OUT_FIELDS]


class BlendCfg(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int32) for n in ("n_rays", "n_samples", "n_views", "height", "width", "h_patch")]


class RenderBar(ctypes.Structure):
    _fields_ = [(n, c_void_p) for n in ("color_base", "color", "depth", "weight_sum", "weight_sum_fg_bg", "weights",
                                        "ray_sums")]


class BrickStore(ctypes.Structure):
    """nudf_brick_store (include/nudf.h): the block-sparse narrow band's layout, device pointers"""
    _fields_ = [("n", ctypes.c_int32), ("c", ctypes.c_int32), ("mc", ctypes.c_int32), ("nbk", ctypes.c_int32),
                ("n_bricks", ctypes.c_int64), ("coarse", c_void_p), ("dir", c_void_p), ("bricks", c_void_p),
                ("keys", c_void_p)]


BRICK = 8   # NUDF_BRICK
COMPACT_SEG = 256   # NUDF_COMPACT_SEG
PT_MAX_VIEWS, PT_MAX_CAND = 64, 8      # NUDF_PT_MAX_VIEWS, NUDF_PT_MAX_CAND


class Lattice(ctypes.Structure):
    """nudf_lattice (include/nudf.h): the lattice a kernel reads, the fp32 array df or a brick store (exactly one set)"""
    _fields_ = [("n0", ctypes.c_int32), ("n1", ctypes.c_int32), ("n2", ctypes.c_int32), ("df", c_void_p),
                ("store", ctypes.POINTER(BrickStore))]


class BandCoords(ctypes.Structure):
    """nudf_band_coords (include/nudf.h): the band lattice's cube coordinates (voxel), or its three fp32 tables with their
    largest steps h and the block test's pad"""
    _fields_ = [("voxel", ctypes.c_double), ("ax", c_void_p * 3), ("h", ctypes.c_double * 3), ("pad", ctypes.c_double)]


PATCH_TYPES = {"l1": 0, "ssd": 1, "ssim": 2, "ncc": 3}


def color_loss_ws_floats(n_rays):
    """NUDF_COLOR_LOSS_WS_FLOATS of include/nudf.h"""
    return 4 * n_rays + 8


class ColorLossArgs(ctypes.Structure):
    _fields_ = [("n_rays", ctypes.c_int32), ("h_patch", ctypes.c_int32), ("patch_type", ctypes.c_int32),
                ("weights", ctypes.c_float * 4)] + [(n, c_void_p) for n in (
                    "color_base", "color", "color_pixel", "gt_color", "pixel_mask", "patch_colors", "gt_patch_colors",
                    "patch_mask", "window")]


LAUNCH_FAMILIES = ["udf_fwd_chain_fused", "tc_layer_reverse_sweep", "tc_layer_tangent", "tc_layer_backward", "tc_layer_other",
                   "tc_weight_gradient", "ffma_gemm", "ray_kernels", "elementwise", "udf_bwd_chain_fused"]

_lib = None

_SIGNATURES = {
    "nudf_abi_version": (ctypes.c_int, []),
    "nudf_last_error": (ctypes.c_char_p, []),
    "nudf_set_engine": (ctypes.c_int, [ctypes.c_int]),
    "nudf_get_engine": (ctypes.c_int, []),
    "nudf_launch_count": (ctypes.c_int64, []),
    "nudf_launch_family_count": (ctypes.c_int, []),
    "nudf_set_launch_timing": (ctypes.c_int, [ctypes.c_int]),
    "nudf_read_launch_timing": (ctypes.c_int, [c_void_p, c_void_p]),
    "nudf_set_tc_mask": (ctypes.c_int, [ctypes.c_int]),
    "nudf_get_tc_mask": (ctypes.c_int, []),
    "nudf_default_tc_mask": (ctypes.c_int, []),
    "nudf_tc_image_elems": (ctypes.c_int64, [ctypes.c_int32, ctypes.c_int32, ctypes.c_int32]),
    "nudf_tc_prepare_weights": (ctypes.c_int, [c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                               ctypes.c_int32, c_void_p, c_void_p]),
    "nudf_dense_forward_tc": (ctypes.c_int, [c_void_p, ctypes.c_int64, c_void_p, ctypes.c_int32, c_void_p, c_void_p,
                                             ctypes.c_int64, ctypes.c_int64, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                             c_void_p]),
    "nudf_wgrad": (ctypes.c_int, [c_void_p, ctypes.c_int64, c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_int32,
                                  ctypes.c_int64, c_void_p, ctypes.c_int64, ctypes.c_int32, c_void_p]),
    "nudf_blend_forward": (ctypes.c_int, [c_void_p] * 7 + [ctypes.c_int64] + [c_void_p] * 4),
    "nudf_blend_backward": (ctypes.c_int, [c_void_p] * 7 + [ctypes.c_int64] + [c_void_p] * 4),
    "nudf_dense_forward": (ctypes.c_int, [c_void_p, ctypes.c_int64, c_void_p, ctypes.c_int64, c_void_p, c_void_p,
                                          ctypes.c_int64, ctypes.c_int64, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                          c_void_p]),
    "nudf_udf_folded_floats": (ctypes.c_int64, [c_void_p]),
    "nudf_udf_fold_weights": (ctypes.c_int, [c_void_p, c_void_p, c_void_p]),
    "nudf_udf_ctx_floats": (ctypes.c_int64, [c_void_p, ctypes.c_int64, ctypes.c_int]),
    "nudf_udf_scratch_floats": (ctypes.c_int64, [c_void_p, ctypes.c_int64]),
    "nudf_udf_forward": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_int64, c_void_p, ctypes.c_int64,
                                        c_void_p, c_void_p, c_void_p]),
    "nudf_udf_forward_split": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_int64, c_void_p, c_void_p, ctypes.c_int64,
                                              c_void_p, c_void_p, c_void_p]),
    "nudf_udf_backward_split": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_int64, c_void_p, c_void_p, ctypes.c_int64,
                                               c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nudf_udf_value": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_int64, c_void_p, c_void_p, c_void_p]),
    "nudf_udf_backward": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_int64, c_void_p, ctypes.c_int64,
                                         c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nudf_udf_unfold_grads": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nudf_color_folded_floats": (ctypes.c_int64, [c_void_p]),
    "nudf_color_fold_weights": (ctypes.c_int, [c_void_p, c_void_p, c_void_p]),
    "nudf_color_ctx_floats": (ctypes.c_int64, [c_void_p, ctypes.c_int64]),
    "nudf_color_scratch_floats": (ctypes.c_int64, [c_void_p, ctypes.c_int64]),
    "nudf_color_forward": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_int32, c_void_p,
                                          ctypes.c_int64, ctypes.c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p]),
    "nudf_color_backward": (ctypes.c_int, [c_void_p, c_void_p, ctypes.c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_void_p, ctypes.c_int64, c_void_p, c_void_p, c_void_p]),
    "nudf_color_unfold_grads": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nudf_nerf_image_floats": (ctypes.c_int64, [c_void_p]),
    "nudf_nerf_prepare": (ctypes.c_int, [c_void_p, c_void_p, c_void_p]),
    "nudf_nerf_ctx_floats": (ctypes.c_int64, [c_void_p, ctypes.c_int64]),
    "nudf_nerf_scratch_floats": (ctypes.c_int64, [c_void_p, ctypes.c_int64]),
    "nudf_nerf_forward": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_int32, ctypes.c_int64, c_void_p,
                                         c_void_p, c_void_p, c_void_p]),
    "nudf_nerf_backward": (ctypes.c_int, [c_void_p, c_void_p, ctypes.c_int64, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p, c_void_p]),
    "nudf_ray_points": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_float,
                                       c_void_p, c_void_p, c_void_p, c_void_p]),
    "nudf_render_composite_forward": (ctypes.c_int, [c_void_p] * 2 + [c_void_p] * 5 + [ctypes.c_int64] + [c_void_p] * 7),
    "nudf_render_view_forward": (ctypes.c_int, [c_void_p] * 2 + [c_void_p] * 5 + [ctypes.c_int64] + [c_void_p] * 8),
    "nudf_render_composite_backward": (ctypes.c_int, [c_void_p] * 2 + [c_void_p] * 5 + [ctypes.c_int64] + [c_void_p] * 14),
    "nudf_up_sample": (ctypes.c_int, [ctypes.c_int32, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_int32,
                                      ctypes.c_int32, ctypes.c_int32, ctypes.c_float, ctypes.c_float, ctypes.c_float,
                                      ctypes.c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nudf_sample_pdf": (ctypes.c_int, [c_void_p, c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32, c_void_p,
                                       c_void_p, c_void_p, c_void_p, c_void_p]),
    "nudf_merge_z": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_int32, ctypes.c_int32,
                                    ctypes.c_int32, c_void_p, c_void_p, c_void_p]),
    "nudf_points_on_rays": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_int32, ctypes.c_int32, c_void_p,
                                           c_void_p]),
    "nudf_gen_rays": (ctypes.c_int, [c_void_p] * 4 + [ctypes.c_int32] + [c_void_p] * 2 + [ctypes.c_int32] * 2 + [c_void_p] * 5),
    "nudf_gen_rays_grid": (ctypes.c_int, [c_void_p] * 2 + [ctypes.c_int32] * 4 + [c_void_p] * 5),
    "nudf_outside_points": (ctypes.c_int, [c_void_p, c_void_p, c_void_p, ctypes.c_int32, ctypes.c_int32, ctypes.c_int32,
                                           ctypes.c_float, c_void_p, c_void_p, c_void_p]),
    "nudf_mc_active": (ctypes.c_int, [c_void_p] * 2 + [ctypes.c_int64, ctypes.c_float, ctypes.c_float] + [c_void_p] * 2),
    "nudf_mc_cell_signs": (ctypes.c_int, [c_void_p] * 2 + [ctypes.c_int64, c_void_p, ctypes.c_int64] + [c_void_p] * 3),
    "nudf_mc_links": (ctypes.c_int, [c_void_p] * 2 + [ctypes.c_int64] + [c_void_p] * 3),
    "nudf_mc_polarity": (ctypes.c_int, [c_void_p, ctypes.c_int64] + [c_void_p] * 7),
    "nudf_mc_count": (ctypes.c_int, [c_void_p] * 2 + [ctypes.c_int64] + [c_void_p] * 3),
    "nudf_mc_emit": (ctypes.c_int, [c_void_p] * 2 + [ctypes.c_int64] + [c_void_p] * 4),
    "nudf_mc_vertices": (ctypes.c_int, [c_void_p] * 2 + [ctypes.c_int64] + [c_void_p] * 2 + [ctypes.c_int64] + [c_void_p] * 2),
    "nudf_pc_sample_count": (ctypes.c_int, [c_void_p, ctypes.c_int64, c_void_p, ctypes.c_int64, ctypes.c_double, c_void_p,
                                            c_void_p]),
    "nudf_pc_sample_emit": (ctypes.c_int, [c_void_p, ctypes.c_int64, c_void_p, ctypes.c_int64, ctypes.c_double, c_void_p,
                                           c_void_p, c_void_p]),
    "nudf_pc_cell_keys": (ctypes.c_int, [c_void_p, ctypes.c_int64, c_void_p, ctypes.c_double, c_void_p, c_void_p, c_void_p]),
    "nudf_pc_radius_count": (ctypes.c_int, [c_void_p] * 3 + [ctypes.c_int64] + [c_void_p] * 2 + [ctypes.c_int64, c_void_p,
                                                                                                  ctypes.c_double, c_void_p,
                                                                                                  ctypes.c_double] + [c_void_p] * 2),
    "nudf_pc_radius_emit": (ctypes.c_int, [c_void_p] * 3 + [ctypes.c_int64] + [c_void_p] * 2 + [ctypes.c_int64, c_void_p,
                                                                                                 ctypes.c_double, c_void_p,
                                                                                                 ctypes.c_double] + [c_void_p] * 3),
    "nudf_pc_greedy_mis": (ctypes.c_int, [c_void_p, c_void_p, ctypes.c_int64] + [c_void_p] * 4),
    "nudf_pc_morton": (ctypes.c_int, [c_void_p, ctypes.c_int64, c_void_p, ctypes.c_double, c_void_p, c_void_p]),
    "nudf_pc_bvh_build": (ctypes.c_int, [c_void_p, ctypes.c_int64, ctypes.c_int64, c_void_p, c_void_p]),
    "nudf_pc_nearest": (ctypes.c_int, [c_void_p, ctypes.c_int64, c_void_p, c_void_p, ctypes.c_int64, c_void_p, ctypes.c_int64,
                                       ctypes.c_double, c_void_p, c_void_p]),
    "nudf_cl_dilate": (ctypes.c_int, [c_void_p] + [ctypes.c_int32] * 3 + [c_void_p] * 2 + [ctypes.c_int32] * 5
                       + [c_void_p] * 2),
    "nudf_cl_vote": (ctypes.c_int, [c_void_p, ctypes.c_int64, c_void_p, ctypes.c_int32, c_void_p] + [ctypes.c_int32] * 3
                     + [c_void_p] * 2),
    "nudf_iso_active": (ctypes.c_int, [c_void_p, ctypes.c_float, c_void_p, c_void_p]),
    "nudf_iso_cells_count": (ctypes.c_int, [c_void_p, ctypes.c_float, ctypes.c_int64, c_void_p, c_void_p]),
    "nudf_iso_cells_emit": (ctypes.c_int, [c_void_p, ctypes.c_float, ctypes.c_int64] + [c_void_p] * 3),
    "nudf_iso_count": (ctypes.c_int, [c_void_p, ctypes.c_float, c_void_p, ctypes.c_int64, c_void_p, c_void_p]),
    "nudf_iso_emit": (ctypes.c_int, [c_void_p, ctypes.c_float, c_void_p, ctypes.c_int64] + [c_void_p] * 3),
    "nudf_iso_vertices": (ctypes.c_int, [c_void_p, ctypes.c_float, c_void_p, ctypes.c_int64, c_void_p, ctypes.c_int64,
                                         c_void_p, c_void_p]),
    "nudf_nb_sublattice": (ctypes.c_int, [ctypes.c_int32] * 2 + [c_void_p] * 4),
    "nudf_nb_block_test": (ctypes.c_int, [c_void_p, ctypes.c_int32, c_void_p, ctypes.c_int32, c_void_p] + [ctypes.c_double] * 2
                           + [c_void_p] * 3),
    "nudf_nb_count": (ctypes.c_int, [c_void_p] + [ctypes.c_int32] * 3 + [c_void_p, ctypes.c_int64] + [c_void_p] * 2),
    "nudf_nb_emit": (ctypes.c_int, [c_void_p] + [ctypes.c_int32] * 3 + [c_void_p, ctypes.c_int64] + [c_void_p] * 5),
    "nudf_sb_mark": (ctypes.c_int, [c_void_p, ctypes.c_int32] + [c_void_p] * 3),
    "nudf_sb_store": (ctypes.c_int, [c_void_p] * 3 + [ctypes.c_int64] + [c_void_p] * 2),
    "nudf_sb_gather": (ctypes.c_int, [c_void_p] * 2 + [ctypes.c_int64] + [c_void_p] * 2),
    "nudf_sb_flat": (ctypes.c_int, [c_void_p] * 2 + [ctypes.c_int64] + [c_void_p] * 2),
    "nudf_uc_step_count": (ctypes.c_int, [c_void_p] * 3 + [ctypes.c_int64] + [c_void_p] * 2),
    "nudf_uc_step_emit": (ctypes.c_int, [c_void_p] * 3 + [ctypes.c_int64] + [c_void_p] * 3),
    "nudf_uc_filter_count": (ctypes.c_int, [c_void_p] * 2 + [ctypes.c_int64, ctypes.c_float] + [c_void_p] * 2),
    "nudf_uc_filter_emit": (ctypes.c_int, [c_void_p] * 2 + [ctypes.c_int64, ctypes.c_float] + [c_void_p] * 3),
    "nudf_uc_resample": (ctypes.c_int, [c_void_p, ctypes.c_int64, ctypes.c_int64, ctypes.c_uint32, ctypes.c_int32,
                                        ctypes.c_float, c_void_p, c_void_p]),
    "nudf_pt_normals": (ctypes.c_int, [c_void_p, ctypes.c_int64, c_void_p, c_void_p]),
    "nudf_pt_rank": (ctypes.c_int, [c_void_p, c_void_p, ctypes.c_int64, c_void_p, c_void_p] + [ctypes.c_int32] * 3
                     + [ctypes.c_float, ctypes.c_int32, c_void_p, c_void_p]),
    "nudf_pt_start_count": (ctypes.c_int, [c_void_p] * 3 + [ctypes.c_int32] * 2 + [c_void_p, ctypes.c_int64, c_void_p,
                                                                                  ctypes.c_float, c_void_p, c_void_p]),
    "nudf_pt_start_emit": (ctypes.c_int, [c_void_p] * 3 + [ctypes.c_int32] * 2 + [c_void_p, ctypes.c_int64, c_void_p,
                                                                                 ctypes.c_float] + [c_void_p] * 6),
    "nudf_pt_trace_count": (ctypes.c_int, [c_void_p] * 6 + [ctypes.c_int64, ctypes.c_float, c_void_p, c_void_p]),
    "nudf_pt_trace_emit": (ctypes.c_int, [c_void_p] * 6 + [ctypes.c_int64, ctypes.c_float] + [c_void_p] * 7),
    "nudf_pt_orient": (ctypes.c_int, [c_void_p] * 3 + [ctypes.c_int64] + [c_void_p] * 3),
    "nudf_pt_gather": (ctypes.c_int, [c_void_p] * 2 + [ctypes.c_int64] + [c_void_p] * 2 + [ctypes.c_int32] * 3
                       + [c_void_p] * 2),
    "nudf_mp_faces": (ctypes.c_int, [c_void_p, ctypes.c_int64, c_void_p, ctypes.c_int64] + [c_void_p] * 6),
    "nudf_mp_hole_count": (ctypes.c_int, [c_void_p, ctypes.c_int64, c_void_p, c_void_p, ctypes.c_int64, c_void_p, c_void_p]),
    "nudf_mp_hole_emit": (ctypes.c_int, [c_void_p] * 3 + [ctypes.c_int64, c_void_p, c_void_p, ctypes.c_int64]
                          + [c_void_p] * 3),
    "nudf_mp_smooth_step": (ctypes.c_int, [c_void_p] * 3 + [ctypes.c_int64, c_void_p, c_void_p, ctypes.c_double, c_void_p]),
    "nudf_mg_vertex_normals": (ctypes.c_int, [c_void_p, ctypes.c_int64, c_void_p, ctypes.c_int64] + [c_void_p] * 5),
    "nudf_mg_refine": (ctypes.c_int, [c_void_p, c_void_p, ctypes.c_int64, ctypes.c_float, c_void_p, c_void_p, ctypes.c_int32]
                       + [c_void_p] * 4),
    "nudf_cc_label": (ctypes.c_int, [c_void_p, c_void_p, ctypes.c_int64, ctypes.c_int64] + [c_void_p] * 3),
    "nudf_color_loss_forward": (ctypes.c_int, [c_void_p] * 5),
    "nudf_color_loss_backward": (ctypes.c_int, [c_void_p] * 9),
}


def exported_symbols():
    """Every entry point include/nudf.h declares (used by the ABI test)."""
    return sorted(_SIGNATURES)


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "libnudf.so not found at %s -- build it with `python -m neuraludf_b200.build` "
                "(there is deliberately no CPU / PyTorch fallback)" % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        if L.nudf_abi_version() != 6:
            raise RuntimeError("libnudf.so ABI version mismatch")
        _lib = L
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().nudf_last_error()
        raise RuntimeError("%s failed (rc=%d): %s" % (what, rc, msg.decode() if msg else "?"))


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def seg_counts(n, device):
    """the counts buffer of a stable compaction (include/nudf.h) over n items: int32 [ceil(n / NUDF_COMPACT_SEG)]"""
    import torch
    return torch.empty(-(-n // COMPACT_SEG), dtype=torch.int32, device=device)


def compact_batches(n, max_batch, device, batch):
    """Runs a stable compaction over n items in batches of max_batch and returns its output count.  batch(lo, hi) readies
    items [lo, hi) and returns launch(counts, offsets=None), which runs the count pass into counts when offsets is None
    and else the emit pass from offsets.  Each batch's outputs follow the previous batches' from a running base kept on
    the device, so that the output count is the only host read."""
    import torch
    base = torch.zeros(1, dtype=torch.int64, device=device)
    for lo in range(0, n, max_batch):
        hi = min(lo + max_batch, n)
        launch = batch(lo, hi)
        counts = seg_counts(hi - lo, device)
        launch(counts)
        csum = torch.cumsum(counts, 0, dtype=torch.int64)
        launch(counts, base + (csum - counts))
        base += csum[-1]
    return int(base.item())

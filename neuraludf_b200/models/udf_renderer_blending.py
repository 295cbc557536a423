"""UDFRendererBlending with the reference's API (mirror of `models/udf_renderer_blending.py` of xxlong0/NeuralUDF),
running on the libnudf CUDA kernels.

`render()` returns the same 32-key dict (reference :688-721); `render_core()` the same 29-key dict (:555-584).
Differences that are deliberate (DESIGN.md "boundary"):
  * one fused evaluation gives the UDF value, feature and exact input-gradient (the reference runs the MLP twice);
  * importance sampling, compositing and the regulariser sums never synchronise with the host (the reference has 13
    blocking syncs per step).  Where the reference drops into pdb on a NaN (:97-101, 265-269, 543-544) the kernels raise a
    device-side status flag; it is read together with render()'s one host read (`sample_dist`, :605) -- i.e. a non-finite
    result of call k raises a RuntimeError at the start of call k+1 -- or on demand with `check_finite()`;
  * `render()` evaluates the NeRF++ background only on the n_outside samples render_core consumes (:493-501);
  * per-sample outputs (`gradients`, `alpha*`, ...) are returned detached -- the trainer only uses them after
    .detach() or for logging (exp_runner_blending.py:309-371, 641-668); `weights` is differentiable.
Pixel / patch blending (fine-tuning stage, :431-480): one fused CUDA kernel per pass (csrc/blend.cu: projection, bilinear
gathers of pixel and homography-warped patch colours, masked-softmax fusion over views), composited with the
differentiable ray weights of the CUDA compositing kernel; patch_projector.py / fields.color_blend keep the op-by-op form,
which runs only for patches larger than 11 x 11 (h_patch_size > 5), img_index or more than 32 source views.
"""
import itertools
import os

import numpy as np
import torch
import torch.nn.functional as F

from .. import ops
from .fields import color_blend
from .patch_projector import PatchProjector


GRID_BLOCK = 64     # the reference queries dense grids in 64^3 blocks (:16-49); 262 144 points per kernel chain here
FUSED_MAX_H_PATCH = 5   # largest patch half-size of the fused blending kernel (11 x 11 pixels, csrc/blend.cu)
FUSED_MAX_VIEWS = 32    # largest number of source views of the fused blending kernel (one lane per view)


def _grid_query_device(bound_min, bound_max, resolution, query_func, device, channels):
    """Evaluate query_func on the resolution^3 lattice spanned by the bounds, block by block; returns a float32 tensor
    [R, R, R] (channels == 0) or [R, R, R, channels] on the device."""
    from ..grid import axis_tables
    axes = axis_tables(bound_min, bound_max, resolution, device)
    out = torch.zeros([resolution] * 3 + ([channels] if channels else []), dtype=torch.float32, device=device)
    starts = range(0, resolution, GRID_BLOCK)
    for i0, j0, k0 in itertools.product(starts, starts, starts):
        blk = [axes[0][i0:i0 + GRID_BLOCK], axes[1][j0:j0 + GRID_BLOCK], axes[2][k0:k0 + GRID_BLOCK]]
        pts = torch.cartesian_prod(*blk)                               # x slowest, z fastest (meshgrid 'ij' order)
        shape = [len(b) for b in blk] + ([channels] if channels else [])
        out[i0:i0 + shape[0], j0:j0 + shape[1], k0:k0 + shape[2]] = query_func(pts).detach().reshape(shape).float()
    return out


def _grid_query(bound_min, bound_max, resolution, query_func, device, channels):
    """_grid_query_device as a float32 numpy array: the grid is assembled on the device and copied to the host once (the
    reference copies and synchronises after every block)."""
    return _grid_query_device(bound_min, bound_max, resolution, query_func, device, channels).cpu().numpy()


def extract_fields(bound_min, bound_max, resolution, query_func, device):
    """Dense scalar grid query (API of the reference's extract_fields, :16-31)."""
    with torch.no_grad():
        return _grid_query(bound_min, bound_max, resolution, query_func, device, 0)


def extract_gradient_fields(bound_min, bound_max, resolution, query_func, device):
    """Dense 3-vector grid query (API of the reference's extract_gradient_fields, :34-49)."""
    return _grid_query(bound_min, bound_max, resolution, query_func, device, 3)


def extract_geometry(bound_min, bound_max, resolution, threshold, query_func, device):
    """reference :52-63.  With PyMCubes importable, exactly the reference's path.  Without it, the lattice stays on the
    device and is meshed there (mesh.iso_marching_cubes_index: fp32 threshold, faces wound towards decreasing values, this
    project's vertex numbering and ambiguous-cell triangulation); the vertices then take the reference's mapping
    (box_vertices).  With NUDF_BAND_MESH=1 in the environment (and no PyMCubes) the lattice is evaluated narrow-band
    (mesh.iso_mesh_band, Lipschitz bound 2): the same mesh when query_func is 2-Lipschitz and gives a point the same bits
    in any batch.  NUDF_BAND_MESH=sparse holds that band block-sparse (mesh.iso_mesh_sparse): the band mesh bit for bit,
    with no resolution^3 array."""
    try:
        import mcubes
    except ImportError:
        mcubes = None
    if mcubes is not None:
        u = extract_fields(bound_min, bound_max, resolution, query_func, device)
        vertices, triangles = mcubes.marching_cubes(u, threshold)
    else:
        from ..mesh import iso_marching_cubes_index, iso_mesh_band, iso_mesh_sparse
        band = {"1": iso_mesh_band, "sparse": iso_mesh_sparse}.get(os.environ.get("NUDF_BAND_MESH"))
        with torch.no_grad():
            if band is not None:
                v, f, _ = band(query_func, bound_min, bound_max, resolution, threshold, device=device)
            else:
                u = _grid_query_device(bound_min, bound_max, resolution, query_func, device, 0)
                v, f, _ = iso_marching_cubes_index(u, u.shape, threshold)
        vertices, triangles = v.cpu().numpy(), f.cpu().numpy()
    return box_vertices(vertices, resolution, bound_min, bound_max), triangles


def box_vertices(vertices, resolution, bound_min, bound_max):
    """lattice-index vertices -> box coordinates, as the reference maps them (:59-62): v / (R - 1) * (b_max - b_min) + b_min,
    the box difference in fp32"""
    b_max_np = bound_max.detach().cpu().numpy()
    b_min_np = bound_min.detach().cpu().numpy()
    return vertices / (resolution - 1.0) * (b_max_np - b_min_np)[None, :] + b_min_np[None, :]


def sample_pdf(bins, weights, n_samples, det=False):
    """Inverse-CDF sampling (reference :66-104).  det=True runs on the device kernel; det=False (never used by the
    renderer) is not implemented."""
    if not det:
        raise NotImplementedError("sample_pdf(det=False) is never called by the renderer")
    return ops.sample_pdf(bins, weights, n_samples)


class UDFRendererBlending:
    def __init__(self, nerf, udf_network, deviation_network, color_network, beta_network, n_samples, n_importance,
                 n_outside, up_sample_steps, perturb, sdf2alpha_type='numerical', upsampling_type='classical',
                 sparse_scale_factor=25000, h_patch_size=3, use_norm_grad_for_cosine=False):
        if sdf2alpha_type != 'numerical':
            raise NotImplementedError("sdf2alpha_type %r: only 'numerical' (all shipped confs) is implemented" %
                                      (sdf2alpha_type,))
        if upsampling_type not in ('classical', 'mix'):
            raise ValueError("upsampling_type must be 'classical' or 'mix'")
        self.nerf = nerf
        self.udf_network = udf_network
        self.deviation_network = deviation_network
        self.color_network = color_network
        self.beta_network = beta_network
        self.n_samples = n_samples
        self.n_importance = n_importance
        self.n_outside = n_outside
        self.perturb = perturb
        self.up_sample_steps = up_sample_steps
        self.sdf2alpha_type = sdf2alpha_type
        self.upsampling_type = upsampling_type
        self.sparse_scale_factor = sparse_scale_factor
        self.h_patch_size = h_patch_size
        self.patch_projector = PatchProjector(self.h_patch_size)
        self.use_norm_grad_for_cosine = use_norm_grad_for_cosine
        self.want_diagnostics = True     # per-sample dict entries (consumed only by validate / visualize_one_ray)

    # ------------------------------------------------------------------------------------------------------------
    # elementwise helpers kept for API parity (reference :151-159, :292-325); not used by the fused path
    # ------------------------------------------------------------------------------------------------------------
    def udf2logistic(self, udf, inv_s, gamma=20, abs_cos_val=1.0, cos_anneal_ratio=None):
        if cos_anneal_ratio is not None:
            abs_cos_val = (abs_cos_val * 0.5 + 0.5) * (1.0 - cos_anneal_ratio) + abs_cos_val * cos_anneal_ratio
        e = torch.exp(-inv_s * udf)
        return abs_cos_val * inv_s * e / (1 + e) ** 2 * gamma

    def sdf2alpha(self, sdf, true_cos, dists, inv_s, cos_anneal_ratio=None, udf_eps=None):
        if cos_anneal_ratio is not None:
            iter_cos = -(F.relu(-true_cos * 0.5 + 0.5) * (1.0 - cos_anneal_ratio) + F.relu(-true_cos) * cos_anneal_ratio)
        else:
            iter_cos = true_cos
        nxt = sdf + iter_cos * dists * 0.5
        prv = sdf - iter_cos * dists * 0.5
        cp, cn = torch.sigmoid(prv * inv_s), torch.sigmoid(nxt * inv_s)
        return ((cp - cn + 1e-5) / (cp + 1e-5)).clip(0.0, 1.0)

    # ------------------------------------------------------------------------------------------------------------
    # hierarchical sampling (reference :197-290, :723-755, :762-866) -- all @no_grad, all on the device
    # ------------------------------------------------------------------------------------------------------------
    def up_sample_unbias(self, rays_o, rays_d, z_vals, udf, sample_dist, n_importance, inv_s, beta, gamma, debug=False):
        return ops.up_sample(0, rays_o, rays_d, z_vals, udf.reshape(z_vals.shape), sample_dist, n_importance, inv_s, beta,
                             float(gamma))

    def up_sample_no_occ_aware(self, rays_o, rays_d, z_vals, udf, sample_dist, n_importance, inv_s, beta, gamma):
        return ops.up_sample(1, rays_o, rays_d, z_vals, udf.reshape(z_vals.shape), sample_dist, n_importance, inv_s, beta,
                             float(gamma))

    def cat_z_vals(self, rays_o, rays_d, z_vals, new_z_vals, udf, net_gradients=None, last=False):
        if last:
            z, _ = ops.merge_z(z_vals, new_z_vals)
            return z, udf
        pts = ops.points_on_rays(rays_o, rays_d, new_z_vals)
        new_udf = self.udf_network.udf_values(pts).reshape(new_z_vals.shape)
        return ops.merge_z(z_vals, new_z_vals, udf, new_udf)

    @torch.no_grad()
    def importance_sample(self, rays_o, rays_d, z_vals, sample_dist):
        pts = ops.points_on_rays(rays_o, rays_d, z_vals)
        udf = self.udf_network.udf_values(pts).reshape(z_vals.shape)
        K = self.up_sample_steps
        for i in range(K):
            new_z = self.up_sample_unbias(rays_o, rays_d, z_vals, udf, sample_dist, self.n_importance // K,
                                          64 * 2 ** i, 64 * 2 ** (i + 1),
                                          gamma=float(np.clip(20 * 2 ** (K - i), 20, 320)))
            z_vals, udf = self.cat_z_vals(rays_o, rays_d, z_vals, new_z, udf, last=(i + 1 == K))
        return z_vals

    @torch.no_grad()
    def importance_sample_mix(self, rays_o, rays_d, z_vals, sample_dist, gamma=None):
        """`gamma`: the clipped gamma as a float, when the caller has already read it (render.render_view reads it once
        per view); otherwise it is read here."""
        pts = ops.points_on_rays(rays_o, rays_d, z_vals)
        udf = self.udf_network.udf_values(pts).reshape(z_vals.shape)
        if gamma is None:
            gamma = float(self.beta_network.get_gamma().clip(1e-6, 1e6))   # one host read, as in the reference (:792)
        K = self.up_sample_steps
        m = self.n_importance // (K + 1)
        for i in range(K):
            new_z = self.up_sample_no_occ_aware(rays_o, rays_d, z_vals, udf, sample_dist, m, 64 * 2 ** i,
                                                64 * 2 ** (i + 1), gamma)
            z_vals, udf = self.cat_z_vals(rays_o, rays_d, z_vals, new_z, udf)
        for i in range(K - 1, K):
            new_z = self.up_sample_unbias(rays_o, rays_d, z_vals, udf, sample_dist, m, 64 * 2 ** i, 64 * 2 ** (i + 1),
                                          gamma=20 if i < 4 else 10)
            z_vals, udf = self.cat_z_vals(rays_o, rays_d, z_vals, new_z, udf, last=(i + 1 == K))
        return z_vals

    # ------------------------------------------------------------------------------------------------------------
    # NeRF++ background (reference :161-195)
    # ------------------------------------------------------------------------------------------------------------
    def _outside(self, rays_o, rays_d, z_vals, sample_dist, nerf, col0):
        """alpha [N, n-col0], sampled colour [N, n-col0, 3] of columns >= col0 of z_vals."""
        N, n = z_vals.shape
        m = n - col0
        if self.n_outside > 0:
            pts4, dists = ops.outside_points(rays_o, rays_d, z_vals, col0, sample_dist)
        else:
            raise NotImplementedError("render_core_outside with n_outside == 0 (3-D NeRF inputs) is not used by any conf")
        raw, rgb = nerf.forward_rays(pts4, rays_d, m)
        alpha = 1.0 - torch.exp(-F.relu(raw.reshape(N, m)) * dists)
        return alpha, rgb.reshape(N, m, 3)

    def render_core_outside(self, rays_o, rays_d, z_vals, sample_dist, nerf, background_rgb=None):
        alpha, sampled_color = self._outside(rays_o, rays_d, z_vals, sample_dist, nerf, 0)
        N = alpha.shape[0]
        trans = torch.cumprod(torch.cat([torch.ones([N, 1], device=alpha.device), 1. - alpha + 1e-7], -1), -1)[:, :-1]
        weights = alpha * trans
        color = (weights[:, :, None] * sampled_color).sum(dim=1)
        if background_rgb is not None:
            color = color + background_rgb * (1.0 - weights.sum(dim=-1, keepdim=True))
        return {'color': color, 'sampled_color': sampled_color, 'alpha': alpha, 'weights': weights}

    # ------------------------------------------------------------------------------------------------------------
    # fine pass (reference :327-584)
    # ------------------------------------------------------------------------------------------------------------
    def render_core(self, rays_o, rays_d, z_vals, sample_dist, udf_network, deviation_network, color_network,
                    beta_network=None, cos_anneal_ratio=None, background_rgb=None, background_alpha=None,
                    background_sampled_color=None, flip_saturation=0.0, color_maps=None, w2cs=None, intrinsics=None,
                    query_c2w=None, img_index=None, rays_uv=None):
        device = z_vals.device
        batch_size, n_samples = z_vals.shape
        rays_o = rays_o.float().contiguous()
        rays_d = rays_d.float().contiguous()
        pts, mid_z_vals, dists = ops.ray_points(rays_o, rays_d, z_vals, sample_dist)

        udf, feature_vector, gradients = udf_network.value_feature_gradient(pts)        # [P,1], [P,F], [P,3]  (:364-368)
        udf = udf[:, 0]

        inv_s = deviation_network(torch.zeros([1, 3], device=device))[:, :1].clip(1e-6, 1e6)     # :373
        beta = beta_network.get_beta().clip(1e-6, 1e6)
        gamma = beta_network.get_gamma().clip(1e-6, 1e6)
        heads = torch.cat([inv_s.reshape(1), beta.reshape(1), gamma.reshape(1)])

        sampled_color_base, sampled_color, blending_weights = color_network.forward_rays(pts, rays_d, n_samples,
                                                                                         feature_vector)   # :425
        n_outside = 0
        if background_alpha is not None:
            n_outside = background_alpha.shape[1] - n_samples
        cfg = ops._make_cfg(batch_size, n_samples, n_outside, sample_dist, cos_anneal_ratio, flip_saturation,
                            self.sparse_scale_factor, self.use_norm_grad_for_cosine, background_rgb)
        comp = ops.composite(udf, gradients, sampled_color_base, sampled_color,
                             background_alpha if n_outside > 0 else None,
                             background_sampled_color if n_outside > 0 else None, heads,
                             (rays_d, pts, mid_z_vals, dists), cfg, want_diag=self.want_diagnostics)
        rs = comp["ray_sums"]
        # regularisers from per-ray partial sums (:531-536, :553); the mask counts are detached like the reference's
        gradient_error = rs[:, 0].sum() / (rs[:, 1].sum().detach() + 1e-5)
        gradient_error_near_surface = rs[:, 2].sum() / (rs[:, 3].sum().detach() + 1e-5)
        sparse_error = rs[:, 4].sum() / batch_size

        g3 = gradients.detach().reshape(batch_size, n_samples, 3)
        blending_weights = blending_weights.reshape(batch_size, n_samples, -1)
        color_pixel, patch_colors, patch_mask = self._blend(
            comp['weights'], pts, rays_d, g3, blending_weights, background_sampled_color, color_maps, w2cs, intrinsics,
            query_c2w, img_index, rays_uv)
        ret = {
            'color_base': comp['color_base'], 'color': comp['color'], 'color_pixel': color_pixel,
            'patch_colors': patch_colors, 'patch_mask': patch_mask, 'weights': comp['weights'],
            's_val': (1.0 / inv_s).expand(batch_size * n_samples, 1), 'beta': 1.0 / beta, 'gamma': gamma,
            'depth': comp['depth'], 'gradient_error': gradient_error,
            'gradient_error_near_surface': gradient_error_near_surface, 'normals': comp['normals'], 'gradients': g3,
            'udf': udf.detach().reshape(batch_size, n_samples), 'mid_z_vals': mid_z_vals, 'dists': dists,
            'sparse_error': sparse_error,
            # extra (not in the reference dict): differentiable per-ray weight sums, blending logits
            'weight_sum': comp['weight_sum'], 'weight_sum_fg_bg': comp['weight_sum_fg_bg'],
            'blending_weights': blending_weights,
        }
        for k in ('gradients_flip', 'inside_sphere', 'gradient_mag', 'true_cos', 'vis_prob', 'alpha', 'alpha_plus',
                  'alpha_minus', 'alpha_occ', 'raw_occ'):
            ret[k] = comp.get(k)
        return ret

    def _blend(self, weights, pts, rays_d, g3, blending_weights, background_sampled_color, color_maps, w2cs, intrinsics,
               query_c2w, img_index, rays_uv):
        """Pixel / patch blending of the fine-tuning stage (reference :431-480 and :503-524): colours warped from the
        source views, blended per sample with the colour network's logits and composited with the ray weights (which
        carry the gradient to the UDF through nudf_render_composite_backward's `weights` adjoint)."""
        if color_maps is None and rays_uv is None:
            return None, None, None
        if color_maps is None:
            raise ValueError("patch blending (rays_uv) needs color_maps as well (the reference fails here too, "
                             "fields.py:505)")
        batch_size, n_samples = g3.shape[:2]
        p3 = pts.reshape(batch_size, n_samples, 3)
        normals = None
        if rays_uv is not None:                                  # flipped unit normals of the local surface plane (:446-448)
            gn = g3 / (torch.linalg.norm(g3, ord=2, dim=-1, keepdim=True) + 1e-5)
            cos = (rays_d[:, None, :] * gn).sum(-1, keepdim=True)
            normals = torch.where(cos == 0, torch.ones_like(cos), -torch.sign(cos)) * gn
        if (img_index is None and color_maps.shape[0] <= FUSED_MAX_VIEWS
                and (rays_uv is None or self.h_patch_size <= FUSED_MAX_H_PATCH)):
            # fused kernel: projection + bilinear gathers + masked-softmax fusion per point (csrc/blend.cu); the small
            # per-point homographies come from torch (3x3 algebra on [V, P] matrices, no gradient).  Pixel blending does
            # not depend on the patch size, so without uv the kernel runs with h_patch = 0 whatever h_patch_size is.
            n_views = color_maps.shape[0]
            proj = (intrinsics[:, :3, :3] @ w2cs[:, :3, :]).reshape(n_views, 12)
            hom, px = None, None
            if rays_uv is not None:
                hom, px = self.patch_projector.homographies(p3, rays_uv, normals, color_maps.shape[2:], intrinsics[0],
                                                            intrinsics, query_c2w, torch.inverse(w2cs))
                hom = hom.reshape(n_views, -1, 9)
            h_patch = self.h_patch_size if rays_uv is not None else 0
            c_pix, c_pat, m_pat = ops.blend_views(blending_weights.reshape(batch_size * n_samples, -1), p3.reshape(-1, 3), proj,
                                                  hom, px, color_maps, batch_size, n_samples, h_patch)
        else:
            # op-by-op path: img_index selection (never used by the runner), patches larger than 11 x 11, > 32 source views
            pix_col, pix_mask = self.patch_projector.pixel_warp(p3, color_maps, intrinsics, w2cs, img_wh=None)
            pat_col, pat_mask = None, None
            if rays_uv is not None:
                pat_col, pat_mask = self.patch_projector.patch_warp(
                    p3, rays_uv, normals, color_maps, intrinsics[0], intrinsics, query_c2w, torch.inverse(w2cs),
                    img_wh=None, detach_normal=True)
            c_pix, _, c_pat, m_pat = color_blend(blending_weights, img_index=img_index, pts_pixel_color=pix_col,
                                                 pts_pixel_mask=pix_mask, pts_patch_color=pat_col, pts_patch_mask=pat_mask)
        c_pix = c_pix.view(batch_size, n_samples, 3)
        if background_sampled_color is not None:
            inside = (torch.linalg.norm(p3, ord=2, dim=-1) < 1.0).float()[:, :, None]
            c_pix = c_pix * inside + background_sampled_color[:, :n_samples] * (1.0 - inside)
            c_pix = torch.cat([c_pix, background_sampled_color[:, n_samples:]], dim=1)
        color_pixel = (c_pix * weights[:, :c_pix.shape[1], None]).sum(dim=1)
        patch_colors, patch_mask = None, None
        if c_pat is not None:
            w_in = weights[:, :n_samples]
            patch_colors = (c_pat.view(batch_size, n_samples, -1, 3) * w_in[:, :, None, None]).sum(dim=1)
            patch_mask = (m_pat.view(batch_size, n_samples).float() * w_in).sum(dim=1)
        return color_pixel, patch_colors, patch_mask

    # ------------------------------------------------------------------------------------------------------------
    # whole render (reference :586-721)
    # ------------------------------------------------------------------------------------------------------------
    def render(self, rays_o, rays_d, near, far, cos_anneal_ratio=None, perturb_overwrite=-1, background_rgb=None,
               flip_saturation=0, color_maps=None, w2cs=None, intrinsics=None, query_c2w=None, img_index=None,
               rays_uv=None):
        device = rays_o.device
        batch_size = len(rays_o)
        if not isinstance(near, torch.Tensor):
            near = torch.Tensor([near]).view(1, 1).to(device)
            far = torch.Tensor([far]).view(1, 1).to(device)
        # the one host sync of render() (:605); the same read carries the device status word of the previous kernels
        sample_dist = ops.check_status(device, ((far - near) / self.n_samples).mean())
        z_vals = torch.linspace(0.0, 1.0, self.n_samples, device=device)
        z_vals = near + (far - near) * z_vals[None, :]
        z_vals_outside = None
        if self.n_outside > 0:
            z_vals_outside = torch.linspace(1e-3, 1.0 - 1.0 / (self.n_outside + 1.0), self.n_outside, device=device)
        n_samples = self.n_samples
        perturb = self.perturb
        if perturb_overwrite >= 0:
            perturb = perturb_overwrite
        if perturb > 0:
            t_rand = torch.rand([batch_size, 1], device=device) - 0.5
            z_vals = z_vals + t_rand * 2.0 / self.n_samples
            if self.n_outside > 0:
                mids = .5 * (z_vals_outside[..., 1:] + z_vals_outside[..., :-1])
                upper = torch.cat([mids, z_vals_outside[..., -1:]], -1)
                lower = torch.cat([z_vals_outside[..., :1], mids], -1)
                t_rand = torch.rand(z_vals_outside.shape, device=device)
                z_vals_outside = lower + (upper - lower) * t_rand
        if self.n_outside > 0:
            z_vals_outside = far / torch.flip(z_vals_outside, dims=[-1]) + 1.0 / self.n_samples
        if z_vals.shape[0] != batch_size:
            z_vals = z_vals.expand(batch_size, -1)
        z_vals = z_vals.contiguous()

        if self.n_importance > 0:
            if self.upsampling_type == 'classical':
                z_vals = self.importance_sample(rays_o, rays_d, z_vals, sample_dist)
            else:
                z_vals = self.importance_sample_mix(rays_o, rays_d, z_vals, sample_dist)
        return self._render_from_z(rays_o, rays_d, z_vals, z_vals_outside, sample_dist, cos_anneal_ratio, background_rgb,
                                   flip_saturation, color_maps, w2cs, intrinsics, query_c2w, img_index, rays_uv)

    def _render_from_z(self, rays_o, rays_d, z_vals, z_vals_outside, sample_dist, cos_anneal_ratio=None,
                       background_rgb=None, flip_saturation=0, color_maps=None, w2cs=None, intrinsics=None, query_c2w=None,
                       img_index=None, rays_uv=None):
        """Everything of render() after the (non-differentiable) sampling phase: NeRF++ background on the outside samples,
        fine pass, sparse_random_error (reference :646-721).  Separate so that tests can feed the reference's own sample
        positions and compare gradients tightly."""
        device = rays_o.device
        batch_size = len(rays_o)
        n_samples = z_vals.shape[1]
        background_alpha = None
        background_sampled_color = None
        if self.n_outside > 0:
            z_out = z_vals_outside.expand(batch_size, -1) if z_vals_outside.shape[0] != batch_size else z_vals_outside
            z_vals_feed, _ = torch.sort(torch.cat([z_vals, z_out], dim=-1), dim=-1)
            if color_maps is None:
                # only the outside columns are consumed by render_core (:493-501)
                a_o, c_o = self._outside(rays_o, rays_d, z_vals_feed.contiguous(), sample_dist, self.nerf, n_samples)
                background_alpha = torch.cat([torch.zeros(batch_size, n_samples, device=device), a_o], dim=1)
                background_sampled_color = torch.cat([torch.zeros(batch_size, n_samples, 3, device=device), c_o], dim=1)
            else:
                # pixel blending mixes the NeRF colour of the inside columns into color_pixel outside the sphere (:507)
                background_alpha, background_sampled_color = self._outside(
                    rays_o, rays_d, z_vals_feed.contiguous(), sample_dist, self.nerf, 0)

        ret_fine = self.render_core(rays_o, rays_d, z_vals, sample_dist, self.udf_network, self.deviation_network,
                                    self.color_network, beta_network=self.beta_network,
                                    cos_anneal_ratio=cos_anneal_ratio, background_rgb=background_rgb,
                                    background_alpha=background_alpha,
                                    background_sampled_color=background_sampled_color, flip_saturation=flip_saturation,
                                    color_maps=color_maps, w2cs=w2cs, intrinsics=intrinsics, query_c2w=query_c2w,
                                    img_index=img_index, rays_uv=rays_uv)

        # sparse_random_error (:681-686) without the data-dependent host branch
        pts_random = torch.rand([1024, 3], device=device).float() * 2 - 1
        udf_random = self.udf_network.udf(pts_random)
        msk = (udf_random < 0.01)
        cnt = msk.sum()
        val = (torch.exp(-self.sparse_scale_factor * udf_random) * msk).sum() / cnt.clamp(min=1)
        sparse_random_error = torch.where(cnt > 10, val, torch.zeros_like(val))

        keys = ['color_base', 'color', 'color_pixel', 'patch_colors', 'patch_mask', 'depth', 'beta', 'gamma', 'normals',
                'gradients', 'gradients_flip', 'weights', 'gradient_error', 'gradient_error_near_surface',
                'inside_sphere', 'udf', 'gradient_mag', 'true_cos', 'vis_prob', 'alpha', 'alpha_plus', 'alpha_minus',
                'mid_z_vals', 'dists', 'sparse_error', 'alpha_occ', 'raw_occ', 'weight_sum', 'weight_sum_fg_bg']
        out = {k: ret_fine[k] for k in keys}
        out['variance'] = ret_fine['s_val']
        out['z_vals'] = z_vals
        out['sparse_random_error'] = sparse_random_error
        return out

    def check_finite(self, device=None):
        """Synchronises and raises RuntimeError if any sampling / compositing kernel since the last check produced a
        non-finite result (the reference's pdb traps, :97-101, 265-269, 543-544)."""
        if device is None:
            device = next(self.udf_network.parameters()).device
        ops.check_status(torch.device(device))

    def extract_geometry(self, bound_min, bound_max, resolution, threshold=0.01, device='cpu'):
        return extract_geometry(bound_min, bound_max, resolution, threshold,
                                lambda pts: self.udf_network.udf_values(pts), device)

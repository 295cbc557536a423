"""Pixel / patch warping of sample points into the source views (fine-tuning stage of NeuralUDF), API mirror of the
reference's `models/patch_projector.py` (`PatchProjector.pixel_warp` :21-43, `.patch_warp` :45-150) and of
`models/projector_utils.py` (`sample_ptsFeatures_from_featureMaps` :52-85).

Status (DESIGN.md, SURVEY 8(f) rank 1): the renderer uses the fused kernel `ops.blend_views` (csrc/blend.cu) fed by
`PatchProjector.homographies` (small batched 3x3 algebra in torch) for patches of up to 11 x 11 pixels (h_patch_size <= 5,
which covers the fine-tuning conf's h_patch_size = 5) and for pixel-only blending at any patch size; `pixel_warp` /
`patch_warp` below are the op-by-op form (`grid_sample`, `einsum`) kept as API mirrors of the reference, as the test
reference of the fused kernel, and as the renderer's path for larger patches, `img_index` and more than 32 source views.
Unlike the reference, `patch_warp` does not modify the caller's `uv` tensor in place.
"""
import torch
import torch.nn.functional as F


def patch_offsets(h_patch_size):
    """[1, (2h+1)^2, 2] pixel offsets (dx, dy), dx fastest (reference build_patch_offset :212-214)."""
    r = torch.arange(-h_patch_size, h_patch_size + 1)
    dy, dx = torch.meshgrid(r, r, indexing="ij")
    return torch.stack([dx, dy], dim=-1).view(1, -1, 2)


def project_points(pts, intrinsics, w2cs, width, height):
    """Normalised grid coordinates of world points in every view.
    pts [N,S,3], intrinsics [V,4,4] (or [V,3,3]), w2cs [V,4,4] -> grid [V,N,S,2] in grid_sample's (-1,1) convention,
    with out-of-image coordinates pushed to 2 (reference cam2pixel :8-48 with padding 'zeros')."""
    proj = intrinsics[:, :3, :3] @ w2cs[:, :3, :]                      # [V,3,4]
    n, s, _ = pts.shape
    flat = pts.reshape(-1, 3)
    cam = torch.einsum("vij,pj->vip", proj[:, :, :3], flat) + proj[:, :, 3:]        # [V,3,P]
    z = cam[:, 2].clamp(min=1e-3)
    xn = 2 * (cam[:, 0] / z) / (width - 1) - 1
    yn = 2 * (cam[:, 1] / z) / (height - 1) - 1
    xn = torch.where((xn > 1) | (xn < -1), torch.full_like(xn, 2.0), xn)
    yn = torch.where((yn > 1) | (yn < -1), torch.full_like(yn, 2.0), yn)
    return torch.stack([xn, yn], dim=-1).view(-1, n, s, 2)


class PatchProjector:
    def __init__(self, patch_size):
        self.h_patch_size = patch_size
        self.offsets = patch_offsets(patch_size)
        self.plane_dist_thresh = 0.001

    def pixel_warp(self, pts, imgs, intrinsics, w2cs, img_wh=None):
        """pts [N,S,3], imgs [V,3,H,W] -> colours [N,S,V,3], validity mask [N,S,V]."""
        if img_wh is None:
            img_wh = [imgs.shape[3], imgs.shape[2]]
        grid = project_points(pts, intrinsics, w2cs, img_wh[0], img_wh[1])
        valid = (grid[..., 0].abs() < 1.0) & (grid[..., 1].abs() < 1.0)
        col = F.grid_sample(imgs, grid, padding_mode="zeros", align_corners=True)          # [V,3,N,S]
        return col.permute(2, 3, 0, 1), valid.permute(1, 2, 0)

    def homographies(self, pts, uv, normals, img_hw, ref_intrinsic, src_intrinsics, ref_c2w, src_c2ws):
        """Plane-induced homographies query pixel -> source pixel for every (view, point), built without gradient like
        the reference (patch_projector.py:100-129), with the fronto-parallel fallback for degenerate planes.
        pts, normals [N,S,3]; uv [N,2] in (-1,1); img_hw = (H, W).  Returns hom [V, N*S, 3, 3] and the query pixel
        coordinates px [N,2]."""
        device = pts.device
        n_rays, n_samples, _ = pts.shape
        n_pts = n_rays * n_samples
        size_h, size_w = img_hw
        n_src = src_intrinsics.shape[0]
        px = torch.stack([(uv[:, 0] + 1) / 2.0 * (size_w - 1), (uv[:, 1] + 1) / 2.0 * (size_h - 1)], dim=-1)   # pixels
        k_ref_inv = torch.inverse(ref_intrinsic[:3, :3])
        k_src = src_intrinsics[:, :3, :3]
        ref_w2c = torch.inverse(ref_c2w)
        src_w2c = torch.inverse(src_c2ws)
        cam_center = ref_c2w[:3, 3].unsqueeze(0)
        rel = src_w2c @ ref_c2w                                                           # ref camera -> src camera
        r_rel, t_rel = rel[:, :3, :3], rel[:, :3, 3:]
        r_ref, t_ref = ref_w2c[:3, :3], ref_w2c[:3, 3:]
        p_flat = pts.reshape(-1, 3)
        n_flat = normals.reshape(-1, 3)
        with torch.no_grad():
            dist_to_cam = torch.norm(pts - cam_center, dim=-1)                            # [N,S]
            n_cam = (r_ref @ n_flat.unsqueeze(-1))                                        # [P,3,1] plane normal, ref frame
            p_cam = r_ref @ p_flat.unsqueeze(-1) + t_ref                                  # [P,3,1]
            d_ref = (n_cam * p_cam).sum(dim=1).unsqueeze(1)                               # plane distance to the ref camera
            src_center = (-r_rel.transpose(1, 2) @ t_rel)                                 # [V,3,1] src camera in ref frame
            d_src = (n_cam.unsqueeze(1) * src_center.unsqueeze(0)).sum(dim=2)             # [P,V,1]
            ok = ((d_ref.abs() > self.plane_dist_thresh) & ((d_ref - d_src).abs() > self.plane_dist_thresh)
                  & ((d_src / d_ref) < 1))
            d1 = d_ref.reshape(-1)
            sgn = torch.sign(d1)
            sgn[sgn == 0] = 1
            d = torch.clamp(d1.abs(), 1e-8) * sgn
            # H = K_src (R_rel + t_rel n^T / d) K_ref^-1 = A_v + b_v (K_ref^-T n)^T / d : one broadcast outer product per
            # (view, point) instead of two batched 3x3 matrix products over V*P matrices; same for the fronto-parallel
            # fallback with n = z axis and d = distance to the reference camera
            a_v = k_src @ r_rel @ k_ref_inv                                               # [V,3,3]
            b_v = (k_src @ t_rel).squeeze(-1)                                             # [V,3]
            q = (n_cam.squeeze(-1) @ k_ref_inv) / d[:, None]                              # [P,3]  (K_ref^-T n) / d
            q_fp = k_ref_inv[2, :].unsqueeze(0) / dist_to_cam.reshape(n_pts, 1)           # [P,3]
            use = ok.view(n_pts, n_src).t().unsqueeze(-1)                                 # [V,P,1]
            q_sel = torch.where(use, q.unsqueeze(0), q_fp.unsqueeze(0))                   # [V,P,3]
            hom = a_v.unsqueeze(1) + b_v[:, None, :, None] * q_sel[:, :, None, :]         # [V,P,3,3]
        return hom, px

    def patch_warp(self, pts, uv, normals, src_imgs, ref_intrinsic, src_intrinsics, ref_c2w, src_c2ws, img_wh=None,
                   detach_normal=False):
        """Plane-induced homography warp of the (2h+1)^2 reference patch around every ray's pixel into each source view.
        pts [N,S,3], uv [N,2] in (-1,1), normals [N,S,3] -> colours [N,S,V,Npx,3], mask [N,S,V,Npx].
        (Op-by-op form, kept as the API mirror and as the test reference of the fused kernel ops.blend_views.)"""
        device = pts.device
        if detach_normal:
            normals = normals.detach()
        n_rays, n_samples, _ = pts.shape
        n_src, _, size_h, size_w = src_imgs.shape
        if img_wh is not None:
            size_w, size_h = img_wh[0], img_wh[1]
        hom, px = self.homographies(pts, uv, normals, (size_h, size_w), ref_intrinsic, src_intrinsics, ref_c2w, src_c2ws)
        pixels = px.view(n_rays, 1, 2) + self.offsets.float().to(device)                  # [N,Npx,2]
        n_px = pixels.shape[1]
        hom = hom.view(n_src, n_rays, -1, 3, 3)
        hp = torch.cat([pixels, torch.ones_like(pixels[..., :1])], dim=-1)                # [N,Npx,3]
        warped = torch.einsum("vprik,pok->vproi", hom, hp).reshape(n_src, -1, 3)
        grid = warped[..., :2] / torch.clamp(warped[..., 2:], 1e-8)
        mask = warped[..., 2] > 0
        h = self.h_patch_size
        mask = mask & (grid[..., 0] < (size_w - h)) & (grid[..., 1] < (size_h - h)) & (grid >= h).all(dim=-1)
        mask = mask.view(n_src, n_rays, n_samples, n_px)
        gx = 2 * grid[..., 0] / (size_w - 1) - 1
        gy = 2 * grid[..., 1] / (size_h - 1) - 1
        gnorm = torch.clamp(torch.stack([gx, gy], dim=-1), -10, 10)
        rgb = F.grid_sample(src_imgs, gnorm.view(n_src, -1, 1, 2), align_corners=True).squeeze(-1).transpose(1, 2)
        rgb = rgb.view(n_src, n_rays, n_samples, n_px, 3)
        return rgb.permute(1, 2, 0, 3, 4).contiguous(), mask.permute(1, 2, 0, 3).contiguous()

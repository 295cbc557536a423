"""Forward-only rendering of whole views: what `Runner.validate()` and `validate_novel_image()` of the reference
(exp_runner_blending.py:604-747) produce, without the training path.

`render_view` renders an [H, W] grid of rays chunk by chunk.  Each chunk runs the sampling of `render()` and then the
UDF, colour and NeRF++ forwards, the pixel blend and `nudf_render_view_forward` (csrc/ray_kernels.cu) outside autograd,
with every per-chunk array carved from one workspace (ViewWorkspace) and no host read.  The compositing is the same
device code as render_core's, so `color` and `depth` equal `render()`'s bit for bit on the same rays.

Deviations from the runner (INTEGRATION.md "Rendering views"):
  * `sample_dist` is ((far - near) / n_samples).mean() over the whole view (the runner takes it per 512-ray call; for
    unit-sphere near / far the two differ only by rounding, far - near = 2);
  * with perturb > 0 the jitter is drawn once per view (torch.rand([N, 1]), then torch.rand([n_outside])), the runner
    draws it per 512-ray call;
  * source views are ranked by fp32 torch.cdist on the CPU with a stable sort; the runner ranks on the device with an
    unstable sort, so exact ties and near-ties (cdist's rounding differs between devices) may order differently;
  * the depth PNG needs matplotlib's colormap; without matplotlib only the .npy of the raw depth is written.

`load_scan` restates the reference's DTU-layout `Dataset` (downsample_factor 1), `rays_between` its `gen_rays_between`,
and `python -m neuraludf_b200.render` renders a checkpoint's views into the runner's file layout.
"""
import ctypes
import glob
import os

import numpy as np
import torch

from . import _lib as L
from . import ops

DEFAULT_WORKSPACE_BYTES = 8 << 30


def _heads(renderer, device):
    """(inv_s, beta, gamma) after render_core's clips (udf_renderer_blending.py:373-377), on the device"""
    inv_s = renderer.deviation_network(torch.zeros([1, 3], device=device))[:, :1].clip(1e-6, 1e6)
    beta = renderer.beta_network.get_beta().clip(1e-6, 1e6)
    gamma = renderer.beta_network.get_gamma().clip(1e-6, 1e6)
    return torch.cat([inv_s.reshape(1), beta.reshape(1), gamma.reshape(1)]).float().contiguous()


class ViewWorkspace:
    """One fp32 buffer holding every array of one chunk of the forward-only view pipeline (render.render_view).

    The network forwards keep no state for a backward pass, so their context buffers are scratch: the UDF, colour and
    NeRF++ forwards (and the sampling stage's UDF value queries) share one region sized for the largest of them.  The
    chunk size is the largest ray count whose arrays fit `budget_bytes`, from the library's nudf_*_ctx_floats queries."""

    def __init__(self, renderer, n_rays, budget_bytes, device, n_views=0):
        lib = L.lib()
        udf_h = renderer.udf_network._handle
        udf_h.refresh()
        col_h = renderer.color_network._handle
        col_h.refresh()
        self.S0, self.S = renderer.n_samples, renderer.n_samples + renderer.n_importance
        self.O = renderer.n_outside
        self.F = udf_h.meta[2] - 1
        self.nb = col_h.meta[3]
        self.blend = n_views > 0
        # NeRF++ columns evaluated per ray: all S+O when the pixel blend needs the inside columns too (render() does the same)
        self.m = (self.S + self.O if self.blend else self.O) if self.O > 0 else 0
        nerf_d = renderer.nerf._handle.desc() if self.O > 0 else None
        S, SO, m = self.S, self.S + self.O, self.m

        def ctx(n):
            c = [lib.nudf_udf_ctx_floats(ctypes.byref(udf_h.desc), n * S, 1),
                 lib.nudf_udf_ctx_floats(ctypes.byref(udf_h.desc), n * self.S0, 0),
                 lib.nudf_color_ctx_floats(ctypes.byref(col_h.desc), n * S)]
            if m:
                c.append(lib.nudf_nerf_ctx_floats(ctypes.byref(nerf_d), n * m))
            return max(c)

        # per ray: pts, mid, dists, udf, feat, grad, cb, c, logits (+ c_pix) of S samples; NeRF++ inputs / outputs of m
        # columns and the [S+O] background arrays; sampling and z-sorting temporaries (z, udf, points of each round)
        self._per_ray = (S * (3 + 1 + 1 + 1 + self.F + 3 + 3 + 3 + self.nb + (3 if self.blend else 0))
                         + m * (4 + 1 + 1 + 3) + SO * (1 + 3) + 8 * SO)
        self._ctx = ctx
        # the sampling stage's UDF value queries allocate their own scratch while the workspace is live: counted twice
        total = lambda n: n * self._per_ray + 2 * ctx(n)
        probe = min(4096, n_rays)
        n = max(1, min(n_rays, int(budget_bytes // 4 * probe // total(probe))))
        while n > 1 and total(n) * 4 > budget_bytes:
            n = max(1, n * 15 // 16)
        self.chunk = n
        self.buf = torch.empty(n * (self._per_ray - 8 * SO) + ctx(n) + 64 * 16, dtype=torch.float32, device=device)

    def carve(self, n):
        """views of the workspace for a chunk of n <= self.chunk rays"""
        S, SO, m = self.S, self.S + self.O, self.m
        off = [0]
        buf = self.buf

        def take(*shape):             # every array starts on a 256-byte boundary (vector loads in the kernels)
            k = 1
            for s in shape:
                k *= s
            t = buf[off[0]:off[0] + k].view(*shape)
            off[0] += -(-k // 64) * 64
            return t
        w = {"pts": take(n * S, 3), "mid": take(n, S), "dists": take(n, S), "udf": take(n * S), "feat": take(n * S, self.F),
             "grad": take(n * S, 3), "cb": take(n * S, 3), "c": take(n * S, 3), "bl": take(n * S, self.nb)}
        if self.blend:
            w["c_pix"] = take(n * S, 3)
        if m:
            w.update(pts4=take(n * m, 4), odists=take(n, m), sigma=take(n * m, 1), rgb=take(n * m, 3), bg_alpha=take(n, SO),
                     bg_color=take(n, SO, 3))
        w["ctx"] = buf[off[0]:]
        assert w["ctx"].numel() >= self._ctx(n)
        return w


@torch.no_grad()
def render_view(renderer, rays_o, rays_d, near, far, *, color_maps=None, w2cs=None, intrinsics=None, rot=None, perturb=0.0,
                cos_anneal_ratio=None, background_rgb=None, workspace_bytes=DEFAULT_WORKSPACE_BYTES, max_chunk=None,
                z_vals=None):
    """Render the rays rays_o / rays_d [H, W, 3] (near / far [H, W, 1]) of one view with `renderer`
    (a UDFRendererBlending).  Returns {color, depth, normal, weight_sum} and, with color_maps / w2cs / intrinsics
    (the source views, as render() takes them), color_pixel: device tensors [H, W, 3] / [H, W, 1].

    normal is validate()'s normal map, sum of gradients_flip * weights * inside_sphere, multiplied by `rot` (3x3, the
    inverse of the view's pose rotation; identity when None).  Arrays of one chunk stay under `workspace_bytes`;
    `max_chunk` caps the rays per chunk.  The result does not depend on the chunk size.  z_vals [H*W, n_samples +
    n_importance], when given, replaces the sampling stage (the fine samples of another renderer, for comparisons)."""
    dev = rays_o.device
    H, W = rays_o.shape[:2]
    N = H * W
    o = rays_o.reshape(N, 3).float().contiguous()
    d = rays_d.reshape(N, 3).float().contiguous()
    near = near.reshape(N, 1).float()
    far = far.reshape(N, 1).float()
    ops._require_cuda(o, d, near, far)
    S0, O = renderer.n_samples, renderer.n_outside
    blend = color_maps is not None
    # the view's one host read (render()'s expression over all rays), with the device status word of earlier kernels
    sample_dist = ops.check_status(dev, ((far - near) / S0).mean())
    t_rand = z_out_rand = None
    if perturb > 0:                                       # render()'s draws (:330-338), once for the whole view
        t_rand = torch.rand([N, 1], device=dev) - 0.5
        if O > 0:
            z_out_rand = torch.rand([O], device=dev)
    gamma = None
    if renderer.n_importance > 0 and renderer.upsampling_type != 'classical':
        gamma = float(renderer.beta_network.get_gamma().clip(1e-6, 1e6))
    heads = _heads(renderer, dev)
    cfg_args = (sample_dist, cos_anneal_ratio, 0.0, renderer.sparse_scale_factor, renderer.use_norm_grad_for_cosine,
                background_rgb, renderer.alpha_rule)
    rot = np.eye(3) if rot is None else np.asarray(rot, dtype=np.float64).reshape(3, 3)

    proj = imgs = None
    n_views = 0
    if blend:
        n_views = color_maps.shape[0]
        proj = (intrinsics[:, :3, :3] @ w2cs[:, :3, :]).reshape(n_views, 12).float().contiguous()
        imgs = color_maps.float().contiguous()
    ws = ViewWorkspace(renderer, N, workspace_bytes, dev, n_views)
    chunk = ws.chunk if max_chunk is None else max(1, min(ws.chunk, int(max_chunk)))

    f = lambda c: torch.empty(N, c, dtype=torch.float32, device=dev)
    out = {"color": f(3), "depth": f(1), "normal": f(3), "weight_sum": f(1)}
    if blend:
        out["color_pixel"] = f(3)
    z_lin = torch.linspace(0.0, 1.0, S0, device=dev)
    z_out0 = torch.linspace(1e-3, 1.0 - 1.0 / (O + 1.0), O, device=dev) if O > 0 else None
    if z_out_rand is not None:
        mids = .5 * (z_out0[..., 1:] + z_out0[..., :-1])
        upper = torch.cat([mids, z_out0[..., -1:]], -1)
        lower = torch.cat([z_out0[..., :1], mids], -1)
        z_out0 = lower + (upper - lower) * z_out_rand
    col_h, nerf_h = renderer.color_network._handle, (renderer.nerf._handle if O > 0 else None)
    udf_h = renderer.udf_network._handle

    for r0 in range(0, N, chunk):
        r1 = min(N, r0 + chunk)
        n = r1 - r0
        oc, dc, nc, fc = o[r0:r1], d[r0:r1], near[r0:r1], far[r0:r1]
        # ---- sampling, as render() (:598-645) ----
        z = nc + (fc - nc) * z_lin[None, :]
        if t_rand is not None:
            z = z + t_rand[r0:r1] * 2.0 / S0
        z = z.contiguous()
        if z_vals is not None:
            z = z_vals[r0:r1].float().contiguous()
        elif renderer.n_importance > 0:
            if renderer.upsampling_type == 'classical':
                z = renderer.importance_sample(oc, dc, z, sample_dist)
            else:
                z = renderer.importance_sample_mix(oc, dc, z, sample_dist, gamma=gamma)
        S = z.shape[1]
        assert S == ws.S, (S, ws.S)
        w = ws.carve(n)
        # ---- NeRF++ background of the outside columns (all columns when the pixel blend needs them) ----
        bg_alpha = bg_color = None
        if O > 0:
            z_feed, _ = torch.sort(torch.cat([z, fc / torch.flip(z_out0, dims=[-1]) + 1.0 / S0], dim=-1), dim=-1)
            z_feed = z_feed.contiguous()
            col0 = 0 if blend else S
            m = S + O - col0
            ops.outside_points_into(oc, dc, z_feed, col0, sample_dist, w["pts4"], w["odists"])
            ops.nerf_forward_into(nerf_h.desc(), nerf_h.images(), w["pts4"], dc, m, w["sigma"], w["rgb"], w["ctx"])
            bg_alpha, bg_color = w["bg_alpha"], w["bg_color"]
            bg_alpha[:, col0:] = 1.0 - torch.exp(-torch.nn.functional.relu(w["sigma"].reshape(n, m)) * w["odists"])
            bg_color[:, col0:] = w["rgb"].reshape(n, m, 3)
        # ---- fine pass ----
        ops.ray_points_into(oc, dc, z, sample_dist, w["pts"], w["mid"], w["dists"])
        udf_h.refresh()
        ops.udf_forward_split_into(udf_h, w["pts"], w["udf"], w["feat"], w["grad"], w["ctx"])
        col_h.refresh()
        ops.color_forward_into(col_h, w["pts"], dc, S, w["feat"], w["cb"], w["c"], w["bl"], w["ctx"])
        c_pix = None
        if blend:
            c_pix = w["c_pix"]
            ops.blend_pixels_into(w["pts"], proj, imgs, w["bl"], n, S, c_pix)
        cfg = ops._make_cfg(n, S, O, *cfg_args)
        ops.view_composite(cfg, heads, dc, w["pts"], w["mid"], w["dists"], w["udf"], w["grad"], w["c"], c_pix, bg_alpha,
                           bg_color, rot, {k: v[r0:r1] for k, v in out.items()})
    return {k: v.reshape(H, W, -1) for k, v in out.items()}


# ---------------------------------------------------------------------------------------------------------------
# DTU-layout scans (the reference's dataset/dataset.py, downsample_factor = 1)
# ---------------------------------------------------------------------------------------------------------------
def decompose_projection(P):
    """load_K_Rt_from_P of dataset.py:14-35 for a 3x4 / 4x4 matrix: (intrinsics [4,4] fp64, pose [4,4] fp32 c2w)."""
    import cv2
    K, R, t = cv2.decomposeProjectionMatrix(np.asarray(P)[:3, :4])[:3]
    K = K / K[2, 2]
    intrinsics = np.eye(4)
    intrinsics[:3, :3] = K
    pose = np.eye(4, dtype=np.float32)
    pose[:3, :3] = R.transpose()
    pose[:3, 3] = (t[:3] / t[3])[:, 0]
    return intrinsics, pose


def source_views(cam_loc, num=8):
    """prepare_ref_src_pairs / get_ref_src_info (dataset.py:129-149): for every camera the `num` nearest other camera
    centres, nearest first.  The distances are torch.cdist of the fp32 centres as the reference computes them (on the
    CPU: with more than 25 cameras cdist takes its matrix-product form, whose rounding can differ from the device's, so
    near-ties may still order differently from a runner on the GPU); exact ties are taken in index order (stable sort)."""
    c = torch.as_tensor(np.asarray(cam_loc), dtype=torch.float32).cpu()
    dist = torch.cdist(c[None], c[None], p=2.0)[0]
    order = torch.sort(dist, dim=1, stable=True).indices
    return order[:, 1:1 + num].numpy()


class Scan:
    """A DTU-layout scan as the reference's Dataset holds it: images [n, H, W, 3] (BGR / 256), intrinsics [n, 4, 4],
    intrinsics_inv, pose [n, 4, 4] (c2w), all fp32 on `device`, plus the file names and source-view table."""

    def __init__(self, data_dir, cameras="cameras.npz", device="cuda", num_src=8):
        import cv2
        self.data_dir = data_dir
        self.images_lis = sorted(glob.glob(os.path.join(data_dir, "image", "*.png")))
        if not self.images_lis:
            raise FileNotFoundError("no image/*.png under %s" % data_dir)
        self.n_images = len(self.images_lis)
        cams = np.load(os.path.join(data_dir, cameras))
        images = np.stack([cv2.imread(f) for f in self.images_lis]) / 256.0
        intr, poses = [], []
        for i in range(self.n_images):
            P = cams["world_mat_%d" % i].astype(np.float32) @ cams["scale_mat_%d" % i].astype(np.float32)
            k, p = decompose_projection(P)
            intr.append(torch.from_numpy(k).float())
            poses.append(torch.from_numpy(p).float())
        self.scale_mats_np = [cams["scale_mat_%d" % i].astype(np.float32) for i in range(self.n_images)]
        self.device = torch.device(device)
        self.images = torch.from_numpy(images.astype(np.float32)).to(self.device)
        self.intrinsics_all = torch.stack(intr).to(self.device)
        self.intrinsics_all_inv = torch.inverse(self.intrinsics_all)
        self.pose_all = torch.stack(poses).to(self.device)
        self.H, self.W = self.images.shape[1], self.images.shape[2]
        self.src = source_views(self.pose_all[:, :3, 3].cpu().numpy(), num_src)

    def image_at(self, idx, level):
        """dataset.py:337-339: the file resized to the view's grid (uint8 BGR)"""
        import cv2
        img = cv2.imread(self.images_lis[idx])
        return cv2.resize(img, (self.W // level, self.H // level)).clip(0, 255)

    def source_info(self, idx):
        """(color_maps [V,3,H,W], w2cs [V,4,4], intrinsics [V,4,4]) of the source views of `idx`, as validate() passes them"""
        s = torch.as_tensor(self.src[idx], device=self.device)
        return self.images[s].permute(0, 3, 1, 2), torch.inverse(self.pose_all[s]), self.intrinsics_all[s]

    def rays_at(self, idx, level):
        """gen_rays_at (dataset.py:151-164) through nudf_gen_rays_grid: rays_o, rays_d, near, far [H/l, W/l, .]"""
        return _rays_grid(self.intrinsics_all_inv[idx, :3, :3], self.pose_all[idx], self.W, self.H, level)


def load_scan(data_dir, cameras="cameras.npz", device="cuda"):
    return Scan(data_dir, cameras, device)


def _rays_grid(ki, pose, W, H, level):
    lib = L.lib()
    dev = pose.device
    Wl, Hl = W // level, H // level
    ki = ki.float().contiguous()
    pose = pose.float().contiguous()
    t = lambda c: torch.empty(Hl, Wl, c, device=dev)
    rays_o, rays_d, near, far = t(3), t(3), t(1), t(1)
    L.check(lib.nudf_gen_rays_grid(L.ptr(ki), L.ptr(pose), W, H, Wl, Hl, L.ptr(rays_o), L.ptr(rays_d), L.ptr(near), L.ptr(far),
                                   L.stream_ptr()), "nudf_gen_rays_grid")
    return rays_o, rays_d, near, far


def pose_between(pose_0, pose_1, ratio):
    """the interpolated c2w pose of gen_rays_between (dataset.py:296-327): slerp of the w2c rotations, linear w2c
    translation, in fp64 on the host, stored to fp32 before the final inverse as the reference does"""
    from scipy.spatial.transform import Rotation, Slerp
    w0 = np.linalg.inv(np.asarray(pose_0, dtype=np.float32))
    w1 = np.linalg.inv(np.asarray(pose_1, dtype=np.float32))
    rot = Slerp([0, 1], Rotation.from_matrix(np.stack([w0[:3, :3], w1[:3, :3]])))(ratio)
    pose = np.diag([1.0, 1.0, 1.0, 1.0]).astype(np.float32)
    pose[:3, :3] = rot.as_matrix()
    pose[:3, 3] = ((1.0 - ratio) * w0 + ratio * w1)[:3, 3]
    return np.linalg.inv(pose)


def rays_between(scan, i, j, ratio, level):
    """gen_rays_between (dataset.py:296-327): rays of the pose interpolated between views i and j, with the intrinsics
    of image 0.  Returns rays_o, rays_d, near, far [H/l, W/l, .] and the c2w pose."""
    pose = pose_between(scan.pose_all[i].cpu().numpy(), scan.pose_all[j].cpu().numpy(), ratio)
    pose_t = torch.from_numpy(pose).float().to(scan.device)
    return _rays_grid(scan.intrinsics_all_inv[0, :3, :3], pose_t, scan.W, scan.H, level) + (pose,)


# ---------------------------------------------------------------------------------------------------------------
# image files, as validate() forms them
# ---------------------------------------------------------------------------------------------------------------
def color_image(color):
    """validate()'s (c * 256).clip(0, 255) of an [H, W, 3] float array (:699)"""
    return (np.asarray(color) * 256).clip(0, 255)


def normal_image(normal):
    """validate()'s (n * 128 + 128).clip(0, 255) with the channels reversed for cv2 (:683, :720)"""
    return (np.asarray(normal) * 128 + 128).clip(0, 255)[:, :, ::-1]


def colorize_depth(depth, vmin, vmax):
    """the runner's colorize_depth (exp_runner_blending.py:847-865, plasma colormap, RGB uint8); None when matplotlib
    cannot be imported"""
    try:
        import matplotlib.cm
    except ImportError:
        return None
    value = np.asarray(depth)
    value = (value - vmin) / (vmax - vmin) if vmin != vmax else value * 0.
    return matplotlib.cm.get_cmap("plasma")(value, bytes=True)[:, :, :3]


def load_checkpoint(path):
    """a runner checkpoint, loaded with weights_only=True; the runner stores `iter_step` (and its optimiser's learning
    rates) as NumPy scalars, which are allowed here"""
    allowed = [np._core.multiarray.scalar, np.dtype, type(np.dtype(np.int64)), type(np.dtype(np.float64)),
               type(np.dtype(np.float32)), type(np.dtype(np.int32))]
    with torch.serialization.safe_globals(allowed):
        return torch.load(path, map_location="cpu", weights_only=True)


def color_network_from_state(cs):
    """A ResidualRenderingNetwork holding the state dict `cs` (the runner's `color_network_fine`), its shape read off the
    weights as networks_from_checkpoint describes"""
    from neuraludf_b200.models import fields as F
    n_lin = 0
    while "lin%d.weight_v" % n_lin in cs:
        n_lin += 1
    d_hidden, in0 = (int(x) for x in cs["lin0.weight_v"].shape)
    d_feature = int(cs["lin_base0.weight_v"].shape[1]) - 3
    col = F.ResidualRenderingNetwork(d_feature=d_feature, mode="no_normal", d_in=6, d_out=3, d_hidden=d_hidden,
                                     n_layers=n_lin - 1, weight_norm=True, multires_view=(in0 - d_hidden - 6) // 6,
                                     squeeze_out=True,
                                     blending_cand_views=int(cs["lin%d.weight_v" % (n_lin - 1)].shape[0]) - 3)
    col.load_state_dict(cs)
    return col


def networks_from_checkpoint(ck, device):
    """UDF, colour, NeRF++, variance and beta networks of a runner checkpoint (exp_runner_blending.py:484-495), their
    shapes read off the weights: the UDF network as mesh.udf_network_from_state; colour lin_base0 [d_hidden, 3 + d_feature],
    lin0 [d_hidden, d_hidden + 6 + 6 multires_view], last main layer [3 + blending views, d_hidden]; NeRF pts_linears.0
    [W, 4 + 8 multires], a layer after a skip [W, W + 4 + 8 multires], views_linears.0 [W/2, W + 3 + 6 multires_view]."""
    from neuraludf_b200.mesh import udf_network_from_state
    from neuraludf_b200.models import fields as F
    udf = udf_network_from_state(ck["udf_network_fine"])
    col = color_network_from_state(ck["color_network_fine"])
    ns = ck["nerf"]
    D = 0
    while "pts_linears.%d.weight" % D in ns:
        D += 1
    Wn, in_pts = (int(x) for x in ns["pts_linears.0.weight"].shape)
    skips = [l - 1 for l in range(1, D) if int(ns["pts_linears.%d.weight" % l].shape[1]) != Wn]
    in_view = int(ns["views_linears.0.weight"].shape[1]) - Wn
    nerf = F.NeRF(D=D, W=Wn, d_in=4, d_in_view=3, multires=(in_pts - 4) // 8, multires_view=(in_view - 3) // 6, output_ch=4,
                  skips=skips, use_viewdirs=True)
    nerf.load_state_dict(ns)
    var = F.SingleVarianceNetwork(init_val=0.0)
    var.load_state_dict(ck["variance_network_fine"])
    beta = F.BetaNetwork()
    beta.load_state_dict(ck["beta_network"])
    return [m.to(device) for m in (udf, col, nerf, var, beta)]


def main(argv=None):
    """python -m neuraludf_b200.render: a runner checkpoint's views (or views between two cameras) as the runner writes
    them (see INTEGRATION.md)"""
    import argparse
    import cv2
    from neuraludf_b200.models.udf_renderer_blending import UDFRendererBlending
    ap = argparse.ArgumentParser(prog="python -m neuraludf_b200.render",
                                 description="Render dataset views of a runner checkpoint (colour, blended colour, normals, "
                                             "depth) or views interpolated between two cameras.")
    ap.add_argument("--ckpt", required=True, help="checkpoint written by the runner")
    ap.add_argument("--scan_dir", required=True, help="DTU-layout scan: image/*.png and the cameras file")
    ap.add_argument("--cameras", default="cameras.npz")
    ap.add_argument("--views", type=int, nargs="*", default=None, help="indices of the dataset views to render")
    ap.add_argument("--between", type=int, nargs=2, metavar=("I", "J"), help="render --frames views from camera I to J")
    ap.add_argument("--frames", type=int, default=60)
    ap.add_argument("--level", type=int, default=4, help="resolution level (the image is divided by it)")
    ap.add_argument("--perturb", type=float, default=0.0)
    ap.add_argument("--anneal_end", type=float, default=25000.0)
    ap.add_argument("--cos_anneal_ratio", type=float, default=None,
                    help="default: the runner's, min(1, iter_step / anneal_end) (1 when anneal_end is 0)")
    ap.add_argument("--only_color", action="store_true", help="write novel_view/pred_{idx}.png and gt_{idx}.png only")
    ap.add_argument("--white_bkgd", action="store_true")
    ap.add_argument("--n_samples", type=int, default=64)
    ap.add_argument("--n_importance", type=int, default=50)
    ap.add_argument("--up_sample_steps", type=int, default=5)
    ap.add_argument("--n_outside", type=int, default=32)
    ap.add_argument("--upsampling_type", default="classical", choices=("classical", "mix"))
    ap.add_argument("--sdf2alpha_type", default="numerical", choices=("numerical", "theorical"),
                    help="the conf's sdf2alpha_type (a checkpoint does not record it)")
    ap.add_argument("--use_norm_grad_for_cosine", action="store_true")
    ap.add_argument("--workspace_gib", type=float, default=DEFAULT_WORKSPACE_BYTES / 2 ** 30)
    ap.add_argument("--out_dir", required=True)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("rendering runs on a CUDA device")
    if a.views is None and a.between is None:
        ap.error("give --views and / or --between")
    dev = torch.device("cuda", torch.cuda.current_device())
    ck = load_checkpoint(a.ckpt)
    udf, col, nerf, var, beta = networks_from_checkpoint(ck, dev)
    ren = UDFRendererBlending(nerf, udf, var, col, beta, n_samples=a.n_samples, n_importance=a.n_importance,
                              n_outside=a.n_outside, up_sample_steps=a.up_sample_steps, perturb=a.perturb,
                              sdf2alpha_type=a.sdf2alpha_type, upsampling_type=a.upsampling_type,
                              use_norm_grad_for_cosine=a.use_norm_grad_for_cosine)
    it = int(ck.get("iter_step", 0))
    ratio = a.cos_anneal_ratio
    if ratio is None:                                      # Runner.get_cos_anneal_ratio (exp_runner_blending.py:193-197)
        ratio = 1.0 if a.anneal_end == 0.0 else float(np.min([1.0, it / a.anneal_end]))
    bg = torch.ones([1, 3]) if a.white_bkgd else None
    scan = load_scan(a.scan_dir, a.cameras, dev)
    kw = dict(perturb=a.perturb, cos_anneal_ratio=ratio, background_rgb=bg, workspace_bytes=int(a.workspace_gib * 2 ** 30))
    written = []

    def write(sub, name, img):
        os.makedirs(os.path.join(a.out_dir, sub), exist_ok=True)
        path = os.path.join(a.out_dir, sub, name)
        cv2.imwrite(path, img)
        written.append(path)

    for idx in a.views or []:
        rays_o, rays_d, near, far = scan.rays_at(idx, a.level)
        cmaps, w2cs, intr = scan.source_info(idx)
        rot = np.linalg.inv(scan.pose_all[idx, :3, :3].cpu().numpy())          # validate(), :681
        out = render_view(ren, rays_o, rays_d, near, far, color_maps=cmaps, w2cs=w2cs, intrinsics=intr, rot=rot, **kw)
        out = {k: v.cpu().numpy() for k, v in out.items()}
        img_fine = color_image(out["color"])
        name = "{:0>8d}_{}.png".format(it, idx)
        if a.only_color:
            write("novel_view", "pred_{}.png".format(idx), img_fine)
            write("novel_view", "gt_{}.png".format(idx), scan.image_at(idx, a.level))
            continue
        write("validations_fine", name, np.concatenate([img_fine, color_image(out["color_pixel"]),
                                                         scan.image_at(idx, a.level)]))
        write("normals", name, normal_image(out["normal"]))
        depth = out["depth"][:, :, 0]
        os.makedirs(os.path.join(a.out_dir, "depth"), exist_ok=True)
        np.save(os.path.join(a.out_dir, "depth", "{:0>8d}_{}.npy".format(it, idx)), depth)
        last = (near.numel() - 1) // 512 * 512                   # validate() passes near / far[0, 0] of its last 512-ray batch
        vis = colorize_depth(depth, float(near.reshape(-1)[last]), float(far.reshape(-1)[last]))
        if vis is not None:
            write("depth", name, vis[:, :, ::-1])
    if a.between is not None:
        i, j = a.between
        for k in range(a.frames):
            r = k / max(a.frames - 1, 1)
            rays_o, rays_d, near, far, _ = rays_between(scan, i, j, r, a.level)
            out = render_view(ren, rays_o, rays_d, near, far, **kw)
            write("render", "{}.png".format(k), color_image(out["color"].cpu().numpy()))
    print("%d files under %s" % (len(written), a.out_dir))
    return written


if __name__ == "__main__":
    main()

"""Field networks with the reference's module API (mirror of `models/fields.py` of xxlong0/NeuralUDF), backed by
the libnudf CUDA kernels.

Same class names, constructor kwargs, parameter names / shapes (`lin{l}.weight_g/.weight_v/.bias`,
`lin_base{l}.*`, `pts_linears.{i}.weight`, `variance`, `beta/gamma/zeta`) and initialisation as the reference, so
`exp_runner_blending.py` constructs them unchanged and reference checkpoints load with `load_state_dict`.

    UDFNetwork                 reference models/fields.py:115-231
    ResidualRenderingNetwork   reference models/fields.py:400-495   (mode 'no_normal', the only one the confs use)
    NeRF                       reference models/fields.py:541-642   (use_viewdirs=True)
    SingleVarianceNetwork      reference models/fields.py:645-655
    BetaNetwork                reference models/fields.py:658-700
    color_blend                reference models/fields.py:498-537   (ft stage only; torch ops on the GPU for now)
"""
import math

import numpy as np
import torch
import torch.nn as nn

from .. import ops
from .embedder import get_embedder


class _WNLinear(nn.Module):
    """Parameter container with the state_dict layout of legacy `nn.utils.weight_norm(nn.Linear)` (dim=0):
    weight_g [out,1] = row norms, weight_v [out,in] = direction, bias [out].  The fold W = g v/||v|| happens once per
    optimiser step inside libnudf (nudf_*_fold_weights), not once per call."""

    def __init__(self, weight, bias):
        super().__init__()
        w = weight.detach().clone()
        self.bias = nn.Parameter(bias.detach().clone())
        self.weight_g = nn.Parameter(w.norm(dim=1, keepdim=True))
        self.weight_v = nn.Parameter(w)

    @property
    def weight(self):
        return torch._weight_norm(self.weight_v, self.weight_g, 0)


def _new_linear(din, dout):
    """nn.Linear's default initialisation, consuming the global RNG exactly like the reference's constructors."""
    lin = nn.Linear(din, dout)
    return lin.weight.data, lin.bias.data


class UDFNetwork(nn.Module):
    """Unsigned-distance MLP: PE -> n_layers softplus(beta=100) layers with a skip concat -> [udf | feature].

    forward / udf / udf_hidden_appearance / gradient follow reference models/fields.py:192-231.  `gradient` is the
    exact input-gradient (reverse sweep inside the kernel library), differentiable w.r.t. the parameters (the
    second-order terms the reference obtains with create_graph=True).
    """

    def __init__(self, d_in, d_out, d_hidden, n_layers, skip_in=(4,), multires=0, scale=1, bias=0.5,
                 geometric_init=True, weight_norm=True, udf_type='abs', udf_shift=None, predict_grad=None):
        # udf_shift / predict_grad: passed by confs/udf_garment_blending.conf:85,89 although the reference's __init__
        # does not accept them (TypeError as shipped); accepted and ignored here.
        super().__init__()
        if not weight_norm:
            raise NotImplementedError("UDFNetwork(weight_norm=False) is not supported by the CUDA path; every shipped "
                                      "conf uses weight_norm=True")
        if udf_type != 'abs':
            raise NotImplementedError("udf_type=%r: only 'abs' (all shipped confs) is implemented" % (udf_type,))
        if d_in != 3:
            raise NotImplementedError("d_in must be 3")
        skip_in = tuple(skip_in)
        if len(skip_in) > 1:
            raise NotImplementedError("at most one skip connection is supported")
        dims = [d_in] + [d_hidden for _ in range(n_layers)] + [d_out]
        self.embed_fn_fine = None
        if multires > 0:
            self.embed_fn_fine, input_ch = get_embedder(multires, input_dims=d_in)
            dims[0] = input_ch
        self.num_layers = len(dims)
        self.skip_in = skip_in
        self.scale = scale
        self.geometric_init = geometric_init
        self.multires = multires
        self.d_out = d_out
        self.udf_type = udf_type
        layers = []
        for l in range(0, self.num_layers - 1):
            out_dim = dims[l + 1] - dims[0] if (l + 1) in skip_in else dims[l + 1]
            w, b = _new_linear(dims[l], out_dim)
            if geometric_init:   # reference models/fields.py:156-173
                if l == self.num_layers - 2:
                    torch.nn.init.normal_(w, mean=np.sqrt(np.pi) / np.sqrt(dims[l]), std=0.0001)
                    torch.nn.init.constant_(b, -bias)
                elif multires > 0 and l == 0:
                    torch.nn.init.constant_(b, 0.0)
                    torch.nn.init.constant_(w[:, 3:], 0.0)
                    torch.nn.init.normal_(w[:, :3], 0.0, np.sqrt(2) / np.sqrt(out_dim))
                elif multires > 0 and l in skip_in:
                    torch.nn.init.constant_(b, 0.0)
                    torch.nn.init.normal_(w, 0.0, np.sqrt(2) / np.sqrt(out_dim))
                    torch.nn.init.constant_(w[:, -(dims[0] - 3):], 0.0)
                else:
                    torch.nn.init.constant_(b, 0.0)
                    torch.nn.init.normal_(w, 0.0, np.sqrt(2) / np.sqrt(out_dim))
            lin = _WNLinear(w, b)
            setattr(self, "lin" + str(l), lin)
            layers.append(lin)
        skip_layer = skip_in[0] if (len(skip_in) == 1 and 1 <= skip_in[0] <= self.num_layers - 2) else -1
        self._handle = ops.UdfHandle(layers, d_in, multires, d_out, skip_layer, scale)

    # -- kernel-backed entry points ------------------------------------------------------------------------------
    def value_and_gradient(self, x):
        """(forward(x) [P,d_out], d udf/d x [P,3]) from ONE fused evaluation (the reference evaluates the network
        twice for this, udf_renderer_blending.py:364 and :368)."""
        return ops.udf_forward(self._handle, x.reshape(-1, 3), True)

    def value_feature_gradient(self, x):
        """(udf [P,1], feature [P,d_out-1], d udf/d x [P,3]) as separate tensors from ONE fused evaluation: render_core's form."""
        return ops.udf_forward_split(self._handle, x.reshape(-1, 3), True)

    def forward(self, inputs):
        out, _ = ops.udf_forward(self._handle, inputs.reshape(-1, 3), False)
        return out

    def udf(self, x):
        return self.forward(x)[:, :1]

    def udf_hidden_appearance(self, x):
        return self.forward(x)

    def udf_values(self, x):
        """udf [P] only, no autograd, no saved activations (importance sampling, grid extraction)."""
        return ops.udf_value(self._handle, x.reshape(-1, 3))

    def value_gradient(self, x):
        """(udf [P], d udf/d x [P,3]) from ONE fused evaluation without the feature output and without autograd (surface
        projection, cloud.udf_point_cloud): the bits of value_and_gradient's udf column and gradient."""
        return ops.udf_value_gradient(self._handle, x.reshape(-1, 3))

    def gradient(self, x):
        if x.is_leaf and x.dtype.is_floating_point:
            x.requires_grad_(True)          # side effect of the reference (fields.py:220); the value is not used
        _, g = ops.udf_forward(self._handle, x.detach().reshape(-1, 3), True)
        return g.unsqueeze(1)


class ResidualRenderingNetwork(nn.Module):
    """Two ReLU stacks (base colour from geometry features, view-dependent residual stack) with sigmoid colour heads
    and `blending_cand_views` blending logits; reference models/fields.py:400-495."""

    def __init__(self, d_feature, mode, d_in, d_out, d_hidden, n_layers, weight_norm=True, multires_view=0,
                 squeeze_out=True, blending_cand_views=10):
        super().__init__()
        if mode != 'no_normal':
            raise NotImplementedError("ResidualRenderingNetwork mode %r: only 'no_normal' (all shipped confs) is "
                                      "implemented on the CUDA path" % (mode,))
        if not weight_norm:
            raise NotImplementedError("weight_norm=False is not supported by the CUDA path")
        if not squeeze_out:
            raise NotImplementedError("squeeze_out=False is not supported")
        if d_in != 6:
            # mode 'no_normal' feeds cat([points, feature]) (3 + d_feature wide) to lin_base0, which the reference sizes
            # d_in - 3 + d_feature: any other d_in is a shape error there, and would fold garbage here
            raise NotImplementedError("ResidualRenderingNetwork mode 'no_normal' needs d_in = 6 (points + view "
                                      "direction), got d_in=%d" % (d_in,))
        self.mode = mode
        self.squeeze_out = squeeze_out
        self.d_out = d_out
        dims_base = [d_in - 3 + d_feature] + [d_hidden for _ in range(n_layers)] + [d_out]
        dims = [d_hidden + d_out + 3] + [d_hidden for _ in range(n_layers)] + [d_out + blending_cand_views]
        self.embedview_fn = None
        if multires_view > 0:
            self.embedview_fn, input_ch = get_embedder(multires_view)
            dims[0] += (input_ch - 3)
        self.num_layers = len(dims)
        main, base = [], []
        for l in range(0, self.num_layers - 1):          # same construction order as the reference (RNG parity)
            w, b = _new_linear(dims[l], dims[l + 1])
            lin = _WNLinear(w, b)
            setattr(self, "lin" + str(l), lin)
            main.append(lin)
        for l in range(0, self.num_layers - 1):
            w, b = _new_linear(dims_base[l], dims_base[l + 1])
            lin = _WNLinear(w, b)
            setattr(self, "lin_base" + str(l), lin)
            base.append(lin)
        self.if_blending = blending_cand_views > 0
        self._handle = ops.ColorHandle(base, main, d_feature, d_hidden, d_out, blending_cand_views, multires_view)

    def forward(self, points, normals, view_dirs, feature_vectors):
        cb, c, bl = ops.color_forward(self._handle, points.reshape(-1, 3), view_dirs.reshape(-1, 3), feature_vectors, 0)
        return (cb, c, bl) if self.if_blending else (cb, c)

    def forward_rays(self, points, rays_d, samples_per_ray, feature_vectors):
        """Same as forward() with view_dirs = rays_d expanded over the samples of each ray, without materialising it."""
        cb, c, bl = ops.color_forward(self._handle, points.reshape(-1, 3), rays_d.reshape(-1, 3), feature_vectors,
                                      samples_per_ray)
        return cb, c, bl


def color_blend(blending_weights, img_index, pts_pixel_color=None, pts_pixel_mask=None, pts_patch_color=None,
                pts_patch_mask=None):
    """Blend per-view pixel / patch colours with a masked softmax over the blending logits
    (reference models/fields.py:498-537).  Fine-tuning stage only; plain torch ops on the GPU (SURVEY 8(f) rank 1)."""
    nviews = pts_pixel_color.shape[-2]
    if img_index is not None:
        logits = torch.index_select(blending_weights, 1, img_index.long())
    else:
        logits = blending_weights[:, :, :nviews]
    sm = torch.softmax(logits, dim=-1)
    w_pix = sm * pts_pixel_mask
    w_pix = w_pix / (w_pix.float().sum(dim=-1, keepdim=True) + 1e-8)
    final_pixel_color = (pts_pixel_color * w_pix[..., None]).sum(dim=-2)
    final_pixel_mask = pts_pixel_mask.float().sum(dim=-1, keepdim=True) > 0
    final_patch_color, final_patch_mask = None, None
    if pts_patch_color is not None:
        npx = pts_patch_color.shape[3]
        patch_mask = pts_patch_mask.sum(dim=-1) > npx - 1
        w_pat = sm * patch_mask
        w_pat = w_pat / (w_pat.float().sum(dim=-1, keepdim=True) + 1e-8)
        final_patch_color = (pts_patch_color * w_pat[:, :, :, None, None]).sum(dim=-3)
        final_patch_mask = patch_mask.sum(dim=-1, keepdim=True) > 0
    return final_pixel_color, final_pixel_mask, final_patch_color, final_patch_mask


class NeRF(nn.Module):
    """NeRF++ background network (reference models/fields.py:541-628), use_viewdirs=True."""

    def __init__(self, D=8, W=256, d_in=3, d_in_view=3, multires=0, multires_view=0, output_ch=4, skips=[4],
                 use_viewdirs=False, occupancy=True):
        super().__init__()
        if not use_viewdirs:
            raise NotImplementedError("NeRF(use_viewdirs=False) asserts False in the reference as well (fields.py:628)")
        if d_in_view != 3:
            raise NotImplementedError("d_in_view must be 3")
        skips = list(skips)
        if len(skips) > 1:
            raise NotImplementedError("at most one skip connection is supported")
        self.D, self.W, self.d_in, self.d_in_view = D, W, d_in, d_in_view
        self.input_ch, self.input_ch_view = d_in, 3
        self.embed_fn, self.embed_fn_view = None, None
        self.occupancy = occupancy
        if multires > 0:
            self.embed_fn, self.input_ch = get_embedder(multires, input_dims=d_in)
        if multires_view > 0:
            self.embed_fn_view, self.input_ch_view = get_embedder(multires_view, input_dims=d_in_view)
        self.skips = skips
        self.use_viewdirs = use_viewdirs
        self.pts_linears = nn.ModuleList(
            [nn.Linear(self.input_ch, W)] +
            [nn.Linear(W, W) if i not in self.skips else nn.Linear(W + self.input_ch, W) for i in range(D - 1)])
        self.views_linears = nn.ModuleList([nn.Linear(self.input_ch_view + W, W // 2)])
        self.feature_linear = nn.Linear(W, W)
        self.alpha_linear = nn.Linear(W, 1)
        self.rgb_linear = nn.Linear(W // 2, 3)
        skip = skips[0] if skips else -1
        self._handle = ops.NerfHandle(self, D, W, d_in, multires, multires_view, skip)

    def forward(self, input_pts, input_views):
        if input_views is None:
            raise NotImplementedError("NeRF.forward(pts, None) (density only) is not on the render path")
        return ops.nerf_forward(self._handle, input_pts.reshape(-1, self.d_in), input_views.reshape(-1, 3), 0)

    def forward_rays(self, input_pts, rays_d, samples_per_ray):
        return ops.nerf_forward(self._handle, input_pts.reshape(-1, self.d_in), rays_d.reshape(-1, 3), samples_per_ray)


class SingleVarianceNetwork(nn.Module):
    """inv_s = exp(10 * variance), reference models/fields.py:645-655."""

    def __init__(self, init_val, requires_grad=True):
        super().__init__()
        self.variance = nn.Parameter(torch.Tensor([init_val]), requires_grad=requires_grad)

    def set_trainable(self):
        self.variance.requires_grad = True

    def forward(self, x):
        return torch.ones([len(x), 1], device=x.device) * torch.exp(self.variance * 10.0)


class BetaNetwork(nn.Module):
    """beta = clip(exp(10 b), 0, 1/beta_min), gamma = exp(10 g), zeta = |z|; reference models/fields.py:658-700."""

    def __init__(self, init_var_beta=0.1, init_var_gamma=0.1, init_var_zeta=0.05, beta_min=0.00005,
                 requires_grad_beta=True, requires_grad_gamma=True, requires_grad_zeta=True):
        super().__init__()
        self.beta = nn.Parameter(torch.Tensor([init_var_beta]), requires_grad=requires_grad_beta)
        self.gamma = nn.Parameter(torch.Tensor([init_var_gamma]), requires_grad=requires_grad_gamma)
        self.zeta = nn.Parameter(torch.Tensor([init_var_zeta]), requires_grad=requires_grad_zeta)
        self.beta_min = beta_min

    def get_beta(self):
        return torch.exp(self.beta * 10).clip(0, 1. / self.beta_min)

    def get_gamma(self):
        return torch.exp(self.gamma * 10)

    def get_zeta(self):
        return self.zeta.abs()

    def set_beta_trainable(self):
        self.beta.requires_grad = True

    @torch.no_grad()
    def set_gamma(self, x):
        self.gamma = nn.Parameter(torch.Tensor([x]).to(self.gamma.device), requires_grad=self.gamma.requires_grad)

    def forward(self):
        return self.get_beta(), self.get_gamma(), self.get_zeta()


class _NotOnRenderPath(nn.Module):
    _why = ""

    def __init__(self, *a, **k):
        super().__init__()
        raise NotImplementedError(self._why)


class SDFNetwork(_NotOnRenderPath):
    _why = ("SDFNetwork (reference models/fields.py:10-112) is never constructed by exp_runner_blending.py "
            "(model_type 'neus' paths are dead code there); out of scope of the UDF render path")


class RenderingNetwork(_NotOnRenderPath):
    _why = ("RenderingNetwork (reference models/fields.py:325-397) returns 1-2 tensors while render_core unpacks 3 "
            "(udf_renderer_blending.py:425); the runner uses ResidualRenderingNetwork")


class BlendingNetwork(_NotOnRenderPath):
    _why = "BlendingNetwork (reference models/fields.py:235-322) is not used by exp_runner_blending.py"

"""The colour and NeRF++ modules refuse shapes the CUDA path cannot run, instead of folding weights of another shape.

The library plans every layer of these networks from a few numbers (d_feature, d_hidden, d_out, views, multires_view; D,
W, d_in, multires, skip) and reads each weight as [n_out, n_in] of its plan.  A parameter of any other shape would be read
with the wrong row length, so the handles compare every parameter with the planned shape before they build a descriptor.
Constructing the modules and their descriptors needs no device."""
import pytest
import torch
import torch.nn as nn

from neuraludf_b200.models import fields as F
from oracle import oracle_torch as O


def _color(**kw):
    args = dict(d_feature=64, mode="no_normal", d_in=6, d_out=3, d_hidden=100, n_layers=3, weight_norm=True, multires_view=2,
                squeeze_out=True, blending_cand_views=12)
    args.update(kw)
    return F.ResidualRenderingNetwork(**args)


def _nerf(**kw):
    args = dict(D=5, W=33, d_in=4, d_in_view=3, multires=10, multires_view=4, output_ch=4, skips=[2], use_viewdirs=True)
    args.update(kw)
    return F.NeRF(**args)


def test_color_no_normal_needs_d_in_6():
    # the reference sizes lin_base0 as d_in - 3 + d_feature = 73 inputs but feeds it cat([points, feature]) = 67 columns
    with pytest.raises(NotImplementedError, match="d_in = 6"):
        _color(d_in=9)


@pytest.mark.parametrize("n_layers,d_hidden,d_feature,d_out,views,mv", [(2, 64, 32, 1, 0, 0), (4, 256, 256, 3, 29, 6),
                                                                        (15, 48, 16, 3, 10, 4), (4, 16, 13, 2, 5, 4)])
def test_color_layer_shapes_match_the_plan(n_layers, d_hidden, d_feature, d_out, views, mv):
    col = _color(n_layers=n_layers, d_hidden=d_hidden, d_feature=d_feature, d_out=d_out, blending_cand_views=views,
                 multires_view=mv)
    cc = O.color_cfg(d_feature=d_feature, d_out=d_out, d_hidden=d_hidden, n_layers=n_layers, multires_view=mv,
                     blending_cand_views=views)
    n_lin = n_layers + 1
    want = [(cc["dims_base"][l + 1], cc["dims_base"][l]) for l in range(n_lin)] + \
           [(cc["dims"][l + 1], cc["dims"][l]) for l in range(n_lin)]
    assert col._handle.layer_shapes() == want
    d = col._handle._make_desc()
    assert d.n_lin == n_lin


@pytest.mark.parametrize("layer", ["lin_base0", "lin1", "lin3"])
def test_color_mismatched_weight_raises(layer):
    col = _color()
    m = getattr(col, layer)
    n_out, n_in = m.weight_v.shape
    m.weight_v = nn.Parameter(torch.zeros(n_out, n_in + 1))
    # the handle keeps the module's layer objects: the swapped parameter is what the next fold would read
    with pytest.raises(RuntimeError, match="the library plans"):
        col._handle._make_desc()


def test_color_mismatched_bias_raises():
    col = _color()
    col.lin2.bias = nn.Parameter(torch.zeros(col.lin2.bias.numel() + 1))
    with pytest.raises(RuntimeError, match="the library plans"):
        col._handle._make_desc()


@pytest.mark.parametrize("D,W,skip,d_in,multires,mv", [(2, 64, None, 3, 0, 0), (4, 100, 0, 4, 6, 2), (16, 32, 14, 4, 10, 4),
                                                       (5, 33, 2, 4, 10, 4)])
def test_nerf_layer_shapes_match_the_plan(D, W, skip, d_in, multires, mv):
    nerf = _nerf(D=D, W=W, skips=[] if skip is None else [skip], d_in=d_in, multires=multires, multires_view=mv)
    d = nerf._handle.desc()
    assert (d.D, d.W, d.skip) == (D, W, -1 if skip is None else skip)
    for lin, shape in nerf._handle.layer_shapes():
        assert tuple(lin.weight.shape) == shape


def test_nerf_mismatched_descriptor_raises():
    nerf = _nerf()
    # a pts layer built without the skip concatenation: [W, W] where the plan reads [W, W + ch]
    nerf.pts_linears[3] = nn.Linear(33, 33)
    with pytest.raises(RuntimeError, match="the library plans"):
        nerf._handle.desc()


@pytest.mark.parametrize("head", ["views", "feature", "alpha", "rgb"])
def test_nerf_mismatched_head_raises(head):
    nerf = _nerf()
    if head == "views":
        nerf.views_linears[0] = nn.Linear(33 + 27, 17)
    else:
        name = head + "_linear"
        old = getattr(nerf, name)
        setattr(nerf, name, nn.Linear(old.in_features + 1, old.out_features))
    with pytest.raises(RuntimeError, match="the library plans"):
        nerf._handle.desc()


def test_nerf_layer_count_raises():
    nerf = _nerf()
    nerf.pts_linears.append(nn.Linear(33, 33))
    with pytest.raises(RuntimeError, match="pts_linears"):
        nerf._handle.desc()

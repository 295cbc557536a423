"""ops.composite reads its udf argument through a row stride and indexes every per-sample tensor by ray and sample with no
bound of its own, so the wrapper works the stride out from the udf it was given and refuses mis-sized tensors with a
ValueError before it touches the library.  Both happen on the host: CPU tensors are enough to check them (a well-shaped
CPU call gets as far as the CUDA-tensor check)."""
import pytest
import torch

from neuraludf_b200 import ops

N, S, O_ = 3, 5, 2
P = N * S


def _args(**over):
    a = dict(udf=torch.rand(P), grads=torch.rand(P, 3), scb=torch.rand(P, 3), sc=torch.rand(P, 3),
             bg_alpha=torch.rand(N, S + O_), bg_color=torch.rand(N, S + O_, 3), heads=torch.tensor([400.0, 150.0, 20.0]),
             geom=(torch.rand(N, 3), torch.rand(P, 3), torch.rand(N, S), torch.rand(N, S)))
    a.update(over)
    return a


def _call(a):
    cfg = ops._make_cfg(N, S, O_, 0.01, None, 0.0, 300.0, False, None)
    return ops.composite(a["udf"], a["grads"], a["scb"], a["sc"], a["bg_alpha"], a["bg_color"], a["heads"], a["geom"], cfg)


@pytest.mark.parametrize("shape", ["P", "P1", "NS", "column"])
def test_udf_layouts_are_accepted(shape):
    base = torch.rand(P, 5)
    udf = {"P": base[:, 0].contiguous(), "P1": base[:, :1].contiguous(), "NS": base[:, 0].reshape(N, S).contiguous(),
           "column": base[:, 2]}[shape]
    view, ld = ops._composite_udf(udf, N, S)
    assert view.shape == (P,) and ld == (5 if shape == "column" else 1)
    assert view.data_ptr() == udf.data_ptr()             # no copy: the kernels read the caller's memory
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        _call(_args(udf=udf))


@pytest.mark.parametrize("udf", [torch.rand(P - 1), torch.rand(P, 2), torch.rand(S, N), torch.rand(N, S, 1), torch.rand(1, P)],
                         ids=["short", "P2", "SN", "NS1", "1P"])
def test_udf_of_another_shape_raises(udf):
    with pytest.raises(ValueError, match="udf of shape"):
        _call(_args(udf=udf))


@pytest.mark.parametrize("name,t", [("grads", torch.rand(P - 1, 3)), ("scb", torch.rand(P, 2)), ("sc", torch.rand(P + 1, 3)),
                                    ("bg_alpha", torch.rand(N, S)), ("bg_color", torch.rand(N, S + O_, 4)),
                                    ("heads", torch.rand(2))])
def test_mis_sized_tensor_raises(name, t):
    with pytest.raises(ValueError, match=name):
        _call(_args(**{name: t}))


@pytest.mark.parametrize("i,name,t", [(0, "rays_d", torch.rand(N + 1, 3)), (1, "pts", torch.rand(P - 1, 3)),
                                      (2, "mid", torch.rand(N, S - 1)), (3, "dists", torch.rand(N + 1, S))])
def test_mis_sized_geometry_raises(i, name, t):
    geom = list(_args()["geom"])
    geom[i] = t
    with pytest.raises(ValueError, match=name):
        _call(_args(geom=tuple(geom)))

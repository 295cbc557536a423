"""CPU-side checks of the drop-in boundary: the C-ABI library loads and exports every symbol include/nudf.h
declares; the product path refuses to run without CUDA (no silent fallback)."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_functions():
    txt = open(os.path.join(ROOT, "include", "nudf.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(nudf_[a-z0-9_]+)\s*\(", txt)))


def test_library_exports_the_declared_abi():
    from neuraludf_b200 import _lib
    assert os.path.exists(_lib.LIB_PATH), "libnudf.so missing: run `python -m neuraludf_b200.build`"
    L = _lib.lib()
    declared = _header_functions()
    assert len(declared) >= 30
    for name in declared:
        assert hasattr(L, name), "libnudf.so does not export %s" % name
    assert sorted(_lib.exported_symbols()) == declared, "python binding and include/nudf.h disagree"
    assert L.nudf_abi_version() == 6


def test_python_constants_match_the_header():
    """every constant _lib mirrors equals include/nudf.h's #define (a smaller COMPACT_SEG would let the count pass write
    past the counts buffer)"""
    from neuraludf_b200 import _lib
    txt = open(os.path.join(ROOT, "include", "nudf.h")).read()
    header = {k: int(v) for k, v in re.findall(r"^#define NUDF_([A-Z0-9_]+)[ \t]+(-?\d+)\b", txt, flags=re.M)}
    mirrors = {"COMPACT_SEG": _lib.COMPACT_SEG, "BRICK": _lib.BRICK, "PT_MAX_VIEWS": _lib.PT_MAX_VIEWS,
               "PT_MAX_CAND": _lib.PT_MAX_CAND, "MAX_LAYERS": _lib.MAX_LAYERS,
               "STATUS_NONFINITE_SAMPLES": _lib.STATUS_NONFINITE_SAMPLES,
               "STATUS_NONFINITE_RENDER": _lib.STATUS_NONFINITE_RENDER}
    mirrors.update(("PATCH_" + name.upper(), v) for name, v in _lib.PATCH_TYPES.items())
    for name, v in mirrors.items():
        assert header.get(name) == v, "_lib mirrors NUDF_%s as %r, include/nudf.h has %r" % (name, v, header.get(name))


def test_descriptor_validation_runs_without_gpu():
    from neuraludf_b200 import _lib
    import ctypes
    L = _lib.lib()
    d = _lib.UdfDesc()
    d.n_lin = 1          # invalid: needs >= 2
    assert L.nudf_udf_folded_floats(ctypes.byref(d)) == -1
    assert b"n_lin" in L.nudf_last_error()
    # a valid DTU-shaped descriptor: sizes are computed on the host
    d = _lib.UdfDesc()
    d.n_lin, d.d_in, d.multires, d.d_out, d.skip_layer, d.scale = 9, 3, 6, 257, 4, 1.0
    dims = [(39, 256), (256, 256), (256, 256), (256, 217), (256, 256), (256, 256), (256, 256), (256, 256), (256, 257)]
    for l, (i, o) in enumerate(dims):
        d.in_dim[l], d.out_dim[l] = i, o
    n = L.nudf_udf_folded_floats(ctypes.byref(d))
    # fp32 folded weights (>= 524 544 floats) followed by the bf16 hi/lo tensor-engine images of every layer
    assert 524544 <= n < 8 * 1024 * 1024
    assert L.nudf_udf_ctx_floats(ctypes.byref(d), 1024, 1) > L.nudf_udf_ctx_floats(ctypes.byref(d), 1024, 0) > 0
    # the activation context must start 16-byte aligned: refused before any device work (the pointers are never read)
    assert L.nudf_udf_forward(ctypes.byref(d), 4096, 4096, 128, None, 0, None, 4100, None) == -1
    assert b"16-byte aligned" in L.nudf_last_error()
    assert L.nudf_udf_value(ctypes.byref(d), 4096, 4096, 128, 8192, 4100, None) == -1
    assert b"16-byte aligned" in L.nudf_last_error()
    n = _lib.NerfDesc()
    n.D, n.W, n.d_in, n.multires, n.multires_view, n.skip = 8, 256, 4, 10, 4, 4
    assert L.nudf_nerf_forward(ctypes.byref(n), None, 4096, 4096, 1, 128, 4096, 4096, 4100, None) == -1
    assert b"16-byte aligned" in L.nudf_last_error()


def test_lattice_descriptor_validation_runs_without_gpu():
    from neuraludf_b200 import _lib
    import ctypes
    L = _lib.lib()
    store = _lib.BrickStore(4, 1, 4, 1, 0, 1, 1, None, None)
    for lat, what in ((_lib.Lattice(4, 4, 4, 1, ctypes.pointer(store)), b"exactly one of df and store"),
                      (_lib.Lattice(4, 4, 4, None, None), b"exactly one of df and store"),
                      (_lib.Lattice(4, 4, 1, 1, None), b"at least 2"),
                      (_lib.Lattice(4, 4, 5, None, ctypes.pointer(store)), b"the store's n")):
        assert L.nudf_mc_links(ctypes.byref(lat), None, 0, None, None, None) == -1
        assert what in L.nudf_last_error()
    lat = _lib.Lattice(4, 4, 4, None, ctypes.pointer(store))
    assert L.nudf_iso_active(ctypes.byref(lat), 0.0, 1, None) == -1
    assert b"df lattice" in L.nudf_last_error()
    lat = _lib.Lattice(4, 4, 5, 1, None)
    assert L.nudf_nb_block_test(ctypes.byref(lat), 1, None, 0, ctypes.byref(_lib.BandCoords(0.5)), 2.0, 0.1, None, 1,
                                None) == -1
    assert b"cubic" in L.nudf_last_error()


def test_render_cfg_alpha_rule_validation_runs_without_gpu():
    from neuraludf_b200 import _lib
    import ctypes
    L = _lib.lib()
    cfg = _lib.RenderCfg()
    cfg.n_rays, cfg.n_samples = 4, 64
    calls = (lambda: L.nudf_render_composite_forward(ctypes.byref(cfg), *[None] * 6, 1, *[None] * 7),
             lambda: L.nudf_render_view_forward(ctypes.byref(cfg), *[None] * 6, 1, *[None] * 8),
             lambda: L.nudf_render_composite_backward(ctypes.byref(cfg), *[None] * 6, 1, *[None] * 14))
    for call in calls:
        cfg.alpha_rule = 2
        assert call() == -1
        assert b"alpha_rule" in L.nudf_last_error()
        cfg.alpha_rule = 1       # a valid rule gets as far as the pointers
        assert call() == -1
        assert b"null pointer" in L.nudf_last_error()


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_no_cpu_fallback():
    from neuraludf_b200.models.fields import UDFNetwork
    net = UDFNetwork(d_in=3, d_out=257, d_hidden=64, n_layers=4, skip_in=(2,), multires=6)
    with pytest.raises(RuntimeError, match="CUDA"):
        net(torch.zeros(4, 3))


def test_state_dict_layout_matches_reference_names():
    from neuraludf_b200.models.fields import UDFNetwork, ResidualRenderingNetwork, NeRF, SingleVarianceNetwork, BetaNetwork
    udf = UDFNetwork(d_in=3, d_out=257, d_hidden=256, n_layers=8, skip_in=(4,), multires=6, bias=0.5, scale=1.0,
                     geometric_init=True, weight_norm=True, udf_type='abs')
    sd = udf.state_dict()
    assert sum(v.numel() for v in sd.values()) == 529076            # SURVEY App. B
    assert tuple(sd["lin3.weight_v"].shape) == (217, 256) and tuple(sd["lin3.weight_g"].shape) == (217, 1)
    assert tuple(sd["lin8.weight_v"].shape) == (257, 256) and tuple(sd["lin0.weight_v"].shape) == (256, 39)
    col = ResidualRenderingNetwork(d_feature=256, mode='no_normal', d_in=6, d_out=3, d_hidden=128, n_layers=4,
                                   weight_norm=True, multires_view=4, squeeze_out=True, blending_cand_views=10)
    sdc = col.state_dict()
    assert sum(v.numel() for v in sdc.values()) == 155808
    assert tuple(sdc["lin0.weight_v"].shape) == (128, 158) and tuple(sdc["lin_base0.weight_v"].shape) == (128, 259)
    nerf = NeRF(D=8, d_in=4, d_in_view=3, W=256, multires=10, multires_view=4, output_ch=4, skips=[4], use_viewdirs=True)
    assert sum(v.numel() for v in nerf.state_dict().values()) == 606596
    assert tuple(nerf.state_dict()["pts_linears.5.weight"].shape) == (256, 340)
    assert list(SingleVarianceNetwork(0.3).state_dict()) == ["variance"]
    assert sorted(BetaNetwork().state_dict()) == ["beta", "gamma", "zeta"]


def test_golden_scene_loads_into_modules(golden):
    from tests.gpu_util import build_modules
    build_modules(golden, device="cpu")
    build_modules(golden, device="cpu", udf_name="udf_small")


def test_launcher_shadows_the_reference_module_names():
    import subprocess
    import sys
    code = ("import sys; sys.path.insert(0, %r); from neuraludf_b200.launch import install_shadow_modules; "
            "install_shadow_modules(); from models.fields import UDFNetwork, ResidualRenderingNetwork, NeRF, "
            "SingleVarianceNetwork, BetaNetwork, SDFNetwork; from models.udf_renderer_blending import "
            "UDFRendererBlending, extract_fields, extract_gradient_fields, sample_pdf; from models.embedder import "
            "get_embedder; import models.fields as f; assert 'neuraludf_b200' in f.__file__; print('ok')" % ROOT)
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr[-2000:]

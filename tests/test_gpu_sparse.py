"""Block-sparse narrow-band meshing (grid.udf_band_sparse, mesh.udf_mesh_sparse, csrc/mesh_sparse.cu and the BrickDf
instantiations of csrc/mesh_udf.cu / mesh_band.cu): the store against udf_band's dense df, the near-surface selection,
and the mesh against udf_mesh_band bit for bit on the C5 network and the analytic fields; udf_mesh_post(sparse=True);
2048^3 against a dense slab of the same lattice, its raw mesh an oriented two-manifold, its memory below N^3 bytes beside
the value chain's batch workspace; determinism; the 2048^3 CLI."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.gpu_util import report
from tests.proto import mesh_cases as C
from tests.test_gpu_band import _Analytic

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def c5(golden):
    _dev()
    from tests.gpu_util import build_modules
    return build_modules(golden, "cuda")[0]


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


@pytest.mark.parametrize("N", [256, 512])
def test_store_reads_udf_band(c5, N):
    from neuraludf_b200 import grid
    df, info = grid.udf_band(c5, N)
    band, sinfo = grid.udf_band_sparse(c5, N)
    assert sinfo["points"] == info["points"] and sinfo["kept_blocks"] == info["kept_blocks"]
    assert sinfo["edge_slope"] == info["edge_slope"]
    for head in range(0, N ** 3, 1 << 26):
        idx = torch.arange(head, min(head + (1 << 26), N ** 3), device=df.device)
        assert _same_bits(band.values(idx), df[idx]), head
    i0, n0 = grid.near_surface_cells(c5, N, df)
    i1, n1 = grid.near_surface_cells_sparse(c5, band)
    assert torch.equal(i0, i1) and _same_bits(n0, n1)
    report("sparse_store", N=N, bricks=sinfo["bricks"], bytes=sinfo["bytes"], dense_bytes=4 * N ** 3)


@pytest.mark.parametrize("N", [128, 256, 512, 1024])
def test_mesh_sparse_equals_band_mesh(c5, N):
    from neuraludf_b200 import mesh
    v0, f0 = mesh.udf_mesh_band(c5, N)
    v1, f1 = mesh.udf_mesh_sparse(c5, N)
    assert f0.shape[0] > 1000
    assert _same_bits(v0, v1) and torch.equal(f0, f1)


@pytest.mark.parametrize("strides", [None, [6, 3, 1], [16, 4, 1]], ids=["default", "6-3-1", "16-4-1"])
@pytest.mark.parametrize("name", sorted(C.CASES))
def test_mesh_sparse_equals_band_mesh_on_fields(name, strides):
    from neuraludf_b200 import mesh
    field = _Analytic(name, _dev())
    for N in (64, 65, 131):
        v0, f0 = mesh.udf_mesh_band(field, N, strides=strides)
        v1, f1 = mesh.udf_mesh_sparse(field, N, strides=strides)
        assert f0.shape[0] > 100
        assert _same_bits(v0, v1) and torch.equal(f0, f1), (name, N)


def test_mesh_post_sparse_equals_band(c5):
    from neuraludf_b200 import mesh
    v0, f0, i0 = mesh.udf_mesh_post(c5, 512)
    v1, f1, i1 = mesh.udf_mesh_post(c5, 512, sparse=True)
    assert f0.shape[0] > 1000
    assert torch.equal(v0, v1) and torch.equal(f0, f1) and i0["mc"] == i1["mc"] and i0["filtered"] == i1["filtered"]
    with pytest.raises(ValueError):
        mesh.udf_mesh_post(c5, 64, dense=True, sparse=True)


def _workspace(c5, max_batch):
    """the value chain's batch workspace: the peak a max_batch udf_values batch and a max_batch / 2 gradient batch (the
    sizes udf_mesh_sparse evaluates) add on their own"""
    g = torch.Generator(device="cpu").manual_seed(0)
    ws = 0
    for fn, n in ((lambda x: c5.udf_values(x), max_batch), (lambda x: c5.gradient(x), max_batch // 2)):
        pts = (torch.rand(n, 3, generator=g) * 2 - 1).cuda()
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        with torch.no_grad():
            out = fn(pts)
        torch.cuda.synchronize()
        ws = max(ws, torch.cuda.max_memory_allocated() - base)
        del pts, out
    return ws


def _peak(fn):
    torch.cuda.empty_cache()
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def _raw_sparse_mesh(c5, N):
    from neuraludf_b200 import grid, mesh
    band, info = grid.udf_band_sparse(c5, N)
    idx, nrm = grid.near_surface_cells_sparse(c5, band)
    v, f, mc = mesh.marching_cubes_sparse(band, nrm, idx)
    return v, f, mc, info


def _vertex_ids(mc, N, planes, p0):
    """global ids of the face vertices of an MC of x-planes [p0, p0 + planes): lattice edge 3 * corner + axis, or
    -(1 + 4 * cell + loop) for a loop centre; and the lowest x-plane each vertex touches"""
    lo = p0 * N * N
    keys, active = mc["face_keys"], mc["active"] + lo
    centre0 = 3 * planes * N * N
    cen = keys >= centre0
    c = torch.where(cen, keys - centre0, torch.zeros_like(keys))
    ids = torch.where(cen, -(1 + 4 * active[c >> 2] + (c & 3)), keys + 3 * lo)
    x = torch.where(cen, active[c >> 2], keys // 3 + lo) // (N * N)
    return ids, x


def _triangles(mc, N, planes, p0, x_lo, x_hi):
    """the faces all of whose vertices lie on x-planes [x_lo, x_hi], as sorted rows of their three sorted vertex ids:
    an unoriented multiset"""
    ids, x = _vertex_ids(mc, N, planes, p0)
    keep = ((x >= x_lo) & (x <= x_hi)).all(1)
    t = torch.sort(ids[keep], dim=1).values.cpu().numpy()
    return t[np.lexsort(t.T[::-1])]


def _edge_vertices(v, mc, N, planes, p0):
    """(global lattice-edge key, fp32 vertex) of the MC's lattice-edge vertices, x in global lattice units"""
    k = mc["vertex_keys"]
    e = k < 3 * planes * N * N
    return k[e] + 3 * p0 * N * N, v[e].double() + torch.tensor([p0, 0.0, 0.0], dtype=torch.float64, device=v.device)


def _is_oriented_two_manifold(f, V):
    e = torch.cat([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    ks, _ = torch.sort(e[:, 0] * V + e[:, 1])
    _, uses = torch.unique(torch.minimum(e[:, 0], e[:, 1]) * V + torch.maximum(e[:, 0], e[:, 1]), return_counts=True)
    return bool((ks[1:] != ks[:-1]).all()) and int(uses.max()) == 2


def test_2048_against_a_dense_slab_and_memory(c5):
    """udf_mesh_sparse's raw MC at 2048^3 against the dense udf_mesh MC of a 64-plane x-slab through the surface: the same
    triangles among those whose vertices lie two planes inside the slab (fp32 vertex bits, unoriented); the raw mesh is an
    oriented two-manifold; the peak memory beside the value chain's batch workspace is below N^3 bytes, at 1024 too."""
    from neuraludf_b200 import mesh
    ws = _workspace(c5, 1 << 21)
    peaks = {}
    for N in (1024, 2048):
        (v, f, mc, info), peak = _peak(lambda: _raw_sparse_mesh(c5, N))
        peaks[N] = peak
        report("sparse_memory", N=N, peak_gb=peak / 1e9, workspace_gb=ws / 1e9, rest_gb=(peak - ws) / 1e9,
               bound_gb=N ** 3 / 1e9, faces=int(f.shape[0]), bricks=info["bricks"], bytes=info["bytes"],
               points=info["points"])
        print("N=%d: peak %.3f GB, workspace %.3f GB, rest %.3f GB (bound %.3f), %d faces, %s" % (
            N, peak / 1e9, ws / 1e9, (peak - ws) / 1e9, N ** 3 / 1e9, f.shape[0], info["bytes"]))
        if N == 2048:
            break
        del v, f, mc
    assert f.shape[0] > 4_000_000
    assert _is_oriented_two_manifold(f, v.shape[0])
    # the slab: 64 x-planes around the plane holding the most vertices, meshed densely (udf_mesh's stages)
    N, planes = 2048, 64
    x = v[:, 0].floor().to(torch.int64)
    centre = int(torch.bincount(x, minlength=N).argmax())
    p0 = min(max(centre - planes // 2, 0), N - planes)
    from neuraludf_b200 import grid
    df = grid.udf_grid(c5, N, lo=p0 * N * N, hi=(p0 + planes) * N * N)
    idx, nrm = grid.near_surface_cells(c5, N, df, lo=p0 * N * N)
    vs, fs, mcs = mesh.marching_cubes_index(df, (planes, N, N), nrm, idx - p0 * N * N)
    del df, idx, nrm
    a = _triangles(mc, N, N, 0, p0 + 2, p0 + planes - 3)
    b = _triangles(mcs, N, planes, p0, p0 + 2, p0 + planes - 3)
    assert len(a) > 10000
    assert np.array_equal(a, b)
    # the lattice-edge vertices both hold: y, z bit for bit; x within the rounding of c + t at the slab's own index c
    ka, va = _edge_vertices(v, mc, N, N, 0)
    kb, vb = _edge_vertices(vs, mcs, N, planes, p0)
    inner = (kb // 3 // (N * N) >= p0 + 2) & (kb // 3 // (N * N) <= p0 + planes - 3)
    kb, vb = kb[inner], vb[inner]
    pos = torch.searchsorted(ka, kb)
    assert bool((ka[pos] == kb).all())
    assert torch.equal(va[pos][:, 1:], vb[:, 1:])
    assert float((va[pos][:, 0] - vb[:, 0]).abs().max()) <= 2.5e-4
    for N, peak in peaks.items():
        assert peak - ws < N ** 3, (N, peak, ws)


def test_deterministic_and_cli_2048(c5, tmp_path):
    from neuraludf_b200 import mesh
    from neuraludf_b200.evaluate import read_ply, write_ply_points
    v0, f0 = mesh.udf_mesh_sparse(c5, 512)
    v1, f1 = mesh.udf_mesh_sparse(c5, 512)
    assert _same_bits(v0, v1) and torch.equal(f0, f1)
    ckpt, out, gt = (os.path.join(str(tmp_path), n) for n in ("ckpt_000100.pth", "mesh.ply", "gt.ply"))
    torch.save({"udf_network_fine": c5.state_dict(), "iter_step": 100}, ckpt)
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-m", "neuraludf_b200.mesh", "--ckpt", ckpt, "--resolution", "2048", "--sparse",
                        "--postprocess", "--dist_threshold_ratio", "5", "--out", out], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    v, f = read_ply(out)
    assert f.shape[0] > 4_000_000 and np.isfinite(v).all()
    write_ply_points(gt, v0.double().cpu().numpy())
    r = subprocess.run([sys.executable, "-m", "neuraludf_b200.evaluate", "deepfashion", "--data", out, "--gt", gt, "--log",
                        os.path.join(str(tmp_path), "eval.txt")], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    report("sparse_cli_2048", faces=int(f.shape[0]), eval=r.stdout.strip().splitlines()[-1:])

"""`get_mesh_udf_fast` on the device: a drop-in for the runner's extract_mesh.py (extract_mesh.py:169-354), served to the
unmodified runner as `extract_mesh` by `launch.install_shadow_modules` under NUDF_DEVICE_MESH=1.

The caller's `func` and `func_grad` are evaluated, never the network behind them: the lattice, the near-surface normals,
the MC, the vertex filter and the post-processing are mesh._mesh_post's (the stages of mesh.udf_mesh_post) on a
CallerField, and the gradient branch runs on csrc/mesh_grad.cu (restated in tests/proto/mesh_grad.py).  There is no N^3
host array and no cache across calls.

Deviations from the reference (DESIGN.md section 7):
  * `samples` is returned as None; passing a non-None `samples` back raises NotImplementedError (incremental
    re-evaluation is not served; with samples None the reference evaluates the whole lattice, as here);
  * the border gradients (extract_mesh.py:306-352) are not evaluated: for a finite udf at the border probes they add a
    signed zero, which leaves `new_verts` unchanged except that a coordinate -0.0 there may become +0.0 in the reference;
    for a udf of +inf there the reference writes NaN.  Their IndexError on a mesh without border edges is kept;
  * the vertex normals follow a restated rule (DESIGN.md section 1), not trimesh itself.
"""
import os

import torch
import torch.nn.functional as F

from neuraludf_b200 import _lib, mesh, mesh_post
from neuraludf_b200._lib import check, ptr

LATTICE_BATCH = 1 << 20         # get_udf_normals_grid_slow's max_batch


class CallerField:
    """The field get_mesh_udf_fast meshes, from the caller's callables: udf_values(points) = func(points) as fp32 [P];
    surface_normals(points) = -normalize(func_grad(points)[:, 0]) (extract_mesh.py:93), with autograd enabled and the points
    requiring grad, as the reference calls it."""

    def __init__(self, func, func_grad):
        self.func, self.func_grad = func, func_grad

    def udf_values(self, pts):
        return self.func(pts).detach().reshape(-1).float()

    def surface_normals(self, pts):
        x = pts.detach().clone().requires_grad_(True)
        with torch.enable_grad():
            g = self.func_grad(x)
        return -F.normalize(g.detach()[:, 0].float(), dim=1)


class UdfMesh:
    """The mesh object get_mesh_udf_fast returns: `vertices` fp64 [V,3] and `faces` int64 [F,3], NumPy -- what
    Runner.extract_udf_mesh reads of its trimesh.Trimesh."""

    def __init__(self, vertices, faces):
        self.vertices, self.faces = vertices, faces


def vertex_normals(verts64, faces):
    """fp32 [V,3] angle-weighted vertex normals of the fp64 mesh (trimesh.geometry.weighted_vertex_normals as DESIGN.md
    section 1 restates it): nudf_mg_vertex_normals over the incidences sorted by (vertex, corner, face)"""
    dev = verts64.device
    V, nf = verts64.shape[0], faces.shape[0]
    out = torch.empty(V, 3, device=dev)
    if V == 0:
        return out
    corner_major = faces.t().reshape(-1)                  # incidence e = corner * F + face
    inc = torch.sort(corner_major, stable=True).indices.contiguous()
    rowptr = torch.zeros(V + 1, dtype=torch.int64, device=dev)
    rowptr[1:] = torch.cumsum(torch.bincount(corner_major, minlength=V), 0)
    terms = torch.empty(9 * nf, dtype=torch.float64, device=dev)
    v = verts64.to(torch.float64).contiguous()
    f = faces.to(torch.int64).contiguous()
    check(_lib.lib().nudf_mg_vertex_normals(ptr(v), V, ptr(f), nf, ptr(rowptr), ptr(inc), ptr(terms), ptr(out),
                                            _lib.stream_ptr()), "nudf_mg_vertex_normals")
    return out


@torch.no_grad()
def refine(func, verts64, faces, eps, N):
    """the gradient branch without its border term (extract_mesh.py:271-304): (new_verts fp32 [V,3] on the device,
    next_indices int64 [7V] NumPy).  func is evaluated at the two probe sets, one call each."""
    L, st = _lib.lib(), _lib.stream_ptr()
    V = verts64.shape[0]
    v32 = verts64.float().contiguous()
    n = vertex_normals(verts64, faces)
    probes = torch.empty(2 * V, 3, device=v32.device)
    new_verts = torch.empty(V, 3, device=v32.device)
    nxt = torch.empty(7 * V, dtype=torch.int64, device=v32.device)
    if V == 0:
        return new_verts, nxt.cpu().numpy()
    check(L.nudf_mg_refine(ptr(v32), ptr(n), V, float(eps), None, None, int(N), ptr(probes), None, None, st), "nudf_mg_refine")
    s1 = func(probes[:V]).detach().reshape(-1).float().contiguous()
    s2 = func(probes[V:]).detach().reshape(-1).float().contiguous()
    check(L.nudf_mg_refine(ptr(v32), ptr(n), V, float(eps), ptr(s1), ptr(s2), int(N), None, ptr(new_verts), ptr(nxt), st),
          "nudf_mg_refine")
    return new_verts, nxt.cpu().numpy()


def get_mesh_udf_fast(func, func_grad, samples=None, indices=None, N_MC=128, gradient=True, eps=0.1, border_gradients=False,
                      smooth_borders=False, dist_threshold_ratio=1., info=None):
    """The reference's get_mesh_udf_fast with its signature and defaults, on the device.

    The N_MC^3 lattice on [-1,1]^3 holds func's values (batches of 2^20 points), negative values set to 0; the normals are
    -normalize(func_grad(x)[:, 0]) where the value is below 2 voxels.  The lattice is dense, or narrow-band (grid.udf_band)
    with NUDF_BAND_MESH=1 in the environment: the same mesh when func is 2-Lipschitz and gives a point the same bits in any
    batch (udf_band warns when the lattice shows a steeper slope); with NUDF_BAND_MESH=sparse that band is held
    block-sparse (grid.udf_band_sparse, its values clamped as the dense lattice's are): the band mesh, with no N^3 array.  Then the MC, the vertex filter (func at every vertex in
    one call) and mesh_post.postprocess(smooth_borders).

    Raises RuntimeError when the MC finds no surface (the reference's MC does), and IndexError when the post-processed mesh
    has no border edge (an empty mesh has none) and smooth_borders or (gradient and border_gradients) holds, where the
    reference's smoothing or border gradients raise.  Returns (verts fp32 cuda [V,3], faces int64 cuda [F,3], mesh) with
    gradient False; else (new_verts fp32 cuda [V,3], faces, mesh, None, next_indices np.int64 [7V]).  `mesh` is a UdfMesh.
    `info`, when given a dict, receives mesh._mesh_post's info and the gradient branch's CUDA-event milliseconds under
    stage_ms["gradient"]."""
    if samples is not None:
        raise NotImplementedError("get_mesh_udf_fast: re-evaluation from a passed-back `samples` is not served on the device; "
                                  "pass samples=None for a full evaluation")
    N = int(N_MC)
    lattice = {"1": "band", "sparse": "sparse"}.get(os.environ.get("NUDF_BAND_MESH"), "dense")
    with torch.no_grad():
        v64, f, minfo = mesh._mesh_post(CallerField(func, func_grad), N, lattice, dist_threshold_ratio, smooth_borders,
                                        max_batch=LATTICE_BATCH)
    if info is not None:
        info.update(minfo)
    if minfo["mc"][1] == 0:
        raise RuntimeError('No surface found at the given iso value.')
    if (smooth_borders or (gradient and border_gradients)) and not mesh_post.has_border(v64, f):
        raise IndexError("get_mesh_udf_fast: the mesh has no border edge to %s"
                         % ("smooth" if smooth_borders else "take border gradients from"))
    m = UdfMesh(v64.cpu().numpy(), f.cpu().numpy())
    if not gradient:
        return v64.float(), f, m
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    new_verts, next_indices = refine(func, v64, f, eps, N)
    ev[1].record()
    if info is not None:
        torch.cuda.synchronize(v64.device)
        info["stage_ms"]["gradient"] = ev[0].elapsed_time(ev[1])
    return new_verts, f, m, None, next_indices

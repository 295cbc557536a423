"""MeshUDF marching cubes on the device: the last stage of a run, UDF -> triangle mesh.

`udf_mesh` is the device-resident pipeline (grid.udf_grid -> grid.near_surface_cells -> CUDA MC -> the reference's vertex
filter, extract_mesh.py:205-214); `udf_marching_cubes` is the MC alone; `udf_mc_lewiner` is a NumPy-in / NumPy-out drop-in
for the reference's `custom_mc._marching_cubes_lewiner.udf_mc_lewiner`, served to the unmodified runner by
`launch.install_shadow_modules` when the reference's Cython build cannot be imported.  The kernels are in
csrc/mesh_udf.cu (stages and deviations documented there); tests/proto/udf_mc.py is their NumPy restatement.
"""
import ctypes

import numpy as np
import torch

from neuraludf_b200 import _lib
from neuraludf_b200._lib import check, ptr


def thresholds(n2):
    """the reference's active-cell thresholds (.pyx:1157-1158): fp32 of 1.05 / 1.74 voxels, voxel = 2 / (n2 - 1)"""
    voxel = 2.0 / (n2 - 1)
    return float(np.float32(1.05 * voxel)), float(np.float32(1.74 * voxel))


@torch.no_grad()
def marching_cubes_index(df, dims, normals, idx=None):
    """(verts [V,3] fp32 in lattice-index units, faces [F,3] int64, info) on df's device.

    df: fp32 lattice of shape `dims` (any layout that flattens to it); normals: dense [prod(dims), 3] (idx None) or the rows
    of the sorted flat indices `idx`.  info: `active` (sorted active cells), `face_keys` [F,3] (vertex keys: lattice edges,
    then loop centres), `mask` (final per-cell pseudo-sign masks), `polarity_rounds` / `polarity_jumps` (union-find
    hooking rounds / pointer-jumping passes).  Faces are wound towards the positive pseudo-side (the reference's 'descent' winding)."""
    L = _lib.lib()
    st = _lib.stream_ptr()
    n0, n1, n2 = (int(d) for d in dims)
    dev = df.device
    if dev.type != "cuda":
        raise ValueError("marching cubes runs on a CUDA device (df is on %s)" % dev)
    df = df.reshape(-1).float().contiguous()
    if df.numel() != n0 * n1 * n2:
        raise ValueError("df has %d values, dims %s need %d" % (df.numel(), (n0, n1, n2), n0 * n1 * n2))
    normals = normals.reshape(-1, 3).float().contiguous()
    if idx is not None:
        idx = idx.reshape(-1).to(torch.int64).contiguous()
        if normals.shape[0] != idx.numel():
            raise ValueError("normals must have one row per idx entry")
    elif normals.shape[0] != df.numel():
        raise ValueError("dense normals must have one row per lattice point")
    avg_t, max_t = thresholds(n2)
    n_cand = n0 * n1 * n2 if idx is None else idx.numel()
    flags = torch.empty(n_cand, dtype=torch.uint8, device=dev)
    check(L.nudf_mc_active(ptr(df), n0, n1, n2, ptr(idx), n_cand, avg_t, max_t, ptr(flags), st), "nudf_mc_active")
    sel = torch.nonzero(flags).reshape(-1)
    cells = (sel if idx is None else idx[sel]).contiguous()
    n = cells.numel()
    empty = (torch.zeros(0, 3, device=dev), torch.zeros(0, 3, dtype=torch.int64, device=dev))
    info = {"active": cells}
    if n == 0:
        info.update(face_keys=empty[1], mask=torch.zeros(0, dtype=torch.uint8, device=dev))
        return empty[0], empty[1], info
    mask0 = torch.empty(n, dtype=torch.uint8, device=dev)
    check(L.nudf_mc_cell_signs(ptr(df), n0, n1, n2, ptr(cells), n, ptr(idx), 0 if idx is None else idx.numel(), ptr(normals),
                               ptr(mask0), st), "nudf_mc_cell_signs")
    links = torch.empty(n * 3, dtype=torch.int64, device=dev)
    check(L.nudf_mc_links(ptr(df), n0, n1, n2, ptr(cells), n, ptr(mask0), ptr(links), st), "nudf_mc_links")
    parent = torch.empty(n, dtype=torch.int64, device=dev)
    hook = torch.empty(n, dtype=torch.int64, device=dev)
    flag = torch.empty(1, dtype=torch.int32, device=dev)
    mask = torch.empty_like(mask0)
    stats = (ctypes.c_int32 * 2)()
    check(L.nudf_mc_polarity(ptr(links), n, ptr(mask0), ptr(parent), ptr(hook), ptr(flag), ptr(mask), stats, st),
          "nudf_mc_polarity")
    info["polarity_rounds"], info["polarity_jumps"] = int(stats[0]), int(stats[1])
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    check(L.nudf_mc_count(ptr(df), n0, n1, n2, ptr(cells), n, ptr(mask), ptr(counts), st), "nudf_mc_count")
    csum = torch.cumsum(counts, 0, dtype=torch.int64)
    n_faces = int(csum[-1])
    offsets = (csum - counts).contiguous()
    keys = torch.empty(3 * n_faces, dtype=torch.int64, device=dev)
    check(L.nudf_mc_emit(ptr(df), n0, n1, n2, ptr(cells), n, ptr(mask), ptr(offsets), ptr(keys), st), "nudf_mc_emit")
    info.update(face_keys=keys.reshape(-1, 3), mask=mask)
    if n_faces == 0:
        return empty[0], empty[1], info
    ukeys, inv = torch.unique(keys, sorted=True, return_inverse=True)
    ukeys = ukeys.contiguous()
    verts = torch.empty(ukeys.numel(), 3, device=dev)
    check(L.nudf_mc_vertices(ptr(df), n0, n1, n2, ptr(cells), n, ptr(mask), ptr(ukeys), ukeys.numel(), ptr(verts), st),
          "nudf_mc_vertices")
    info["vertex_keys"] = ukeys
    return verts, inv.reshape(-1, 3).to(torch.int64), info


def udf_marching_cubes(df, N, idx, normals):
    """MeshUDF marching cubes of the N^3 lattice on [-1,1]^3 (grid.py's order): device verts [V,3] in world coordinates and
    faces [F,3] int64.  idx / normals: grid.near_surface_cells (sorted flat indices, unit vectors towards the surface), or
    idx=None with dense normals [N^3,3]."""
    verts, faces, _ = marching_cubes_index(df, (N, N, N), normals, idx)
    voxel = 2.0 / (N - 1)
    return verts * voxel - 1.0, faces


def _compact(verts, faces):
    used = torch.zeros(verts.shape[0], dtype=torch.bool, device=verts.device)
    used[faces.reshape(-1)] = True
    remap = torch.cumsum(used.to(torch.int64), 0) - 1
    return verts[used], remap[faces]


@torch.no_grad()
def udf_mesh(udf_network, N, dist_threshold_ratio=1.0, lo=0, hi=None, max_batch=1 << 21):
    """UDF network -> filtered mesh, all on the device: (verts [V,3] world, faces [F,3] int64).

    The lattice is N^3 on [-1,1]^3; [lo, hi) selects a slab of whole x-planes (multiples of N^2; default all), so that ranks
    can mesh disjoint slabs -- adjacent slabs must share one plane for the cells between them to be meshed.  Faces with a
    vertex whose udf is at or above voxel * dist_threshold_ratio are dropped (extract_mesh.py:205-214) and unused vertices
    removed."""
    from neuraludf_b200 import grid
    hi = N ** 3 if hi is None else hi
    if lo % (N * N) or hi % (N * N) or not 0 <= lo < hi <= N ** 3:
        raise ValueError("lo / hi must select whole x-planes of the N^3 lattice")
    planes = (hi - lo) // (N * N)
    voxel = 2.0 / (N - 1)
    df = grid.udf_grid(udf_network, N, max_batch=max_batch, lo=lo, hi=hi)
    idx, normals = grid.near_surface_cells(udf_network, N, df, max_batch=max(max_batch // 2, 1), lo=lo)
    verts, faces, _ = marching_cubes_index(df, (planes, N, N), normals, idx - lo)
    verts = verts * voxel - 1.0
    verts[:, 0] += (lo // (N * N)) * voxel
    if faces.shape[0] == 0:
        return verts, faces
    vd = udf_network.udf_values(verts).reshape(-1)
    keep = vd[faces].max(dim=1).values < voxel * dist_threshold_ratio
    return _compact(verts, faces[keep])


def udf_mc_lewiner(volume, grads, spacing=(1., 1., 1.), gradient_direction='descent', step_size=1, allow_degenerate=True,
                   use_classic=False, mask=None):
    """Drop-in for custom_mc._marching_cubes_lewiner.udf_mc_lewiner on the CUDA kernels.

    volume [n0,n1,n2] udf, grads [n0,n1,n2,3] unit vectors towards the surface (NumPy).  Returns NumPy (vertices [V,3] in
    array-index order times `spacing`, faces [F,3] int32 wound for `gradient_direction`, normals [V,3] fp32: the normalised
    trilinearly interpolated grads, values [V] fp32: the trilinearly interpolated udf).  Same errors as the reference;
    `step_size` != 1 and `mask` are not supported.  `allow_degenerate` and `use_classic` are accepted and ignored
    (degenerate triangles are kept, as with the reference's default)."""
    if not isinstance(volume, np.ndarray) or volume.ndim != 3:
        raise ValueError('Input volume should be a 3D numpy array.')
    if volume.shape[0] < 2 or volume.shape[1] < 2 or volume.shape[2] < 2:
        raise ValueError("Input array must be at least 2x2x2.")
    volume = np.ascontiguousarray(volume, np.float32)
    if len(spacing) != 3:
        raise ValueError("`spacing` must consist of three floats.")
    step_size = int(step_size)
    if step_size < 1:
        raise ValueError('step_size must be at least one.')
    if step_size != 1:
        raise NotImplementedError("udf_mc_lewiner: only step_size=1 is implemented on the device")
    if mask is not None:
        raise NotImplementedError("udf_mc_lewiner: `mask` is not implemented on the device")
    if gradient_direction not in ('descent', 'ascent'):
        raise ValueError("Incorrect input %s in `gradient_direction`, see docstring." % (gradient_direction))
    grads = np.ascontiguousarray(grads, np.float32)
    if grads.shape != volume.shape + (3,):
        raise ValueError("grads must have shape volume.shape + (3,)")
    dev = torch.device("cuda", torch.cuda.current_device())
    df = torch.from_numpy(volume).to(dev)
    g = torch.from_numpy(grads).to(dev).reshape(-1, 3)
    verts, faces, info = marching_cubes_index(df, volume.shape, g, None)
    if faces.shape[0] == 0:
        raise RuntimeError('No surface found at the given iso value.')
    # normals and values: trilinear interpolation of the corner grads / udf in the vertex's cell (exact along a lattice
    # edge; loop-centre vertices lie inside their cell)
    n0, n1, n2 = volume.shape
    hi = torch.tensor([n0 - 2, n1 - 2, n2 - 2], device=dev)
    base = torch.minimum(verts.floor().to(torch.int64).clamp(min=0), hi)
    w = verts - base
    flat = df.reshape(-1)
    nrm = torch.zeros_like(verts)
    values = torch.zeros(verts.shape[0], device=dev)
    for c in range(8):
        o = [(c >> 2) & 1, (c >> 1) & 1, c & 1]
        wc = torch.ones(verts.shape[0], device=dev)
        for k in range(3):
            wc = wc * (w[:, k] if o[k] else 1 - w[:, k])
        gi = (base[:, 0] + o[0]) * n1 * n2 + (base[:, 1] + o[1]) * n2 + base[:, 2] + o[2]
        nrm += wc[:, None] * g[gi]
        values += wc * flat[gi]
    nrm = torch.nn.functional.normalize(nrm, dim=1)
    if gradient_direction == 'ascent':
        faces = faces.flip(1)
    vertices = verts.cpu().numpy()
    if not np.array_equal(spacing, (1, 1, 1)):
        vertices = vertices * np.r_[spacing]
    return vertices, faces.to(torch.int32).cpu().numpy(), nrm.cpu().numpy(), values.cpu().numpy()

"""MeshUDF marching cubes on the device: the last stage of a run, UDF -> triangle mesh.

`udf_mesh` is the device-resident pipeline (grid.udf_grid -> grid.near_surface_cells -> CUDA MC -> the reference's vertex
filter, extract_mesh.py:205-214); `udf_mesh_band` is the same with the lattice evaluated narrow-band (grid.udf_band);
`udf_mesh_post` adds the runner's post-processing (mesh_post.py) and returns the mesh `Runner.extract_udf_mesh` exports;
`python -m neuraludf_b200.mesh` meshes a runner checkpoint to PLY; `udf_marching_cubes` is the MC alone; `udf_mc_lewiner` is a NumPy-in / NumPy-out drop-in
for the reference's `custom_mc._marching_cubes_lewiner.udf_mc_lewiner`, served to the unmodified runner by
`launch.install_shadow_modules` when the reference's Cython build cannot be imported.  The kernels are in
csrc/mesh_udf.cu (stages and deviations documented there); tests/proto/udf_mc.py is their NumPy restatement.
`iso_marching_cubes_index` / `iso_marching_cubes` are threshold marching cubes on the same kernels (the runner's
validate_mesh without PyMCubes; `python -m neuraludf_b200.mesh --threshold T`), restated in tests/proto/iso_mc.py;
`iso_mesh_band` is the same with the lattice evaluated narrow-band (grid.iso_band; `--threshold T --band`), and
`iso_mesh_sparse` the same again with the band held block-sparse (grid.iso_band_sparse; `--threshold T --band --sparse`).
`udf_mesh_sparse` is `udf_mesh_band` on the block-sparse band (grid.udf_band_sparse, `marching_cubes_sparse`): the same
mesh with no N^3 array, for lattices up to 2048^3 (`--sparse`).
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
    lat = _lib.Lattice(n0, n1, n2, df.data_ptr(), None)
    return _mc_stages(ctypes.byref(lat), n2, n0 * n1 * n2 if idx is None else idx.numel(), idx, normals, dev)


def _mc_stages(lat, n2, n_cand, idx, normals, dev):
    """the MeshUDF MC driver of marching_cubes_index and marching_cubes_sparse on the lattice descriptor `lat` (dense df or
    brick store); idx the sorted candidate indices (None: every cell) and normals their rows"""
    L = _lib.lib()
    st = _lib.stream_ptr()
    n_idx = 0 if idx is None else idx.numel()
    avg_t, max_t = thresholds(n2)
    flags = torch.empty(n_cand, dtype=torch.uint8, device=dev)
    check(L.nudf_mc_active(lat, ptr(idx), n_cand, avg_t, max_t, ptr(flags), st), "nudf_mc_active")
    sel = torch.nonzero(flags).reshape(-1)
    cells = (sel if idx is None else idx[sel]).contiguous()
    n = cells.numel()
    empty = (torch.zeros(0, 3, device=dev), torch.zeros(0, 3, dtype=torch.int64, device=dev))
    info = {"active": cells}
    if n == 0:
        info.update(face_keys=empty[1], mask=torch.zeros(0, dtype=torch.uint8, device=dev))
        return empty[0], empty[1], info
    mask0 = torch.empty(n, dtype=torch.uint8, device=dev)
    check(L.nudf_mc_cell_signs(lat, ptr(cells), n, ptr(idx), n_idx, ptr(normals), ptr(mask0), st), "nudf_mc_cell_signs")
    links = torch.empty(n * 3, dtype=torch.int64, device=dev)
    check(L.nudf_mc_links(lat, ptr(cells), n, ptr(mask0), ptr(links), st), "nudf_mc_links")
    parent = torch.empty(n, dtype=torch.int64, device=dev)
    hook = torch.empty(n, dtype=torch.int64, device=dev)
    flag = torch.empty(1, dtype=torch.int32, device=dev)
    mask = torch.empty_like(mask0)
    stats = (ctypes.c_int32 * 2)()
    check(L.nudf_mc_polarity(ptr(links), n, ptr(mask0), ptr(parent), ptr(hook), ptr(flag), ptr(mask), stats, st),
          "nudf_mc_polarity")
    info["polarity_rounds"], info["polarity_jumps"] = int(stats[0]), int(stats[1])
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    check(L.nudf_mc_count(lat, ptr(cells), n, ptr(mask), ptr(counts), st), "nudf_mc_count")
    csum = torch.cumsum(counts, 0, dtype=torch.int64)
    n_faces = int(csum[-1])
    offsets = (csum - counts).contiguous()
    keys = torch.empty(3 * n_faces, dtype=torch.int64, device=dev)
    check(L.nudf_mc_emit(lat, ptr(cells), n, ptr(mask), ptr(offsets), ptr(keys), st), "nudf_mc_emit")
    info.update(face_keys=keys.reshape(-1, 3), mask=mask)
    if n_faces == 0:
        return empty[0], empty[1], info
    ukeys, inv = torch.unique(keys, sorted=True, return_inverse=True)
    ukeys = ukeys.contiguous()
    verts = torch.empty(ukeys.numel(), 3, device=dev)
    check(L.nudf_mc_vertices(lat, ptr(cells), n, ptr(mask), ptr(ukeys), ukeys.numel(), ptr(verts), st), "nudf_mc_vertices")
    info["vertex_keys"] = ukeys
    return verts, inv.reshape(-1, 3).to(torch.int64), info


@torch.no_grad()
def marching_cubes_sparse(band, normals, idx):
    """marching_cubes_index on the N^3 lattice of a grid.SparseBand (every df read through the brick store): the same
    (verts [V,3] fp32 in lattice-index units, faces [F,3] int64, info).  idx / normals: the sorted flat candidate indices
    and their rows (grid.near_surface_cells_sparse); there is no dense form."""
    idx = idx.reshape(-1).to(torch.int64).contiguous()
    normals = normals.reshape(-1, 3).float().contiguous()
    if normals.shape[0] != idx.numel():
        raise ValueError("normals must have one row per idx entry")
    return _mc_stages(band.lattice(), band.N, idx.numel(), idx, normals, band.device)


def _iso_level(level):
    """the level as the kernels compare it: rounded to fp32 once (the lattice is fp32); non-finite -> ValueError"""
    lv = float(level)
    if not np.isfinite(lv) or not np.isfinite(np.float32(lv)):
        raise ValueError("level must be finite (got %r)" % (level,))
    return float(np.float32(lv))


@torch.no_grad()
def iso_marching_cubes_index(df, dims, level):
    """Threshold marching cubes of the fp32 lattice df (shape `dims`, on a CUDA device) at `level`, all on the device:
    (verts [V,3] fp64 in lattice-index units, column k along array axis k; faces [F,3] int64; info).

    The MeshUDF construction (csrc/mesh_udf.cu) on v = fl32(f - fl32(level)): a cell is active when some corner has v > 0,
    some v <= 0 and none is NaN; ambiguous faces by the asymptotic decider; each loop triangulated with no chord in a cube
    face, so every interior edge has exactly two faces.  Edge points sit at t = v_a / (v_a - v_b) (fp64); loop centres at
    the mean of their loop's edge points.  Vertices are numbered by ascending key (lattice edges 3 * corner + axis, then loop
    centres).  Faces are wound so that their normals point towards decreasing values (from the > level side into the
    <= level side: skimage's 'descent').  info: `active` (sorted active cells), `face_keys` [F,3], `vertex_keys`."""
    L = _lib.lib()
    st = _lib.stream_ptr()
    n0, n1, n2 = (int(d) for d in dims)
    if min(n0, n1, n2) < 2:
        raise ValueError("lattice dimensions must be at least 2 (got %s)" % ((n0, n1, n2),))
    level = _iso_level(level)
    dev = df.device
    if dev.type != "cuda":
        raise ValueError("marching cubes runs on a CUDA device (df is on %s)" % dev)
    df = df.reshape(-1)
    if df.dtype != torch.float32:
        raise ValueError("df must be float32 (got %s)" % df.dtype)
    df = df.contiguous()
    if df.numel() != n0 * n1 * n2:
        raise ValueError("df has %d values, dims %s need %d" % (df.numel(), (n0, n1, n2), n0 * n1 * n2))
    flags = torch.empty(df.numel(), dtype=torch.uint8, device=dev)
    check(L.nudf_iso_active(ptr(df), n0, n1, n2, level, ptr(flags), st), "nudf_iso_active")
    cells = torch.nonzero(flags).reshape(-1).contiguous()
    del flags
    lat = _lib.Lattice(n0, n1, n2, df.data_ptr(), None)
    return _iso_stages(ctypes.byref(lat), cells, level, dev)


def _iso_stages(lat, cells, level, dev):
    """the threshold MC stages after the active cells (sorted `cells`) on the lattice descriptor `lat` (a flat array or a
    brick store): iso_marching_cubes_index's returns"""
    L = _lib.lib()
    st = _lib.stream_ptr()
    n = cells.numel()
    empty = (torch.zeros(0, 3, dtype=torch.float64, device=dev), torch.zeros(0, 3, dtype=torch.int64, device=dev))
    info = {"active": cells, "face_keys": empty[1], "vertex_keys": torch.zeros(0, dtype=torch.int64, device=dev)}
    if n == 0:
        return empty[0], empty[1], info
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    check(L.nudf_iso_lat_count(lat, level, ptr(cells), n, ptr(counts), st), "nudf_iso_lat_count")
    csum = torch.cumsum(counts, 0, dtype=torch.int64)
    n_faces = int(csum[-1])
    offsets = (csum - counts).contiguous()
    del counts, csum
    keys = torch.empty(3 * n_faces, dtype=torch.int64, device=dev)
    check(L.nudf_iso_lat_emit(lat, level, ptr(cells), n, ptr(offsets), ptr(keys), st), "nudf_iso_lat_emit")
    del offsets
    info["face_keys"] = keys.reshape(-1, 3)
    if n_faces == 0:
        return empty[0], empty[1], info
    ukeys, inv = torch.unique(keys, sorted=True, return_inverse=True)
    ukeys = ukeys.contiguous()
    verts = torch.empty(ukeys.numel(), 3, dtype=torch.float64, device=dev)
    check(L.nudf_iso_lat_vertices(lat, level, ptr(cells), n, ptr(ukeys), ukeys.numel(), ptr(verts), st),
          "nudf_iso_lat_vertices")
    info["vertex_keys"] = ukeys
    return verts, inv.reshape(-1, 3).to(torch.int64), info


def _iso_cells(lat, n_positions, level, dev):
    """sorted active cells of the lattice descriptor `lat` at the fp32 `level` from its n_positions storage positions
    (nudf_iso_lat_cells_*: no scan of every cell)"""
    L = _lib.lib()
    st = _lib.stream_ptr()
    n_seg = -(-n_positions // _lib.ISO_SEG)
    counts = torch.empty(n_seg, dtype=torch.int32, device=dev)
    check(L.nudf_iso_lat_cells_count(lat, level, n_seg, ptr(counts), st), "nudf_iso_lat_cells_count")
    csum = torch.cumsum(counts, 0, dtype=torch.int64)
    total = int(csum[-1]) if n_seg else 0
    offsets = (csum - counts).contiguous()
    del counts, csum
    cells = torch.empty(total, dtype=torch.int64, device=dev)
    if total:
        check(L.nudf_iso_lat_cells_emit(lat, level, n_seg, ptr(offsets), ptr(cells), st), "nudf_iso_lat_cells_emit")
    del offsets
    return torch.sort(cells).values


@torch.no_grad()
def iso_active_cells(lattice, level, dims=None):
    """The sorted active cells of threshold meshing at `level` (rounded to fp32), found from the lattice's stored points
    with no scan of every cell: a grid.SparseBand, or an fp32 CUDA array of shape `dims`.  They equal
    iso_marching_cubes_index's info["active"] (nonzero of nudf_iso_active) of the same values, for any field."""
    level = _iso_level(level)
    if isinstance(lattice, torch.Tensor):
        n0, n1, n2 = (int(d) for d in dims)
        df = lattice.reshape(-1)
        if df.dtype != torch.float32 or df.device.type != "cuda" or df.numel() != n0 * n1 * n2:
            raise ValueError("df must be a float32 CUDA array of %d values" % (n0 * n1 * n2))
        df = df.contiguous()
        lat = _lib.Lattice(n0, n1, n2, df.data_ptr(), None)
        return _iso_cells(ctypes.byref(lat), df.numel(), level, df.device)
    return _iso_cells(lattice.lattice(), lattice.mc ** 3 + lattice.n_bricks * _lib.BRICK ** 3, level, lattice.device)


@torch.no_grad()
def iso_marching_cubes_sparse(band, level):
    """iso_marching_cubes_index on the R^3 lattice of a grid.SparseBand (grid.iso_band_sparse), every value read through
    the brick store: the same (fp64 verts [V,3] in lattice-index units, int64 faces [F,3], info) as on the array the store
    reads as, with no array of R^3 elements.  The active cells come from the stored points (iso_active_cells)."""
    level = _iso_level(level)
    cells = iso_active_cells(band, level)
    return _iso_stages(band.lattice(), cells, level, band.device)


@torch.no_grad()
def iso_mesh_band(query, bound_min, bound_max, resolution, level, lipschitz=2.0, strides=None, max_batch=1 << 21,
                  device=None):
    """Threshold marching cubes of extract_geometry's lattice (R = `resolution` points per axis on the box, torch.linspace
    coordinates) at `level`, the lattice evaluated narrow-band (grid.iso_band): iso_marching_cubes_index's (fp64 verts [V,3]
    in lattice-index units, int64 faces [F,3], info), with grid.iso_band's info under info["band"].

    Exact when `query` is `lipschitz`-Lipschitz at the lattice points and gives a point the same bits in any batch:
    iso_band's df then equals the dense lattice wherever that is below level + L D (D: the largest cell diagonal) and every
    point left out is above the level, so a cell with a culled corner is inactive as its dense corners make it, and the
    later stages read df only at the corners of active cells.  grid.iso_band warns when the lattice shows a slope above
    `lipschitz`."""
    from neuraludf_b200 import grid
    R = int(resolution)
    df, binfo = grid.iso_band(query, bound_min, bound_max, R, level, lipschitz=lipschitz, strides=strides,
                              max_batch=max_batch, device=device)
    verts, faces, info = iso_marching_cubes_index(df, (R, R, R), level)
    info["band"] = binfo
    return verts, faces, info


@torch.no_grad()
def iso_mesh_sparse(query, bound_min, bound_max, resolution, level, lipschitz=2.0, strides=None, max_batch=1 << 21,
                    device=None):
    """`iso_mesh_band` on the block-sparse band (grid.iso_band_sparse, iso_marching_cubes_sparse): the same (fp64 verts,
    int64 faces, info with info["band"]), with no array of R^3 elements, for lattices up to 2048^3.

    The store reads iso_band's df at every lattice point whatever the field, and the active cells, faces and vertices are
    those of that df, so the mesh is iso_mesh_band's bit for bit; it is the dense one under iso_mesh_band's conditions."""
    from neuraludf_b200 import grid
    band, binfo = grid.iso_band_sparse(query, bound_min, bound_max, resolution, level, lipschitz=lipschitz,
                                       strides=strides, max_batch=max_batch, device=device)
    verts, faces, info = iso_marching_cubes_sparse(band, level)
    info["band"] = binfo
    return verts, faces, info


def iso_marching_cubes(volume, isovalue):
    """Threshold marching cubes with `mcubes.marching_cubes(volume, isovalue)`'s call signature, on the CUDA kernels:
    NumPy (vertices fp64 [V,3] in array-index units, triangles int64 [F,3]).

    `volume` is meshed as fp32 and `isovalue` is rounded to fp32 once.  A level that nothing crosses gives empty (0, 3)
    arrays.  A volume that is not 3-D or has a dimension below 2, or a non-finite level, raises ValueError.  Faces are wound
    towards decreasing values (the convention NeuS-family code relies on when it meshes -sdf at 0).  The vertex numbering
    and the triangulation of ambiguous cells are this project's (iso_marching_cubes_index), not PyMCubes'."""
    volume = np.asarray(volume)
    if volume.ndim != 3:
        raise ValueError("volume must be a 3-D array (got %d dimensions)" % volume.ndim)
    if min(volume.shape) < 2:
        raise ValueError("volume must be at least 2 x 2 x 2 (got %s)" % (volume.shape,))
    _iso_level(isovalue)
    dev = torch.device("cuda", torch.cuda.current_device())
    df = torch.from_numpy(np.ascontiguousarray(volume, np.float32)).to(dev)
    verts, faces, _ = iso_marching_cubes_index(df, volume.shape, isovalue)
    return verts.cpu().numpy(), faces.cpu().numpy()


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
    hi = N ** 3 if hi is None else hi
    if lo % (N * N) or hi % (N * N) or not 0 <= lo < hi <= N ** 3:
        raise ValueError("lo / hi must select whole x-planes of the N^3 lattice")
    return _udf_mesh(udf_network, N, "dense", dist_threshold_ratio, max_batch=max_batch, lo=lo, hi=hi)


def _no_mark(stage):
    pass


def _mc_lattice(udf_network, N, df, lo, max_batch, mark=_no_mark):
    """near-surface normals -> MC of the lattice values df (whole x-planes from flat index lo): (verts [V,3] fp32 in the
    slab's lattice-index units, faces [F,3] int64); mark(stage) is called after the normals and after the MC"""
    from neuraludf_b200 import grid
    planes = df.numel() // (N * N)
    idx, normals = grid.near_surface_cells(udf_network, N, df, max_batch=max(max_batch // 2, 1), lo=lo)
    mark("normals")
    verts, faces, _ = marching_cubes_index(df, (planes, N, N), normals, idx - lo)
    mark("mc")
    return verts, faces


def _udf_mc(udf_network, N, lattice, lipschitz=2.0, strides=None, max_batch=1 << 21, lo=0, hi=None, mark=_no_mark):
    """The raw MeshUDF MC of the N^3 lattice evaluated `lattice`: "dense" (grid.udf_grid of the slab [lo, hi)), "band"
    (grid.udf_band) or "sparse" (grid.udf_band_sparse): (verts [V,3] fp32 in the slab's lattice-index units, faces [F,3]
    int64).  Negative lattice values are set to 0 (extract_mesh.py:196; a UDF network gives none) after the normals'
    selection, which reads them unchanged either way (< 2 voxels); on the sparse lattice in the coarse array and bricks.  The lattice is released on return.  mark(stage) is
    called after the lattice, the normals and the MC."""
    from neuraludf_b200 import grid
    if lattice == "sparse":
        band, _ = grid.udf_band_sparse(udf_network, N, lipschitz=lipschitz, strides=strides, max_batch=max_batch)
        mark("lattice")
        idx, normals = grid.near_surface_cells_sparse(udf_network, band, max_batch=max(max_batch // 2, 1))
        band.coarse.masked_fill_(band.coarse < 0, 0.0)              # the clamp below, on what the store holds
        band.bricks.masked_fill_(band.bricks < 0, 0.0)
        mark("normals")
        verts, faces, _ = marching_cubes_sparse(band, normals, idx)
        mark("mc")
        return verts, faces
    if lattice == "dense":
        df = grid.udf_grid(udf_network, N, max_batch=max_batch, lo=lo, hi=hi)
    else:
        df, _ = grid.udf_band(udf_network, N, lipschitz=lipschitz, strides=strides, max_batch=max_batch)
    df.masked_fill_(df < 0, 0.0)
    mark("lattice")
    return _mc_lattice(udf_network, N, df, lo, max_batch, mark)


def _udf_mesh(udf_network, N, lattice, dist_threshold_ratio, lipschitz=2.0, strides=None, max_batch=1 << 21, lo=0, hi=None):
    """_udf_mc's MC with the vertex filter: udf_mesh, udf_mesh_band or udf_mesh_sparse as `lattice` names it"""
    verts, faces = _udf_mc(udf_network, N, lattice, lipschitz, strides, max_batch, lo, hi)
    return _vertex_filter(udf_network, N, verts, faces, dist_threshold_ratio, lo, max_batch if lattice == "sparse" else None)


def _lattice_kind(dense, sparse):
    """the lattice _udf_mc evaluates for udf_mesh_post's / the CLI's dense and sparse switches"""
    return "dense" if dense else ("sparse" if sparse else "band")


def _batched_values(udf_network, pts, max_batch):
    """udf_values of pts [P,3] in batches of max_batch (None: one call), flat: the same bits when udf_values is batch-invariant"""
    if max_batch is None:
        return udf_network.udf_values(pts).reshape(-1)
    return torch.cat([udf_network.udf_values(pts[h:h + max_batch]).reshape(-1) for h in range(0, pts.shape[0], max_batch)])


def _vertex_filter(udf_network, N, verts, faces, dist_threshold_ratio, lo, max_batch=None):
    """world coordinates and the vertex filter of extract_mesh.py:205-214 for an MC of whole x-planes from flat index lo;
    the udf at the vertices in batches of max_batch (None: one call)"""
    voxel = 2.0 / (N - 1)
    verts = verts * voxel - 1.0
    verts[:, 0] += (lo // (N * N)) * voxel
    if faces.shape[0] == 0:
        return verts, faces
    vd = _batched_values(udf_network, verts, max_batch)
    keep = vd[faces].max(dim=1).values < voxel * dist_threshold_ratio
    return _compact(verts, faces[keep])


@torch.no_grad()
def udf_mesh_band(udf_network, N, dist_threshold_ratio=1.0, lipschitz=2.0, strides=None, max_batch=1 << 21):
    """`udf_mesh` with the lattice evaluated narrow-band (grid.udf_band) instead of densely: the same (verts, faces).

    Exact when the field is `lipschitz`-Lipschitz and `udf_values` / `gradient` give the same bits for a point in any batch:
    udf_band's df then equals the dense one below 2 voxels and is >= 2 voxels (+inf) elsewhere, so near_surface_cells picks
    the same points and normals, an unevaluated (+inf) corner fails the MC's active-cell test (max <= 1.74 voxel) exactly
    as its dense value >= 2 voxels does, and the later MC stages read df only at the corners of active cells
    (csrc/mesh_udf.cu).  grid.udf_band warns when the lattice shows a slope above `lipschitz`."""
    return _udf_mesh(udf_network, N, "band", dist_threshold_ratio, lipschitz, strides, max_batch)


@torch.no_grad()
def udf_mesh_sparse(udf_network, N, dist_threshold_ratio=1.0, lipschitz=2.0, strides=None, max_batch=1 << 21):
    """`udf_mesh_band` on the block-sparse band (grid.udf_band_sparse, near_surface_cells_sparse, marching_cubes_sparse):
    the same (verts, faces), with no array of N^3 elements.

    Exact under udf_mesh_band's conditions: the store then reads udf_band's df at every lattice point (DESIGN.md section 1),
    so every stage sees the same values.  The store is released before the vertex filter, which evaluates the vertices in
    batches of max_batch (at 2048^3 a single batch of every vertex would need tens of GB of value-chain workspace)."""
    return _udf_mesh(udf_network, N, "sparse", dist_threshold_ratio, lipschitz, strides, max_batch)


@torch.no_grad()
def udf_mesh_post(udf_network, N, dist_threshold_ratio=5.0, dense=False, lipschitz=2.0, strides=None, smooth_borders=True,
                  max_batch=1 << 21, sparse=False):
    """The mesh `Runner.extract_udf_mesh` exports, before its world transform and final merge: (fp64 verts [V,3], int64
    faces [F,3], info) on the device.

    The lattice is evaluated narrow-band (`udf_mesh_band`'s, `lipschitz` / `strides`), with `sparse` narrow-band into the
    block-sparse store (`udf_mesh_sparse`'s, the same mesh), or with `dense` whole (`udf_mesh`'s); the normals and MC are
    theirs.  The vertices are then formed as the reference holds them, fp64(fp32 MC vertex) *
    fp64(voxel) - 1 in fp64, the vertex filter of extract_mesh.py:205-214 evaluates the udf at their fp32 rounding, and
    `mesh_post.postprocess` does the rest of get_mesh_udf_fast (extract_mesh.py:215-265; the runner passes
    `dist_threshold_ratio` 5 and `smooth_borders` True).  info: postprocess's, plus `mc` ((V, F) of the raw MC),
    `filtered` (faces after the vertex filter) and `stage_ms` (_mesh_post's)."""
    if dense and sparse:
        raise ValueError("udf_mesh_post: dense and sparse exclude each other")
    return _mesh_post(udf_network, N, _lattice_kind(dense, sparse), dist_threshold_ratio, smooth_borders, lipschitz, strides,
                      max_batch)


def _mesh_post(field, N, lattice, dist_threshold_ratio, smooth_borders, lipschitz=2.0, strides=None, max_batch=1 << 21):
    """get_mesh_udf_fast up to its gradient branch (extract_mesh.py:194-265) on `field`, the lattice evaluated as _udf_mc's
    `lattice` names it: (fp64 verts [V,3], int64 faces [F,3], info) on the device.  `field` is a UDF network (its
    udf_values and runner-normalised gradient: udf_mesh_post) or anything with udf_values(points [P,3]) -> [P] and
    surface_normals(points) -> unit vectors towards the surface [P,3] (extract_mesh.CallerField).

    The vertices are formed as the reference holds them, fp64(fp32 MC vertex) * fp64(voxel) - 1 in fp64; the vertex filter
    evaluates the field at their fp32 rounding in one call (in batches of max_batch on the sparse lattice) and keeps the
    faces whose vertices are all below voxel * dist_threshold_ratio; mesh_post.postprocess does the rest.  info:
    postprocess's, plus `mc` ((V, F) of the raw MC), `filtered` (faces after the vertex filter) and `stage_ms` (CUDA-event
    milliseconds of the lattice, normals, mc, filter and post stages)."""
    from neuraludf_b200 import mesh_post
    voxel = 2.0 / (N - 1)
    events = [("start", torch.cuda.Event(enable_timing=True))]
    events[0][1].record()

    def mark(stage):
        events.append((stage, torch.cuda.Event(enable_timing=True)))
        events[-1][1].record()

    verts, faces = _udf_mc(field, N, lattice, lipschitz, strides, max_batch, mark=mark)
    v64 = verts.double() * voxel - 1.0
    n_mc = faces.shape[0]
    if n_mc:
        vd = _batched_values(field, v64.float(), max_batch if lattice == "sparse" else None)
        faces = faces[vd[faces].max(dim=1).values < voxel * dist_threshold_ratio]
    mark("filter")
    v, f, info = mesh_post.postprocess(v64, faces, smooth_borders=smooth_borders)
    mark("post")
    info["mc"], info["filtered"] = (verts.shape[0], n_mc), int(faces.shape[0])
    torch.cuda.synchronize(v.device)
    info["stage_ms"] = {b[0]: a[1].elapsed_time(b[1]) for a, b in zip(events, events[1:])}
    return v, f, info


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


def udf_network_from_state(sd, scale=1.0):
    """A UDFNetwork holding the state dict `sd` (the runner's `udf_network_fine`), its n_layers, d_hidden, d_out, skip_in and
    multires read off the weight shapes: lin0 is [d_hidden, 3 + 6 multires], a layer feeding the skip is
    [d_hidden - (3 + 6 multires), d_hidden], the last one [d_out, d_hidden].  `scale` is not stored in the weights (every
    shipped conf uses 1.0)."""
    from neuraludf_b200.models.fields import UDFNetwork
    n_lin = 0
    while "lin%d.weight_v" % n_lin in sd:
        n_lin += 1
    if n_lin < 2:
        raise ValueError("not a UDFNetwork state dict (no lin0 / lin1 .weight_v)")
    d_hidden, input_ch = (int(x) for x in sd["lin0.weight_v"].shape)
    if (input_ch - 3) % 6:
        raise ValueError("lin0 takes %d inputs: not 3 + 6 multires" % input_ch)
    skip_in = tuple(l + 1 for l in range(n_lin - 2) if int(sd["lin%d.weight_v" % l].shape[0]) == d_hidden - input_ch)
    net = UDFNetwork(d_in=3, d_out=int(sd["lin%d.weight_v" % (n_lin - 1)].shape[0]), d_hidden=d_hidden, n_layers=n_lin - 1,
                     skip_in=skip_in, multires=(input_ch - 3) // 6, scale=scale, geometric_init=False, weight_norm=True,
                     udf_type="abs")
    net.load_state_dict(sd)
    return net


def threshold_box(cameras=None):
    """The box and world transform of the runner's validate_mesh: (bbox_min, bbox_max) fp32 [3] as dataset/dataset.py:112-123
    forms object_bbox_min / max from the cameras file's fp32 scale_mat_0 (both camera roles read the same file in the shipped
    confs) and its fp64 object scale_mat_0, or +-1.01 without a cameras file; and the fp32 scale_mat_0 (None without)."""
    bmin = np.array([-1.01, -1.01, -1.01, 1.0])
    bmax = np.array([1.01, 1.01, 1.01, 1.0])
    if cameras is None:
        return bmin[:3].astype(np.float32), bmax[:3].astype(np.float32), None
    cam = np.load(cameras)
    sm = cam["scale_mat_0"].astype(np.float32)
    obj = cam["scale_mat_0"]
    lo = np.linalg.inv(sm) @ obj @ bmin[:, None]
    hi = np.linalg.inv(sm) @ obj @ bmax[:, None]
    return lo[:3, 0].astype(np.float32), hi[:3, 0].astype(np.float32), sm


def main(argv=None):
    """python -m neuraludf_b200.mesh: a runner checkpoint's UDF network -> PLY mesh (see INTEGRATION.md)"""
    import argparse
    from neuraludf_b200.evaluate import write_ply_mesh
    ap = argparse.ArgumentParser(prog="python -m neuraludf_b200.mesh",
                                 description="Mesh the UDF network of a runner checkpoint: the mesh as udf_mesh makes it, with "
                                             "--postprocess the mesh the runner's extract_udf_mesh exports, or with --threshold "
                                             "the mesh the runner's validate_mesh exports.")
    ap.add_argument("--ckpt", required=True, help="checkpoint written by the runner (its udf_network_fine state dict is used)")
    ap.add_argument("--resolution", type=int, default=512, help="lattice points per axis")
    ap.add_argument("--cameras", default=None, help="cameras_sphere.npz: map the mesh to world space with its scale_mat_0 "
                                                    "(with --threshold it also sets the box, as the runner's dataset does)")
    ap.add_argument("--threshold", type=float, default=None,
                    help="threshold meshing of the udf at this level on validate_mesh's lattice (the box +-1.01, or the "
                         "object box of --cameras) instead of the MeshUDF pipeline: the mesh the runner's "
                         "validate_mesh(world_space=True) exports with --cameras; the runner passes --threshold 0.005")
    ap.add_argument("--dist_threshold_ratio", type=float, default=None, help="vertex filter in voxels (default 1)")
    ap.add_argument("--band", action="store_true",
                    help="with --threshold: evaluate the lattice narrow-band (grid.iso_band) and mesh it on the device, "
                         "the same mesh when the udf is --lipschitz-Lipschitz")
    ap.add_argument("--lipschitz", type=float, default=None, help="Lipschitz bound of the band's culling test (default 2)")
    ap.add_argument("--scale", type=float, default=1.0, help="the conf's udf_network.scale")
    ap.add_argument("--dense", action="store_true", help="evaluate the whole lattice (udf_mesh) instead of the narrow band")
    ap.add_argument("--sparse", action="store_true",
                    help="hold the narrow band block-sparse (udf_mesh_sparse, or iso_mesh_sparse with --threshold "
                         "--band): the same mesh with no N^3 array, for --resolution up to 2048")
    ap.add_argument("--postprocess", action="store_true",
                    help="apply the runner's post-processing (merge, duplicate and degenerate faces, hole filling, border "
                         "smoothing, the final merge after --cameras): the mesh Runner.extract_udf_mesh writes; the runner "
                         "passes --dist_threshold_ratio 5")
    ap.add_argument("--out", required=True, help="output PLY")
    a = ap.parse_args(argv)
    if a.sparse and (a.dense or (a.threshold is not None and not a.band)):
        ap.error("--sparse cannot be combined with %s" % ("--dense" if a.dense else "--threshold without --band"))
    if a.band and a.threshold is None:
        ap.error("--band needs --threshold (the MeshUDF lattice is evaluated narrow-band without it)")
    if a.threshold is not None:
        for flag, given in (("--postprocess", a.postprocess), ("--dense", a.dense),
                            ("--lipschitz", a.lipschitz is not None and not a.band),
                            ("--dist_threshold_ratio", a.dist_threshold_ratio is not None)):
            if given:
                ap.error("--threshold cannot be combined with %s" % flag)
    a.dist_threshold_ratio = 1.0 if a.dist_threshold_ratio is None else a.dist_threshold_ratio
    a.lipschitz = 2.0 if a.lipschitz is None else a.lipschitz
    if not torch.cuda.is_available():
        raise SystemExit("meshing runs on a CUDA device")
    ck = torch.load(a.ckpt, map_location="cpu", weights_only=True)
    net = udf_network_from_state(ck["udf_network_fine"] if "udf_network_fine" in ck else ck, a.scale).cuda()
    if a.threshold is not None:                   # exp_runner_blending.py:746-761, renderer.extract_geometry
        from neuraludf_b200.models.udf_renderer_blending import box_vertices, extract_geometry
        bmin, bmax, sm = threshold_box(a.cameras)
        bmin, bmax = torch.tensor(bmin, dtype=torch.float32), torch.tensor(bmax, dtype=torch.float32)
        if a.band:                                # extract_geometry's device path with NUDF_BAND_MESH=1 (or =sparse)
            v, faces, _ = (iso_mesh_sparse if a.sparse else iso_mesh_band)(lambda pts: net.udf_values(pts), bmin, bmax, a.resolution, a.threshold,
                                        lipschitz=a.lipschitz, device=torch.device("cuda"))
            v, faces = box_vertices(v.cpu().numpy(), a.resolution, bmin, bmax), faces.cpu().numpy()
        else:
            v, faces = extract_geometry(bmin, bmax, a.resolution, a.threshold, lambda pts: net.udf_values(pts),
                                        torch.device("cuda"))
        if sm is not None:
            v = v * sm[0, 0] + sm[:3, 3][None]
        write_ply_mesh(a.out, v, faces)
        print("%s: %d vertices, %d faces" % (a.out, v.shape[0], faces.shape[0]))
        return v, np.asarray(faces)
    if a.postprocess:
        verts, faces, _ = udf_mesh_post(net, a.resolution, a.dist_threshold_ratio, dense=a.dense, lipschitz=a.lipschitz,
                                        sparse=a.sparse)
    else:
        verts, faces = _udf_mesh(net, a.resolution, _lattice_kind(a.dense, a.sparse), a.dist_threshold_ratio, a.lipschitz)
    v = verts.double().cpu().numpy()
    if a.cameras is not None:                     # exp_runner_blending.py:792-794, with the dataset's fp32 scale_mat_0
        sm = np.load(a.cameras)["scale_mat_0"].astype(np.float32)
        v = v * sm[0, 0] + sm[:3, 3][None]
    if a.postprocess:                             # exp_runner_blending.py:796: Trimesh(...) merges once more
        from neuraludf_b200.mesh_post import export_merge
        vt, faces = export_merge(torch.from_numpy(v).to(verts.device), faces)
        v = vt.cpu().numpy()
    write_ply_mesh(a.out, v, faces)
    print("%s: %d vertices, %d faces" % (a.out, v.shape[0], faces.shape[0]))
    return v, faces.cpu().numpy()


if __name__ == "__main__":
    main()

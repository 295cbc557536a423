"""Dense UDF grid queries for mesh extraction with a device-side hand-off (SURVEY.md 8(f) rank 2, BASELINE config 5).

The reference fills an N^3 lattice by shipping every batch of points host -> device -> host and then evaluates the gradient
where `udf < 2 voxels`, again batch by batch through the host (`extract_mesh.py:18-105 get_udf_normals_grid_slow`).  Here
the lattice coordinates are generated on the device, the value sweep runs on the fused value-chain kernel, the
near-surface cells are compacted on the device and only they go through the fused value + reverse-sweep kernel; the result
is handed over as the dense distance grid plus a SPARSE list of near-surface cells (flat index + unit normal) -- 67 MB +
~7 MB at 256^3 instead of the reference's 67 MB + 201 MB dense normal grid and its ~130 blocking copies.
`get_udf_normals_grid_slow` keeps the reference's return convention for `udf_mc_lewiner` (the Cython MeshUDF marching cubes,
out of scope).  `udf_band` is the coarse-to-fine alternative to the dense sweep: it evaluates the lattice only where a
Lipschitz bound cannot rule out udf < 2 voxels (kernels in csrc/mesh_band.cu).  `iso_band` does the same for the threshold
lattice of validate_mesh (any box, torch.linspace coordinates): it evaluates every point a threshold mesh at `level` can
read.  `udf_band_sparse` runs udf_band's levels into a block-sparse store (SparseBand: a coarse dense array plus 8^3
bricks, csrc/mesh_sparse.cu) instead of an N^3 array, and `near_surface_cells_sparse` selects the band from it: what
mesh.udf_mesh_sparse meshes at 2048^3.  `iso_band_sparse` runs iso_band's levels into the same store: what
mesh.iso_mesh_sparse meshes."""
import ctypes
import math
import warnings

import torch
import torch.nn.functional as F

from neuraludf_b200 import _lib
from neuraludf_b200._lib import check, ptr


def lattice_points(head, count, N, device):
    """points `head .. head+count-1` of the N^3 lattice on [-1,1]^3 in the reference's order (x slowest, z fastest;
    extract_mesh.py:38-51), generated on the device"""
    return _index_points(torch.arange(head, head + count, device=device, dtype=torch.int64), N)


def _index_points(idx, N):
    """fp32 points [P,3] of the flat lattice indices idx on the N^3 lattice on [-1,1]^3"""
    voxel = 2.0 / (N - 1)
    k = idx % N
    j = torch.div(idx, N, rounding_mode="floor") % N
    i = torch.div(torch.div(idx, N, rounding_mode="floor"), N, rounding_mode="floor") % N
    return torch.stack([i.float() * voxel - 1.0, j.float() * voxel - 1.0, k.float() * voxel - 1.0], dim=-1)


@torch.no_grad()
def udf_grid(udf_network, N, max_batch=1 << 21, lo=0, hi=None):
    """udf at the lattice points [lo, hi) (default: all N^3) as a flat device tensor -- one fused-chain launch per batch,
    no host round trips.  Slab partitioning for multi-GPU sweeps: give each rank its own [lo, hi)."""
    device = _device(udf_network)
    hi = N ** 3 if hi is None else hi
    out = torch.empty(hi - lo, device=device)
    for head in range(lo, hi, max_batch):
        n = min(max_batch, hi - head)
        out[head - lo:head - lo + n] = udf_network.udf_values(lattice_points(head, n, N, device))
    return out


@torch.no_grad()
def near_surface_cells(udf_network, N, df_flat=None, max_batch=1 << 20, dist_voxels=2.0, lo=0):
    """(flat lattice indices [M] int64, unit vectors pointing towards the surface [M,3]) of the cells with
    udf < dist_voxels * voxel (extract_mesh.py:77-98): compaction and gradient evaluation stay on the device."""
    if df_flat is None:
        df_flat = udf_grid(udf_network, N)
    voxel = 2.0 / (N - 1)
    idx = torch.nonzero(df_flat < dist_voxels * voxel).reshape(-1) + lo
    return idx, _surface_normals(udf_network, N, idx, max_batch)


def _runner_normals(udf_network, pts):
    """unit vectors towards the surface at pts from a UDF network's gradient, normalised as the runner's func_grad does"""
    g = udf_network.gradient(pts)[:, 0]
    g = g / (torch.linalg.norm(g, ord=2, dim=-1, keepdim=True) + 1e-5)              # exp_runner_blending.py:767-771 (func_grad)
    return -F.normalize(g, dim=1)                                                    # extract_mesh.py:93


def _surface_normals(udf_network, N, idx, max_batch):
    """unit vectors towards the surface at the flat lattice indices idx (extract_mesh.py:77-98), batches of max_batch: the
    field's own `surface_normals(points)` when it has one (extract_mesh.CallerField: a caller's func_grad), else the UDF
    network's runner-normalised gradient"""
    at = getattr(udf_network, "surface_normals", None) or (lambda pts: _runner_normals(udf_network, pts))
    normals = torch.empty(idx.numel(), 3, device=idx.device)
    for head in range(0, idx.numel(), max_batch):
        sel = idx[head:head + max_batch]
        normals[head:head + sel.numel()] = at(_index_points(sel, N))
    return normals


def default_strides(N):
    """the band schedule udf_band uses when none is given: halving strides from the largest power of two <= (N - 1) / 16
    down to 1 (DESIGN.md section 8 compares schedules)"""
    s = 1
    while 2 * s <= (N - 1) // 16:
        s *= 2
    out = [s]
    while out[-1] > 1:
        out.append(out[-1] // 2)
    return out


def _check_strides(strides):
    strides = [int(s) for s in strides]
    if not strides or strides[-1] != 1 or any(s < 1 for s in strides):
        raise ValueError("strides must be positive and end with 1, got %s" % (strides,))
    if any(a <= b or a % b for a, b in zip(strides, strides[1:])):
        raise ValueError("each stride must be a proper multiple of the next, got %s" % (strides,))
    return strides


def _device(udf_network):
    try:
        return next(udf_network.parameters()).device
    except (AttributeError, StopIteration):
        return torch.device("cuda", torch.cuda.current_device())


def _coords(N, axes=None, spacing=None, pad=0.0):
    """the nudf_band_coords of the N^3 band lattice, by reference: the cube [-1,1]^3 (axes None) or the fp32 tables `axes`
    (three contiguous [N] device tensors) with their largest steps `spacing` and the block test's `pad`"""
    if axes is None:
        return ctypes.byref(_lib.BandCoords(voxel=2.0 / (N - 1)))
    if len(axes) != 3 or any(x.dtype != torch.float32 or x.shape != (N,) or not x.is_contiguous() for x in axes):
        raise ValueError("axes must be three contiguous float32 tables of %d coordinates" % N)
    return ctypes.byref(_lib.BandCoords(0.0, (ctypes.c_void_p * 3)(*(x.data_ptr() for x in axes)),
                                        (ctypes.c_double * 3)(*(float(h) for h in spacing or (0.0, 0.0, 0.0))), float(pad)))


def band_sublattice(N, s, device, axes=None):
    """(flat indices [m^3] int64, points [m^3,3] fp32) of the stride-s lattice: 0, s, 2 s, ... and N - 1 per axis;
    coordinates on [-1,1]^3, or from the three fp32 tables `axes` (iso_band)"""
    m = -(-(N - 1) // s) + 1
    idx = torch.empty(m ** 3, dtype=torch.int64, device=device)
    pts = torch.empty(m ** 3, 3, device=device)
    check(_lib.lib().nudf_nb_sublattice(N, s, _coords(N, axes), ptr(idx), ptr(pts), _lib.stream_ptr()), "nudf_nb_sublattice")
    return idx, pts


class _DenseLattice:
    """The N^3 lattice as one flat fp32 array `df`, +inf where never stored: the store of udf_band and iso_band."""

    def __init__(self, df, N):
        self.df, self.N = df, N

    @property
    def device(self):
        return self.df.device

    def lattice(self):
        """the nudf_lattice descriptor, by reference"""
        return ctypes.byref(_lib.Lattice(self.N, self.N, self.N, self.df.data_ptr(), None))

    def store(self, idx, vals):
        self.df[idx] = vals

    def level_kept(self, flags, s):
        pass


def band_block_test(df, N, s, parent=None, parent_s=0, lipschitz=2.0, tau=None, flags=True, axes=None, spacing=None, pad=0.0):
    """(kept flags [nb^3] uint8 or None, largest edge slope) of the blocks of stride s (csrc/mesh_band.cu): candidates are every
    block, or those inside a kept block of `parent` (stride parent_s).  df: the flat fp32 lattice, or a store with lattice()
    (SparseBand).  On [-1,1]^3 the threshold `tau` defaults to 2 voxels; with the fp32 tables `axes` the table rule: r from
    the block's table coordinates plus `pad`, `tau` as given, edge slopes over `spacing` (the largest step per axis)."""
    lat = _DenseLattice(df, N).lattice() if torch.is_tensor(df) else df.lattice()
    device = df.device
    nb = -(-(N - 1) // s)
    out = torch.empty(nb ** 3, dtype=torch.uint8, device=device) if flags else None
    slope = torch.zeros(1, dtype=torch.int32, device=device)
    tau = 2.0 * (2.0 / (N - 1)) if tau is None else tau
    check(_lib.lib().nudf_nb_lat_block_test(lat, s, ptr(parent), parent_s, _coords(N, axes, spacing, pad), float(lipschitz),
                                            float(tau), ptr(out), ptr(slope), _lib.stream_ptr()), "nudf_nb_lat_block_test")
    return out, float(slope.view(torch.float32))


def band_points(flags, N, s, t, axes=None):
    """(flat indices [M] int64, points [M,3] fp32, kept block count): the stride-t points that the kept blocks of stride s
    emit, each point once (the lowest-numbered kept block holding it), blocks ascending, each in lexicographic order;
    coordinates on [-1,1]^3, or from the three fp32 tables `axes` (iso_band)"""
    (out,) = _band_chunks(flags, N, s, t, axes)
    return out


def _band_chunks(flags, N, s, t, axes=None, chunk=None):
    """band_points in its order, cut between kept blocks into chunks of about `chunk` points (None: one chunk), so that a
    level need not hold all its points at once: yields (idx, pts, kept blocks) per chunk, at least one"""
    L = _lib.lib()
    st = _lib.stream_ptr()
    co = _coords(N, axes)
    kept = torch.nonzero(flags).reshape(-1)
    n = kept.numel()
    counts = torch.empty(n, dtype=torch.int32, device=flags.device)
    check(L.nudf_nb_count(ptr(flags), N, s, t, ptr(kept), n, ptr(counts), st), "nudf_nb_count")
    csum = torch.cumsum(counts, 0, dtype=torch.int64)
    total = int(csum[-1]) if chunk is not None and n else 0
    cuts = []
    if chunk is not None and total > chunk:
        cuts = torch.searchsorted(csum, torch.arange(chunk, total, chunk, device=flags.device), right=True).tolist()
    bounds = [0] + sorted(set(cuts) - {0, n}) + [n]
    head = 0
    for a, b in zip(bounds, bounds[1:]):
        end = int(csum[b - 1]) if b else 0
        offsets = (csum[a:b] - counts[a:b] - head).contiguous()
        idx = torch.empty(end - head, dtype=torch.int64, device=flags.device)
        pts = torch.empty(end - head, 3, device=flags.device)
        check(L.nudf_nb_emit(ptr(flags), N, s, t, ptr(kept[a:b]), b - a, ptr(offsets), co, ptr(idx), ptr(pts), st),
              "nudf_nb_emit")
        if b == n:                          # the level's block lists are not held while its last chunk is evaluated
            del kept, counts, csum, offsets
        yield idx, pts, b - a
        head = end


def _coarse_to_fine(store, values, N, strides, lipschitz, tau, max_batch, chunk=None, axes=None, spacing=None, pad=0.0):
    """The level loop of udf_band, iso_band and udf_band_sparse: fills `store` (store(idx, vals), lattice(), device and
    level_kept(flags, s), called after each block test that hands flags on) and returns info without the wrappers' own keys.
    values(pts [P,3]) -> [P] fp32, called in batches of max_batch; each level is emitted in chunks of about `chunk` points
    (None: whole); coordinates and block test as band_block_test's."""
    info = {"strides": strides, "points": [], "kept_blocks": [], "edge_slope": []}
    events = []

    def mark():
        events.append(torch.cuda.Event(enable_timing=True))
        events[-1].record()

    def evaluate(idx, pts):
        for head in range(0, idx.numel(), max_batch):
            store.store(idx[head:head + max_batch], values(pts[head:head + max_batch]))
        return int(idx.numel())

    mark()
    info["points"].append(evaluate(*band_sublattice(N, strides[0], store.device, axes)))
    mark()
    parent = None
    for k, s in enumerate(strides):
        last = k + 1 == len(strides)
        flags, slope = band_block_test(store, N, s, parent, strides[k - 1] if k else 0, lipschitz, tau, not last, axes,
                                       spacing, pad)
        info["edge_slope"].append(slope)
        if last:
            break
        store.level_kept(flags, s)
        n_points = n_kept = 0
        for idx, pts, n in _band_chunks(flags, N, s, strides[k + 1], axes, chunk):
            n_points += evaluate(idx, pts)
            n_kept += n
            del idx, pts
        info["points"].append(n_points)
        info["kept_blocks"].append(n_kept)
        mark()
        parent = flags
    del parent, flags
    mark()
    torch.cuda.synchronize(store.device)
    ms = [a.elapsed_time(b) for a, b in zip(events, events[1:])]
    # level 0: the stride-strides[0] lattice; level k: block test at strides[k-1], emission and evaluation of strides[k]
    # points; slope_ms: the slope pass over the finest level
    info["level_ms"], info["slope_ms"] = ms[:-1], ms[-1]
    info["max_edge_slope"] = max(info["edge_slope"])
    return info


def _warn_slope(info, lipschitz, what, miss):
    """the RuntimeWarning of the band builders when a lattice edge is steeper than `lipschitz`"""
    if info["max_edge_slope"] > lipschitz:
        warnings.warn("%s: a lattice edge has slope %.3f > lipschitz=%.3f: the field is not %.3f-Lipschitz, so %s"
                      % (what, info["max_edge_slope"], lipschitz, lipschitz, miss), RuntimeWarning, stacklevel=3)


@torch.no_grad()
def udf_band(udf_network, N, lipschitz=2.0, strides=None, max_batch=1 << 21):
    """Narrow-band udf lattice, coarse to fine: (df [N^3] fp32 flat, +inf where never evaluated; info).

    Level 0 evaluates the stride-strides[0] lattice; each next level evaluates, inside the blocks of the current stride that a
    Lipschitz bound cannot rule out (csrc/mesh_band.cu), the points of the next stride.  If the field is `lipschitz`-
    Lipschitz and `udf_values` gives the same bits for a point in any batch, `df` equals grid.udf_grid bit for bit wherever
    that is < 2 voxels (near_surface_cells' band), and every +inf stands for a value >= 2 voxels.  `udf_network`: any object
    with `udf_values(points [P,3]) -> [P]`.  info: strides, points evaluated per level, kept blocks per level, edge_slope per
    level (the largest |du| / edge length over the lattice edges of each level's candidate blocks) and its maximum
    `max_edge_slope` -- a lower bound on the field's Lipschitz constant: a RuntimeWarning is issued when it exceeds
    `lipschitz` -- and level_ms (CUDA events)."""
    strides = _check_strides(default_strides(N) if strides is None else strides)
    lattice = _DenseLattice(torch.full((N ** 3,), float("inf"), device=_device(udf_network)), N)
    info = _coarse_to_fine(lattice, lambda pts: udf_network.udf_values(pts).reshape(-1), N, strides, lipschitz,
                           2.0 * (2.0 / (N - 1)), max_batch)
    _warn_slope(info, lipschitz, "udf_band", "the band may miss points with udf < 2 voxels")
    return lattice.df, info


def sparse_coarse_stride(strides):
    """the stride c of SparseBand's coarse array for a schedule: its smallest stride >= 8 (one brick edge), else its first"""
    big = [s for s in strides if s >= _lib.BRICK]
    return big[-1] if big else strides[0]


class SparseBand:
    """The block-sparse narrow-band lattice of udf_band_sparse (nudf_brick_store in include/nudf.h; the reader BrickDf in
    csrc/df_access.cuh).  The points of the stride-c lattice (per axis 0, c, 2 c, ... and N - 1) are held in the dense
    array `coarse` [mc^3], mc = ceil((N - 1) / c) + 1; every other point in an 8^3 brick: `dir` [nbk^3] int32
    (nbk = ceil(N / 8)) gives each brick's slot in `bricks` [slots * 512] or -1, `keys` [slots] the brick number of each
    slot, ascending.  A point never stored reads +inf, as in udf_band's df.  `values(idx)` reads flat lattice indices."""

    def __init__(self, N, c, device):
        self.N, self.c = int(N), int(c)
        self.mc = -(-(self.N - 1) // self.c) + 1
        self.nbk = -(-self.N // _lib.BRICK)
        self.coarse = torch.full((self.mc ** 3,), float("inf"), device=device)
        self.dir = torch.full((self.nbk ** 3,), -1, dtype=torch.int32, device=device)
        self.bricks = torch.empty(0, device=device)
        self.keys = torch.empty(0, dtype=torch.int64, device=device)
        self._missing = torch.zeros(1, dtype=torch.int32, device=device)

    @property
    def device(self):
        return self.coarse.device

    @property
    def n_bricks(self):
        return self.keys.numel()

    def _desc(self):
        """the nudf_brick_store descriptor (host struct of device pointers), kept alive until the next call"""
        self._d = _lib.BrickStore(self.N, self.c, self.mc, self.nbk, self.n_bricks, self.coarse.data_ptr(),
                                  self.dir.data_ptr(), self.bricks.data_ptr() if self.n_bricks else None,
                                  self.keys.data_ptr() if self.n_bricks else None)
        return self._d

    def lattice(self):
        """the nudf_lattice descriptor naming the store, by reference"""
        return ctypes.byref(_lib.Lattice(self.N, self.N, self.N, None, ctypes.pointer(self._desc())))

    def nbytes(self):
        """bytes held: coarse, dir, bricks (with keys)"""
        return {"coarse": self.coarse.numel() * 4, "dir": self.dir.numel() * 4,
                "bricks": self.bricks.numel() * 4 + self.keys.numel() * 8}

    def allocate(self, flags, s):
        """slots for every brick that meets the closed box of a kept block of stride s (flags: the block test's)"""
        L = _lib.lib()
        marks = torch.zeros(self.nbk ** 3, dtype=torch.int32, device=self.device)
        check(L.nudf_sb_mark(ctypes.byref(self._desc()), s, ptr(flags), ptr(marks), _lib.stream_ptr()), "nudf_sb_mark")
        keys = torch.nonzero(marks).reshape(-1)
        del marks
        self.dir.fill_(-1)
        self.dir[keys] = torch.arange(keys.numel(), dtype=torch.int32, device=self.device)
        self.keys = keys.contiguous()
        self.bricks = torch.full((keys.numel() * _lib.BRICK ** 3,), float("inf"), device=self.device)

    def level_kept(self, flags, s):
        """udf_band_sparse's levels: the bricks are allocated after the block test at stride c"""
        if s == self.c:
            self.allocate(flags, s)

    def store(self, idx, vals):
        """write vals [P] fp32 at the flat lattice indices idx [P]; a point with no storage raises at check_stored()"""
        vals = vals.reshape(-1).float().contiguous()
        check(_lib.lib().nudf_sb_store(ctypes.byref(self._desc()), ptr(idx), ptr(vals), idx.numel(), ptr(self._missing),
                                       _lib.stream_ptr()), "nudf_sb_store")

    def check_stored(self):
        if int(self._missing.item()):
            raise RuntimeError("SparseBand: a value was stored outside the coarse lattice and every brick")

    def values(self, idx):
        """fp32 values at the flat lattice indices idx (int64 device tensor)"""
        idx = idx.reshape(-1).to(torch.int64).contiguous()
        out = torch.empty(idx.numel(), device=self.device)
        check(_lib.lib().nudf_sb_gather(ctypes.byref(self._desc()), ptr(idx), idx.numel(), ptr(out), _lib.stream_ptr()),
              "nudf_sb_gather")
        return out

    def flat_index(self, pos):
        """flat lattice indices of storage positions pos (int64: [0, mc^3) coarse, then mc^3 + slot * 512 + local)"""
        out = torch.empty(pos.numel(), dtype=torch.int64, device=self.device)
        check(_lib.lib().nudf_sb_flat(ctypes.byref(self._desc()), ptr(pos), pos.numel(), ptr(out), _lib.stream_ptr()),
              "nudf_sb_flat")
        return out


@torch.no_grad()
def udf_band_sparse(udf_network, N, lipschitz=2.0, strides=None, max_batch=1 << 21):
    """udf_band's lattice without an N^3 array: (SparseBand, info).

    The levels are udf_band's -- the same sub-lattice, block tests (reading the store), point emission and evaluation --
    so the same RuntimeWarning when max_edge_slope exceeds `lipschitz`.  The points of strides >= c
    (sparse_coarse_stride) go to the coarse array; after the block test at stride c, every brick meeting a kept stride-c
    block is allocated, and the points of the finer strides, all inside those blocks, go to the bricks.  A level is
    emitted and evaluated in chunks of about max_batch points.  If `udf_values` gives a point the same bits in any batch,
    SparseBand.values equals udf_band's df at every lattice point, +inf included (DESIGN.md section 1).  info: udf_band's
    keys, plus coarse_stride, bricks (slots allocated) and bytes (SparseBand.nbytes, and the largest block-test flags
    array)."""
    strides = _check_strides(default_strides(N) if strides is None else strides)
    c = sparse_coarse_stride(strides)
    band = SparseBand(N, c, _device(udf_network))
    info = _coarse_to_fine(band, lambda pts: udf_network.udf_values(pts).reshape(-1), N, strides, lipschitz,
                           2.0 * (2.0 / (N - 1)), max_batch, chunk=max_batch)
    band.check_stored()
    info.update(coarse_stride=c, bricks=band.n_bricks,
                bytes=dict(band.nbytes(), flags=max([(-(-(N - 1) // s)) ** 3 for s in strides[:-1]], default=0)))
    _warn_slope(info, lipschitz, "udf_band_sparse", "the band may miss points with udf < 2 voxels")
    return band, info


@torch.no_grad()
def near_surface_cells_sparse(udf_network, band, max_batch=1 << 20, dist_voxels=2.0):
    """near_surface_cells on a SparseBand: (sorted flat lattice indices [M] int64, unit vectors towards the surface [M,3])
    of the points with udf < dist_voxels * voxel, the same comparison as near_surface_cells' (fp32 values against the
    threshold), over the coarse array and the bricks only.  Equal to near_surface_cells on udf_band's df when band equals
    it (udf_band_sparse)."""
    voxel = 2.0 / (band.N - 1)
    thr = dist_voxels * voxel
    pos = torch.cat([torch.nonzero(band.coarse < thr).reshape(-1),
                     torch.nonzero(band.bricks < thr).reshape(-1) + band.coarse.numel()])
    idx = torch.sort(band.flat_index(pos.contiguous())).values
    del pos
    return idx, _surface_normals(udf_network, band.N, idx, max_batch)


def axis_tables(bound_min, bound_max, resolution, device):
    """the coordinates of the threshold lattice on the box, per axis: torch.linspace(bound_min[a], bound_max[a], resolution)
    (fp32 [resolution], on `device`), the tables the dense sweep of extract_geometry evaluates"""
    return [torch.linspace(float(bound_min[a]), float(bound_max[a]), resolution, device=device) for a in range(3)]


def table_spacing(axes):
    """(h, e), three floats each, from the fp32 tables in fp64 (exact): h[a] the largest step |x[i+1] - x[i]| of table a and
    e[a] its largest excursion against its direction, min over the two directions of max_{i<j} (x[i] - x[j]) or
    max_{i<j} (x[j] - x[i]).  0 for a monotone table.  A point between two others on the lattice lies within e[a] of the
    interval their coordinates span, which is what iso_band's culling needs of the rounding in torch.linspace."""
    rows = []
    for x in axes:
        x = x.double()
        up = (torch.cummax(x, 0).values - x).max()
        down = (x - torch.cummin(x, 0).values).max()
        rows.append(torch.stack([(x[1:] - x[:-1]).abs().max(), torch.minimum(up, down)]))
    v = torch.stack(rows).cpu().tolist()
    return [r[0] for r in v], [r[1] for r in v]


def iso_cull(level, lipschitz, h, e):
    """(tau, pad) of iso_band's block test, fp64: D = sqrt(h_x^2 + h_y^2 + h_z^2) bounds the distance between two corners of
    one lattice cell; tau = level + L D, plus 1e-6 (|level| + L D) of slack against the rounding of D, tau and the block
    radius, so that tau exceeds the exact level + L D; pad = 1.000001 |e| enlarges every block radius by the tables'
    excursion (table_spacing)"""
    d = math.sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2])
    ld = lipschitz * d
    tau = (level + ld) + 1e-6 * (abs(level) + ld)
    pad = 1.000001 * math.sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2])
    return tau, pad


def _iso_setup(level, resolution, lipschitz, strides, bound_min, bound_max, device):
    """iso_band's checks, tables and block-test constants: (level, N, lipschitz, strides, device, axes, h, tau, pad)"""
    from neuraludf_b200.mesh import _iso_level
    level = _iso_level(level)
    N = int(resolution)
    if N < 2:
        raise ValueError("resolution must be at least 2 (got %r)" % (resolution,))
    lipschitz = float(lipschitz)
    if not 0.0 < lipschitz < float("inf"):
        raise ValueError("lipschitz must be positive and finite (got %r)" % (lipschitz,))
    strides = _check_strides(default_strides(N) if strides is None else strides)
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    axes = axis_tables(bound_min, bound_max, N, device)
    if any(x.dtype != torch.float32 for x in axes):
        raise ValueError("the lattice tables must be float32 (torch's default dtype is %s)" % torch.get_default_dtype())
    h, e = table_spacing(axes)
    tau, pad = iso_cull(level, lipschitz, h, e)
    return level, N, lipschitz, strides, device, axes, h, tau, pad


@torch.no_grad()
def iso_band(query, bound_min, bound_max, resolution, level, lipschitz=2.0, strides=None, max_batch=1 << 21, device=None):
    """Narrow-band threshold lattice, coarse to fine: (df [R^3] fp32 flat, +inf where never evaluated; info).

    The lattice is extract_geometry's: R = `resolution` points per axis on the box [bound_min, bound_max], coordinates from
    axis_tables (the dense sweep's torch.linspace tables, read by the kernels, so the points are that sweep's bit for bit),
    flat index (i R + j) R + k.  The level is rounded to fp32 once (mesh.iso_marching_cubes_index's rule); a non-finite
    level raises ValueError.  The levels run as udf_band's, with the block test of csrc/mesh_band.cu's table rule: a block
    is culled when min(corner value) - L r >= tau, r half its diagonal in table coordinates, tau = level + L D (iso_cull).
    If `query` is `lipschitz`-Lipschitz at the lattice points and gives a point the same bits in any batch, df equals the
    dense lattice bit for bit wherever that is below tau, every +inf stands for a value >= tau, and the threshold marching
    cubes of df at `level` (mesh.iso_mesh_band) is the dense one exactly (the argument is beside the kernels).
    `query`: any callable points [P,3] fp32 -> [P] or [P,1].  info: udf_band's keys, with the same RuntimeWarning when
    max_edge_slope exceeds `lipschitz`, plus tau (the threshold compared with, slack included), pad and spacing (the largest
    step per axis)."""
    level, N, lipschitz, strides, device, axes, h, tau, pad = _iso_setup(level, resolution, lipschitz, strides, bound_min,
                                                                         bound_max, device)
    lattice = _DenseLattice(torch.full((N ** 3,), float("inf"), device=device), N)
    info = _coarse_to_fine(lattice, lambda pts: query(pts).detach().reshape(-1).float(), N, strides, lipschitz, tau,
                           max_batch, axes=axes, spacing=h, pad=pad)
    info.update(tau=tau, pad=pad, spacing=h)
    _warn_slope(info, lipschitz, "iso_band", "a threshold mesh may miss cells")
    return lattice.df, info


@torch.no_grad()
def iso_band_sparse(query, bound_min, bound_max, resolution, level, lipschitz=2.0, strides=None, max_batch=1 << 21,
                    device=None):
    """iso_band's lattice without an R^3 array: (SparseBand, info).

    The checks, tables, block test (the table rule, reading the store), levels and RuntimeWarning are iso_band's; the store
    and its brick allocation are udf_band_sparse's (the points of strides >= c in the coarse array, the finer ones in the
    bricks meeting a kept stride-c block), and each level is emitted and evaluated in chunks of about max_batch points.  If
    `query` gives a point the same bits in any batch, SparseBand.values equals iso_band's df at every lattice point, +inf
    included, whatever the field (DESIGN.md section 1); mesh.iso_marching_cubes_sparse meshes it.  info: iso_band's keys,
    plus coarse_stride, bricks and bytes as udf_band_sparse reports them."""
    level, N, lipschitz, strides, device, axes, h, tau, pad = _iso_setup(level, resolution, lipschitz, strides, bound_min,
                                                                         bound_max, device)
    c = sparse_coarse_stride(strides)
    band = SparseBand(N, c, device)
    info = _coarse_to_fine(band, lambda pts: query(pts).detach().reshape(-1).float(), N, strides, lipschitz, tau, max_batch,
                           chunk=max_batch, axes=axes, spacing=h, pad=pad)
    band.check_stored()
    info.update(tau=tau, pad=pad, spacing=h, coarse_stride=c, bricks=band.n_bricks,
                bytes=dict(band.nbytes(), flags=max([(-(-(N - 1) // s)) ** 3 for s in strides[:-1]], default=0)))
    _warn_slope(info, lipschitz, "iso_band_sparse", "a threshold mesh may miss cells")
    return band, info


@torch.no_grad()
def get_udf_normals_grid_slow(udf_network, N=56, max_batch=1 << 20):
    """Same returns as the reference's function of this name (df_values [N,N,N], vecs [N,N,N,3], samples [N^3,7], on the
    host) -- assembled on the device, copied once."""
    device = next(udf_network.parameters()).device
    df = udf_grid(udf_network, N, max_batch)
    idx, normals = near_surface_cells(udf_network, N, df, max(max_batch // 4, 1))
    samples = torch.zeros(N ** 3, 7, device=device)
    samples[:, 0:3] = lattice_points(0, N ** 3, N, device)
    samples[:, 3] = df
    samples[idx, 4:] = normals
    samples = samples.cpu()
    return samples[:, 3].reshape(N, N, N), samples[:, 4:].reshape(N, N, N, 3), samples

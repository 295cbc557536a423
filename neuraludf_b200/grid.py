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
read."""
import math
import warnings

import torch
import torch.nn.functional as F

from neuraludf_b200 import _lib
from neuraludf_b200._lib import check, ptr


def lattice_points(head, count, N, device):
    """points `head .. head+count-1` of the N^3 lattice on [-1,1]^3 in the reference's order (x slowest, z fastest;
    extract_mesh.py:38-51), generated on the device"""
    voxel = 2.0 / (N - 1)
    idx = torch.arange(head, head + count, device=device, dtype=torch.int64)
    k = idx % N
    j = torch.div(idx, N, rounding_mode="floor") % N
    i = torch.div(torch.div(idx, N, rounding_mode="floor"), N, rounding_mode="floor") % N
    return torch.stack([i.float() * voxel - 1.0, j.float() * voxel - 1.0, k.float() * voxel - 1.0], dim=-1)


@torch.no_grad()
def udf_grid(udf_network, N, max_batch=1 << 21, lo=0, hi=None):
    """udf at the lattice points [lo, hi) (default: all N^3) as a flat device tensor -- one fused-chain launch per batch,
    no host round trips.  Slab partitioning for multi-GPU sweeps: give each rank its own [lo, hi)."""
    device = next(udf_network.parameters()).device
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
    device = next(udf_network.parameters()).device
    if df_flat is None:
        df_flat = udf_grid(udf_network, N)
    voxel = 2.0 / (N - 1)
    idx = torch.nonzero(df_flat < dist_voxels * voxel).reshape(-1) + lo
    normals = torch.empty(idx.numel(), 3, device=device)
    for head in range(0, idx.numel(), max_batch):
        sel = idx[head:head + max_batch]
        k = sel % N
        j = torch.div(sel, N, rounding_mode="floor") % N
        i = torch.div(torch.div(sel, N, rounding_mode="floor"), N, rounding_mode="floor") % N
        pts = torch.stack([i.float() * voxel - 1.0, j.float() * voxel - 1.0, k.float() * voxel - 1.0], dim=-1)
        g = udf_network.gradient(pts)[:, 0]
        g = g / (torch.linalg.norm(g, ord=2, dim=-1, keepdim=True) + 1e-5)          # exp_runner_blending.py:767-771 (func_grad)
        normals[head:head + sel.numel()] = -F.normalize(g, dim=1)                    # extract_mesh.py:93
    return idx, normals


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


def band_sublattice(N, s, device):
    """(flat indices [m^3] int64, points [m^3,3] fp32) of the stride-s lattice: 0, s, 2 s, ... and N - 1 per axis"""
    L = _lib.lib()
    m = -(-(N - 1) // s) + 1
    idx = torch.empty(m ** 3, dtype=torch.int64, device=device)
    pts = torch.empty(m ** 3, 3, device=device)
    check(L.nudf_nb_sublattice(N, s, 2.0 / (N - 1), ptr(idx), ptr(pts), _lib.stream_ptr()), "nudf_nb_sublattice")
    return idx, pts


def band_block_test(df, N, s, parent=None, parent_s=0, lipschitz=2.0, dist_voxels=2.0, flags=True):
    """(kept flags [nb^3] uint8 or None, largest edge slope) of the blocks of stride s (csrc/mesh_band.cu): candidates are every
    block, or those inside a kept block of `parent` (stride parent_s)"""
    L = _lib.lib()
    voxel = 2.0 / (N - 1)
    nb = -(-(N - 1) // s)
    out = torch.empty(nb ** 3, dtype=torch.uint8, device=df.device) if flags else None
    slope = torch.zeros(1, dtype=torch.int32, device=df.device)
    check(L.nudf_nb_block_test(ptr(df), N, s, ptr(parent), parent_s, voxel, float(lipschitz), dist_voxels * voxel, ptr(out),
                               ptr(slope), _lib.stream_ptr()), "nudf_nb_block_test")
    return out, float(slope.view(torch.float32))


def band_points(flags, N, s, t, axes=None):
    """(flat indices [M] int64, points [M,3] fp32, kept block count): the stride-t points that the kept blocks of stride s
    emit, each point once (the lowest-numbered kept block holding it), blocks ascending, each in lexicographic order;
    coordinates on [-1,1]^3, or from the three fp32 tables `axes` (iso_band)"""
    L = _lib.lib()
    st = _lib.stream_ptr()
    kept = torch.nonzero(flags).reshape(-1)
    n = kept.numel()
    counts = torch.empty(n, dtype=torch.int32, device=flags.device)
    check(L.nudf_nb_count(ptr(flags), N, s, t, ptr(kept), n, ptr(counts), st), "nudf_nb_count")
    csum = torch.cumsum(counts, 0, dtype=torch.int64)
    total = int(csum[-1]) if n else 0
    offsets = (csum - counts).contiguous()
    idx = torch.empty(total, dtype=torch.int64, device=flags.device)
    pts = torch.empty(total, 3, device=flags.device)
    if axes is None:
        check(L.nudf_nb_emit(ptr(flags), N, s, t, ptr(kept), n, ptr(offsets), 2.0 / (N - 1), ptr(idx), ptr(pts), st),
              "nudf_nb_emit")
    else:
        check(L.nudf_nb_emit_box(ptr(flags), N, s, t, ptr(kept), n, ptr(offsets), *_table_ptrs(axes, N), ptr(idx), ptr(pts),
                                 st), "nudf_nb_emit_box")
    return idx, pts, n


def _table_ptrs(axes, N):
    if len(axes) != 3 or any(x.dtype != torch.float32 or x.shape != (N,) or not x.is_contiguous() for x in axes):
        raise ValueError("axes must be three contiguous float32 tables of %d coordinates" % N)
    return [ptr(x) for x in axes]


def band_sublattice_box(axes, s):
    """band_sublattice with the coordinates of the fp32 tables `axes` (three [N] device tensors)"""
    L = _lib.lib()
    N = axes[0].numel()
    m = -(-(N - 1) // s) + 1
    idx = torch.empty(m ** 3, dtype=torch.int64, device=axes[0].device)
    pts = torch.empty(m ** 3, 3, device=axes[0].device)
    check(L.nudf_nb_sublattice_box(N, s, *_table_ptrs(axes, N), ptr(idx), ptr(pts), _lib.stream_ptr()),
          "nudf_nb_sublattice_box")
    return idx, pts


def band_block_test_box(df, axes, s, parent, parent_s, spacing, pad, lipschitz, tau, flags=True):
    """band_block_test on the lattice of the tables `axes` (csrc/mesh_band.cu's table rule): r from the block's table
    coordinates plus `pad`, `tau` as given, edge slopes over `spacing` (the largest step per axis)"""
    L = _lib.lib()
    N = axes[0].numel()
    nb = -(-(N - 1) // s)
    out = torch.empty(nb ** 3, dtype=torch.uint8, device=df.device) if flags else None
    slope = torch.zeros(1, dtype=torch.int32, device=df.device)
    check(L.nudf_nb_block_test_box(ptr(df), N, s, ptr(parent), parent_s, *_table_ptrs(axes, N), *(float(x) for x in spacing),
                                   float(pad), float(lipschitz), float(tau), ptr(out), ptr(slope), _lib.stream_ptr()),
          "nudf_nb_block_test_box")
    return out, float(slope.view(torch.float32))


def _coarse_to_fine(values, N, strides, device, max_batch, sublattice, block_test, points):
    """The level loop of udf_band and iso_band: (df [N^3] fp32 flat, +inf where never evaluated; info without
    max_edge_slope).  values(pts [P,3]) -> [P] fp32; sublattice(s) -> (idx, pts); block_test(df, s, parent, parent_s,
    flags) -> (flags or None, slope); points(flags, s, t) -> (idx, pts, kept blocks)."""
    df = torch.full((N ** 3,), float("inf"), device=device)
    info = {"strides": strides, "points": [], "kept_blocks": [], "edge_slope": []}
    events = []

    def mark():
        events.append(torch.cuda.Event(enable_timing=True))
        events[-1].record()

    def evaluate(idx, pts):
        for head in range(0, idx.numel(), max_batch):
            df[idx[head:head + max_batch]] = values(pts[head:head + max_batch])
        info["points"].append(int(idx.numel()))

    mark()
    evaluate(*sublattice(strides[0]))
    mark()
    parent = None
    for k, s in enumerate(strides):
        last = k + 1 == len(strides)
        flags, slope = block_test(df, s, parent, strides[k - 1] if k else 0, not last)
        info["edge_slope"].append(slope)
        if last:
            break
        idx, pts, n_kept = points(flags, s, strides[k + 1])
        info["kept_blocks"].append(n_kept)
        evaluate(idx, pts)
        del idx, pts
        mark()
        parent = flags
    mark()
    torch.cuda.synchronize(device)
    ms = [a.elapsed_time(b) for a, b in zip(events, events[1:])]
    # level 0: the stride-strides[0] lattice; level k: block test at strides[k-1], emission and evaluation of strides[k]
    # points; slope_ms: the slope pass over the finest level
    info["level_ms"], info["slope_ms"] = ms[:-1], ms[-1]
    info["max_edge_slope"] = max(info["edge_slope"])
    return df, info


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
    device = _device(udf_network)
    df, info = _coarse_to_fine(
        lambda pts: udf_network.udf_values(pts).reshape(-1), N, strides, device, max_batch,
        lambda s: band_sublattice(N, s, device),
        lambda df, s, parent, parent_s, flags: band_block_test(df, N, s, parent, parent_s, lipschitz, flags=flags),
        lambda flags, s, t: band_points(flags, N, s, t))
    if info["max_edge_slope"] > lipschitz:
        warnings.warn("udf_band: a lattice edge has slope %.3f > lipschitz=%.3f: the field is not %.3f-Lipschitz, so the band "
                      "may miss points with udf < 2 voxels" % (info["max_edge_slope"], lipschitz, lipschitz), RuntimeWarning,
                      stacklevel=2)
    return df, info


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
    df, info = _coarse_to_fine(
        lambda pts: query(pts).detach().reshape(-1).float(), N, strides, device, max_batch,
        lambda s: band_sublattice_box(axes, s),
        lambda df, s, parent, parent_s, flags: band_block_test_box(df, axes, s, parent, parent_s, h, pad, lipschitz, tau,
                                                                   flags),
        lambda flags, s, t: band_points(flags, N, s, t, axes))
    info.update(tau=tau, pad=pad, spacing=h)
    if info["max_edge_slope"] > lipschitz:
        warnings.warn("iso_band: a lattice edge has slope %.3f > lipschitz=%.3f: the field is not %.3f-Lipschitz, so a "
                      "threshold mesh may miss cells" % (info["max_edge_slope"], lipschitz, lipschitz), RuntimeWarning,
                      stacklevel=2)
    return df, info


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

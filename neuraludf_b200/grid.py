"""Dense UDF grid queries for mesh extraction with a device-side hand-off (SURVEY.md 8(f) rank 2, BASELINE config 5).

The reference fills an N^3 lattice by shipping every batch of points host -> device -> host and then evaluates the gradient
where `udf < 2 voxels`, again batch by batch through the host (`extract_mesh.py:18-105 get_udf_normals_grid_slow`).  Here
the lattice coordinates are generated on the device, the value sweep runs on the fused value-chain kernel, the
near-surface cells are compacted on the device and only they go through the fused value + reverse-sweep kernel; the result
is handed over as the dense distance grid plus a SPARSE list of near-surface cells (flat index + unit normal) -- 67 MB +
~7 MB at 256^3 instead of the reference's 67 MB + 201 MB dense normal grid and its ~130 blocking copies.
`get_udf_normals_grid_slow` keeps the reference's return convention for `udf_mc_lewiner` (the Cython MeshUDF marching cubes,
out of scope).  `udf_band` is the coarse-to-fine alternative to the dense sweep: it evaluates the lattice only where a
Lipschitz bound cannot rule out udf < 2 voxels (kernels in csrc/mesh_band.cu)."""
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


def band_points(flags, N, s, t):
    """(flat indices [M] int64, points [M,3] fp32, kept block count): the stride-t points that the kept blocks of stride s
    emit, each point once (the lowest-numbered kept block holding it), blocks ascending, each in lexicographic order"""
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
    check(L.nudf_nb_emit(ptr(flags), N, s, t, ptr(kept), n, ptr(offsets), 2.0 / (N - 1), ptr(idx), ptr(pts), st),
          "nudf_nb_emit")
    return idx, pts, n


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
    df = torch.full((N ** 3,), float("inf"), device=device)
    info = {"strides": strides, "points": [], "kept_blocks": [], "edge_slope": []}
    events = []

    def mark():
        events.append(torch.cuda.Event(enable_timing=True))
        events[-1].record()

    def evaluate(idx, pts):
        for head in range(0, idx.numel(), max_batch):
            df[idx[head:head + max_batch]] = udf_network.udf_values(pts[head:head + max_batch]).reshape(-1)
        info["points"].append(int(idx.numel()))

    mark()
    evaluate(*band_sublattice(N, strides[0], device))
    mark()
    parent = None
    for k, s in enumerate(strides):
        last = k + 1 == len(strides)
        flags, slope = band_block_test(df, N, s, parent, strides[k - 1] if k else 0, lipschitz, flags=not last)
        info["edge_slope"].append(slope)
        if last:
            break
        idx, pts, n_kept = band_points(flags, N, s, strides[k + 1])
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
    if info["max_edge_slope"] > lipschitz:
        warnings.warn("udf_band: a lattice edge has slope %.3f > lipschitz=%.3f: the field is not %.3f-Lipschitz, so the band "
                      "may miss points with udf < 2 voxels" % (info["max_edge_slope"], lipschitz, lipschitz), RuntimeWarning,
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

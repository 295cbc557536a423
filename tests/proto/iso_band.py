"""NumPy restatement of the narrow-band kernels' table form (csrc/mesh_band.cu: nudf_nb_*_box) and of grid.iso_band's
level chain: the lattice of three fp32 axis tables on any box, the fp64 block test of the table spacing rule (same operation
order and slack as the kernel and grid.iso_cull), and point emission (udf_band.emit's order, coordinates from the tables)."""
import math

import numpy as np

from tests.proto import udf_band as B


def table_spacing(axes):
    """grid.table_spacing: (h, e) per axis, fp64 from the fp32 tables"""
    h, e = [], []
    for x in axes:
        x = np.asarray(x, np.float32).astype(np.float64)
        h.append(float(np.abs(x[1:] - x[:-1]).max()))
        up = (np.maximum.accumulate(x) - x).max()
        down = (x - np.minimum.accumulate(x)).max()
        e.append(float(min(up, down)))
    return h, e


def iso_cull(level, lipschitz, h, e):
    """grid.iso_cull: (tau with slack, pad)"""
    d = math.sqrt(h[0] * h[0] + h[1] * h[1] + h[2] * h[2])
    ld = lipschitz * d
    return (level + ld) + 1e-6 * (abs(level) + ld), 1.000001 * math.sqrt(e[0] * e[0] + e[1] * e[1] + e[2] * e[2])


def points(axes, idx):
    """fp32 [P,3] lattice points of the flat indices"""
    N = len(axes[0])
    return np.stack([np.asarray(axes[0], np.float32)[idx // (N * N)], np.asarray(axes[1], np.float32)[(idx // N) % N],
                     np.asarray(axes[2], np.float32)[idx % N]], 1)


def lattice(axes):
    """the whole lattice [N^3,3] fp32 in flat order (extract_geometry's cartesian product)"""
    N = len(axes[0])
    return points(axes, np.arange(N ** 3, dtype=np.int64))


def block_test(df, axes, s, parent=None, parent_s=0, spacing=None, pad=0.0, lipschitz=2.0, tau=0.0):
    """(kept flags [nb^3] uint8, largest edge slope as fp32) of the blocks of stride s; df: fp32 [N^3]"""
    ax = [np.asarray(x, np.float32).astype(np.float64) for x in axes]
    N = len(ax[0])
    nb, lo, hi = B._blocks(N, s)
    bx, by, bz = (a.reshape(-1) for a in np.meshgrid(np.arange(nb), np.arange(nb), np.arange(nb), indexing="ij"))
    cand = np.ones(nb ** 3, bool)
    if parent is not None:
        pnb = -(-(N - 1) // parent_s)
        cand = parent[((lo[bx] // parent_s) * pnb + lo[by] // parent_s) * pnb + lo[bz] // parent_s] != 0
    b = np.nonzero(cand)[0]
    x0, y0, z0 = lo[bx[b]], lo[by[b]], lo[bz[b]]
    ex, ey, ez = hi[bx[b]] - x0, hi[by[b]] - y0, hi[bz[b]] - z0
    u = np.stack([df[((x0 + ((c >> 2) & 1) * ex) * N + (y0 + ((c >> 1) & 1) * ey)) * N + z0 + (c & 1) * ez]
                  for c in range(8)], 1)
    nan = np.isnan(u).any(1)
    mn = np.where(nan, 0.0, np.nanmin(np.where(np.isnan(u), np.inf, u), 1)).astype(np.float64)
    dx, dy, dz = (np.abs(ax[a][o + e] - ax[a][o]) for a, o, e in ((0, x0, ex), (1, y0, ey), (2, z0, ez)))
    rr = (0.5 * np.sqrt(dx * dx + dy * dy + dz * dz)) * 1.000001 + pad
    bound = mn - lipschitz * rr
    keep = nan | ~(bound >= tau)
    flags = np.zeros(nb ** 3, np.uint8)
    flags[b] = keep
    slope = np.float32(0.0)
    e = [ex, ey, ez]
    for c in range(8):
        for a in range(3):
            bit = 4 >> a
            if c & bit:
                continue
            a0, a1 = u[:, c], u[:, c | bit]
            ok = np.isfinite(a0) & np.isfinite(a1)
            if ok.any():
                with np.errstate(invalid="ignore", divide="ignore"):      # a zero step: 0 / 0 is NaN, which fmaxf skips
                    sl = (np.abs(a1[ok].astype(np.float64) - a0[ok].astype(np.float64))
                          / (e[a][ok].astype(np.float64) * spacing[a])).astype(np.float32)
                sl = sl[~np.isnan(sl)]
                if sl.size:
                    slope = max(slope, sl.max())
    return flags, float(slope)


def band(values, axes, strides, level, lipschitz=2.0):
    """the level chain of grid.iso_band: (df [N^3] fp32 with +inf where never evaluated, per-level emitted indices,
    per-level kept flags, tau).  values(flat indices) -> fp32 values at those lattice points; level: already fp32"""
    N = len(axes[0])
    h, e = table_spacing(axes)
    tau, pad = iso_cull(level, lipschitz, h, e)
    df = np.full(N ** 3, np.inf, np.float32)
    idx = B.sublattice(N, strides[0])
    df[idx] = values(idx)
    levels, flags_all = [idx], []
    parent = None
    for k, s in enumerate(strides[:-1]):
        flags, _ = block_test(df, axes, s, parent, strides[k - 1] if k else 0, h, pad, lipschitz, tau)
        idx = B.emit(flags, N, s, strides[k + 1])
        df[idx] = values(idx)
        levels.append(idx)
        flags_all.append(flags)
        parent = flags
    return df, levels, flags_all, tau

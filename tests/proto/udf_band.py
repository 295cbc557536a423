"""NumPy restatement of the narrow-band lattice kernels (csrc/mesh_band.cu) and of grid.udf_band's level chain: the stride-s
sub-lattice, the fp64 block test (same operation order and slack as the kernel), and point emission with the
lowest-numbered-kept-block ownership rule, in the kernels' output order."""
import numpy as np


def exact_udf(name, p, xp=np):
    """udf of the mesh fixtures' analytic surfaces (tests/proto/mesh_cases.py), exactly 1-Lipschitz everywhere.  mesh_cases'
    closest-point form gives 0 at the sphere's centre and on the cylinder's axis (its |p| guard), which lattices with an
    odd N sample; the culling rule assumes a Lipschitz field, so the band tests use the distances themselves.  xp: numpy or
    torch, p [P,3] fp64."""
    if name == "sphere":
        return xp.abs(xp.sqrt((p * p).sum(1)) - 0.5)
    if name == "patch":
        dx = xp.clip(xp.abs(p[:, 0]) - 0.5, 0.0, None)
        dy = xp.clip(xp.abs(p[:, 1]) - 0.5, 0.0, None)
        return xp.sqrt(dx * dx + dy * dy + (p[:, 2] - 0.1) ** 2)
    if name == "plane":
        return xp.abs(p[:, 2])
    if name == "cylinder":
        dr = xp.sqrt(p[:, 0] * p[:, 0] + p[:, 1] * p[:, 1]) - 0.4
        dz = xp.clip(xp.abs(p[:, 2]) - 0.5, 0.0, None)
        return xp.sqrt(dr * dr + dz * dz)
    raise KeyError(name)


def axis_coords(N, s):
    return np.minimum(np.arange(-(-(N - 1) // s) + 1, dtype=np.int64) * s, N - 1)


def sublattice(N, s):
    c = axis_coords(N, s)
    x, y, z = np.meshgrid(c, c, c, indexing="ij")
    return ((x * N + y) * N + z).reshape(-1)


def _blocks(N, s):
    nb = -(-(N - 1) // s)
    lo = np.arange(nb, dtype=np.int64) * s
    return nb, lo, np.minimum(lo + s, N - 1)


def block_test(df, N, s, parent=None, parent_s=0, lipschitz=2.0, dist_voxels=2.0):
    """(kept flags [nb^3] uint8, largest edge slope as fp32) of the blocks of stride s; df: fp32 [N^3]"""
    voxel = 2.0 / (N - 1)
    tau = dist_voxels * voxel
    nb, lo, hi = _blocks(N, s)
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
    r = 0.5 * np.sqrt((ex * ex + ey * ey + ez * ez).astype(np.float64)) * voxel
    rr = r * 1.000001 + 1e-6
    bound = mn - lipschitz * rr
    keep = nan | ~(bound >= tau * 1.000001)
    flags = np.zeros(nb ** 3, np.uint8)
    flags[b] = keep
    slope = np.float32(0.0)
    e = [ex, ey, ez]
    for c in range(8):
        for ax in range(3):
            bit = 4 >> ax
            if c & bit:
                continue
            a0, a1 = u[:, c], u[:, c | bit]
            ok = np.isfinite(a0) & np.isfinite(a1)
            if ok.any():
                sl = (np.abs(a1[ok].astype(np.float64) - a0[ok].astype(np.float64)) / (e[ax][ok] * voxel)).astype(np.float32)
                slope = max(slope, sl.max())
    return flags, float(slope)


def emit(flags, N, s, t):
    """flat indices of the stride-t points the kept blocks of stride s emit, in the kernels' order"""
    nb, lo, hi = _blocks(N, s)
    kept = np.nonzero(flags)[0]
    b = np.stack([kept // (nb * nb), (kept // nb) % nb, kept % nb], 1)
    k = s // t + 1
    j = np.stack([a.reshape(-1) for a in np.meshgrid(np.arange(k), np.arange(k), np.arange(k), indexing="ij")], 1)
    L = lo[b]                                        # [K, 3]
    H = hi[b]
    m = (H - L + t - 1) // t + 1
    J = np.broadcast_to(j[None], (len(kept), len(j), 3))
    valid = (J < m[:, None, :]).all(2)
    cls = np.where(J == 0, -1, np.where(J == m[:, None, :] - 1, 1, 0))
    valid &= ~(cls != 0).all(2)
    owned = np.ones(valid.shape, bool)
    for d in range(1, 27):
        dd = np.array([d // 9 - 1, (d // 3) % 3 - 1, d % 3 - 1])
        if not dd.any():
            continue
        ok = ((dd[None, None] == 0) | (dd[None, None] == cls)).all(2)
        q = b[:, None, :] + dd[None, None]
        ok &= ((q >= 0) & (q < nb)).all(2)
        qb = (q[..., 0] * nb + q[..., 1]) * nb + q[..., 2]
        qb = np.where(ok, qb, 0)
        owned &= ~(ok & (qb < kept[:, None]) & (flags[qb] != 0))
    P = np.minimum(L[:, None, :] + J * t, H[:, None, :])
    sel = valid & owned
    return ((P[..., 0] * N + P[..., 1]) * N + P[..., 2])[sel]


def band(values, N, strides, lipschitz=2.0):
    """the level chain of grid.udf_band: (df [N^3] fp32 with +inf where never evaluated, per-level emitted indices,
    per-level kept flags).  values(flat indices) -> fp32 udf at those lattice points"""
    df = np.full(N ** 3, np.inf, np.float32)
    idx = sublattice(N, strides[0])
    df[idx] = values(idx)
    levels, flags_all = [idx], []
    parent = None
    for k, s in enumerate(strides[:-1]):
        flags, _ = block_test(df, N, s, parent, strides[k - 1] if k else 0, lipschitz)
        idx = emit(flags, N, s, strides[k + 1])
        df[idx] = values(idx)
        levels.append(idx)
        flags_all.append(flags)
        parent = flags
    return df, levels, flags_all

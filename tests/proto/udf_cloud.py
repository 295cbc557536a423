"""NumPy restatement of the surface point cloud (neuraludf_b200/cloud.py, csrc/udf_cloud.cu, DESIGN.md section 1): the
projection step, the filter, the densify hash and jitter in fp32 with one rounding per operation, the dense-lattice seeds,
and the whole pipeline; plus analytic test fields with their exact udf and gradient (written with explicit operations, so
that NumPy and torch on the device give the same fp64 bits) and samples of their surfaces."""
import numpy as np

M32 = 0xFFFFFFFF
MAX_ROUNDS = 4


def mix32(x):
    """lowbias32 (udf_cloud.cu's mix32), on uint64 arrays holding uint32 values"""
    x = np.asarray(x, np.uint64) & M32
    x ^= x >> np.uint64(16)
    x = (x * np.uint64(0x7FEB352D)) & M32
    x ^= x >> np.uint64(15)
    x = (x * np.uint64(0x846CA68B)) & M32
    x ^= x >> np.uint64(16)
    return x


def cloud_hash(seed, r, i, k):
    """hash(seed, r, i, k) = mix(mix(seed + 0x9e3779b9 (4 r + k)) ^ i), all mod 2^32"""
    a = mix32((int(seed) + 0x9E3779B9 * (4 * int(r) + int(k))) & M32)
    return mix32(a ^ (np.asarray(i, np.uint64) & M32))


def lattice_points(idx, N):
    """fp32 coordinates fl(fl(i fl32(voxel)) - 1) of the flat lattice indices idx (grid._index_points)"""
    idx = np.asarray(idx, np.int64)
    v = np.float32(2.0 / (N - 1))
    ijk = np.stack([idx // (N * N), (idx // N) % N, idx % N], 1).astype(np.float32)
    return ijk * v - np.float32(1.0)


def seeds(values, N, dist_voxels=2.0):
    """(flat indices, fp32 points) of every lattice point with udf < fp32(dist_voxels voxel), ascending: what the sparse band
    selects when the field is Lipschitz.  values(points fp32 [P,3]) -> fp32 [P]"""
    idx = np.arange(N ** 3, dtype=np.int64)
    u = values(lattice_points(idx, N))
    idx = idx[u < np.float32(dist_voxels * (2.0 / (N - 1)))]
    return idx, lattice_points(idx, N)


def step(p, u, g):
    """(survivors [S,3] fp32 in order, keep mask): q = p - (u / n) g, n = sqrt((gx gx + gy gy) + gz gz)"""
    p, u, g = (np.asarray(a, np.float32) for a in (p, u, g))
    with np.errstate(all="ignore"):
        n = np.sqrt((g[:, 0] * g[:, 0] + g[:, 1] * g[:, 1]) + g[:, 2] * g[:, 2])
        s = u / n
        q = p - s[:, None] * g
    keep = np.isfinite(u) & np.isfinite(g).all(1) & (n != 0) & ((q >= -1) & (q <= 1)).all(1)
    return q[keep], keep


def filter_points(p, u, thr):
    u = np.asarray(u, np.float32)
    return np.asarray(p, np.float32)[u < np.float32(thr)]


def resample(pool, m, seed, r, voxel):
    """m jittered copies of points of pool (nudf_uc_resample)"""
    pool = np.asarray(pool, np.float32)
    i = np.arange(m, dtype=np.uint64)
    c = (cloud_hash(seed, r, i, 0) % np.uint64(len(pool))).astype(np.int64)
    out = np.empty((m, 3), np.float32)
    v = np.float32(voxel)
    for a in range(3):
        t = (cloud_hash(seed, r, i, 1 + a) >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)
        out[:, a] = pool[c, a] + (t - np.float32(0.5)) * v
    return out


def project(field, p, steps):
    counts = []
    for _ in range(steps):
        p, _ = step(p, *field.value_gradient(p))
        counts.append(len(p))
    return p, counts


def point_cloud(field, N, n_points, steps=5, ratio=1.0, seed=0):
    """cloud.udf_point_cloud restated: (points fp32 [M,3], info with seeds, steps, filtered, rounds, rounds_used, points,
    truncated).  field: values(p) and value_gradient(p) -> (u, g), fp32, per point"""
    voxel = 2.0 / (N - 1)
    thr = np.float32(ratio * voxel)
    _, p = seeds(field.values, N)
    n_seeds = len(p)
    p, counts = project(field, p, steps)
    pool = filter_points(p, field.values(p), thr)
    kept, n_kept, rounds = [pool], len(pool), []
    while n_kept < n_points and len(pool) and len(rounds) < MAX_ROUNDS:
        m = n_points - n_kept
        new, s = project(field, resample(pool, m, seed, len(rounds), voxel), steps)
        new = filter_points(new, field.values(new), thr)
        rounds.append(dict(drawn=m, steps=s, kept=len(new)))
        kept.append(new)
        n_kept += len(new)
    out = np.concatenate(kept)[:n_points]
    return out, dict(seeds=n_seeds, steps=counts, filtered=len(pool), rounds=rounds, rounds_used=len(rounds),
                     points=len(out), truncated=max(n_kept - n_points, 0))


# ---- analytic fields ------------------------------------------------------------------------------------------------------
def _sign(x, xp):
    one = x * 0.0 + 1.0                     # an array of x's dtype (torch.where of two scalars would give fp32)
    return xp.where(x < 0, -one, one)


def udf_grad(name, p, xp=np):
    """(udf, gradient) fp64 of the analytic surfaces of tests/proto/mesh_cases.py at fp64 points p [P,3], with explicit
    operations only.  The gradient is (p - closest point) / udf; on the surface (udf 0) a unit normal.  xp: numpy or torch."""
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    zero = x * 0.0
    if name == "sphere":
        r = xp.sqrt((x * x + y * y) + z * z)
        s = _sign(r - 0.5, xp)
        return xp.abs(r - 0.5), xp.stack([s * (x / r), s * (y / r), s * (z / r)], 1)
    if name == "plane":
        return xp.abs(z), xp.stack([zero, zero, _sign(z, xp)], 1)
    if name == "patch":
        dx = xp.clip(xp.abs(x) - 0.5, 0.0, None) * _sign(x, xp)
        dy = xp.clip(xp.abs(y) - 0.5, 0.0, None) * _sign(y, xp)
        dz = z - 0.1
        u = xp.sqrt((dx * dx + dy * dy) + dz * dz)
        on = u == 0
        d = xp.where(on, 1.0, u)
        return u, xp.stack([xp.where(on, 0.0, dx / d), xp.where(on, 0.0, dy / d), xp.where(on, 1.0, dz / d)], 1)
    if name == "cylinder":
        rho = xp.sqrt(x * x + y * y)
        dr = rho - 0.4
        dz = xp.clip(xp.abs(z) - 0.5, 0.0, None) * _sign(z, xp)
        u = xp.sqrt(dr * dr + dz * dz)
        on = u == 0
        d = xp.where(on, 1.0, u)
        ex, ey = x / rho, y / rho
        return u, xp.stack([xp.where(on, ex, (dr * ex) / d), xp.where(on, ey, (dr * ey) / d), xp.where(on, 0.0, dz / d)], 1)
    raise KeyError(name)


CASES = {"sphere": 64, "patch": 64, "plane": 65, "cylinder": 64}        # the mesh fixtures' lattices


class Analytic:
    """an analytic field behind the fp32 values / value_gradient interface of point_cloud (fp64, rounded once)"""

    def __init__(self, name):
        self.name = name

    def values(self, p):
        return self.value_gradient(p)[0]

    def value_gradient(self, p):
        with np.errstate(all="ignore"):         # the sphere's centre and the cylinder's axis, far from any seed
            u, g = udf_grad(self.name, np.asarray(p, np.float64))
        return u.astype(np.float32), g.astype(np.float32)


def surface_samples(name, n, seed=0):
    """n fp64 points on the analytic surface, area-uniform"""
    rng = np.random.default_rng(seed)
    if name == "sphere":
        v = rng.normal(size=(n, 3))
        return 0.5 * v / np.linalg.norm(v, axis=1, keepdims=True)
    if name == "plane":
        return np.stack([rng.uniform(-1, 1, n), rng.uniform(-1, 1, n), np.zeros(n)], 1)
    if name == "patch":
        return np.stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.5, 0.5, n), np.full(n, 0.1)], 1)
    if name == "cylinder":
        t = rng.uniform(0, 2 * np.pi, n)
        return np.stack([0.4 * np.cos(t), 0.4 * np.sin(t), rng.uniform(-0.5, 0.5, n)], 1)
    raise KeyError(name)

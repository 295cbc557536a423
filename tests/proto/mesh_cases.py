"""Analytic UDF test fields of the mesh fixtures (oracle/make_golden_mesh.py) and their checks: the lattice values, the unit
vectors towards the surface, and the exact udf at arbitrary points (the vertex filter of extract_mesh.py:205-214)."""
import numpy as np


def lattice(N):
    x = np.linspace(-1.0, 1.0, N)
    return np.stack(np.meshgrid(x, x, x, indexing="ij"), -1).reshape(-1, 3)        # float64, x slowest


def _closest_sphere(p, r=0.5):
    n = np.linalg.norm(p, axis=1, keepdims=True)
    return p / np.maximum(n, 1e-12) * r


def _closest_patch(p, z0=0.1, h=0.5):
    c = p.copy()
    c[:, 0] = np.clip(p[:, 0], -h, h)
    c[:, 1] = np.clip(p[:, 1], -h, h)
    c[:, 2] = z0
    return c


def _closest_plane(p):
    c = p.copy()
    c[:, 2] = 0.0
    return c


def _closest_cylinder(p, r=0.4, h=0.5):
    """open cylinder (no caps) of radius r around the z axis, |z| <= h"""
    c = p.copy()
    rho = np.linalg.norm(p[:, :2], axis=1, keepdims=True)
    c[:, :2] = p[:, :2] / np.maximum(rho, 1e-12) * r
    c[:, 2] = np.clip(p[:, 2], -h, h)
    return c


CASES = {                               # name: (closest-point function, N, surface area)
    "sphere": (_closest_sphere, 64, 4 * np.pi * 0.25),
    "patch": (_closest_patch, 64, 1.0),
    "plane": (_closest_plane, 65, 4.0),
    "cylinder": (_closest_cylinder, 64, 2 * np.pi * 0.4 * 1.0),
}


def udf(name, p):
    return np.linalg.norm(CASES[name][0](p) - p, axis=1)


def field(name):
    """(df [N^3] fp32, normals [N^3,3] fp32 towards the surface (zero on it), N)"""
    fn, N, _ = CASES[name]
    p = lattice(N)
    v = fn(p) - p
    d = np.linalg.norm(v, axis=1)
    nrm = np.where(d[:, None] > 0, v / np.maximum(d, 1e-300)[:, None], 0.0)
    return d.astype(np.float32), nrm.astype(np.float32), N


def vertex_filter(verts_world, faces, vd, N, ratio=1.0):
    """faces whose vertices all have udf < voxel * ratio (extract_mesh.py:213-214)"""
    voxel = 2.0 / (N - 1)
    return faces[np.max(vd[faces], axis=1) < voxel * ratio]


def mesh_stats(verts, faces):
    """boundary edges, non-manifold edges, edges used twice in the same direction, Euler characteristic, area"""
    f = np.asarray(faces, np.int64)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    _, c = np.unique(np.sort(e, 1), axis=0, return_counts=True)
    _, cd = np.unique(e, axis=0, return_counts=True)
    used = np.unique(f)
    v = np.asarray(verts, np.float64)
    area = 0.5 * np.linalg.norm(np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]), axis=1).sum()
    return {"boundary": int((c == 1).sum()), "nonmanifold": int((c > 2).sum()), "same_direction": int((cd > 1).sum()),
            "euler": int(len(used) - len(c) + len(f)), "area": float(area)}


def sample_surface(verts, faces, n, seed=0):
    rng = np.random.default_rng(seed)
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64)
    a = 0.5 * np.linalg.norm(np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]), axis=1)
    k = rng.choice(len(f), size=n, p=a / a.sum())
    r1, r2 = rng.random(n), rng.random(n)
    s = np.sqrt(r1)
    return (1 - s)[:, None] * v[f[k, 0]] + (s * (1 - r2))[:, None] * v[f[k, 1]] + (s * r2)[:, None] * v[f[k, 2]]


def chamfer(va, fa, vb, fb, n=20000):
    """symmetric Chamfer distance (mean of the two mean nearest-neighbour distances) between surface samples"""
    from scipy.spatial import cKDTree
    a, b = sample_surface(va, fa, n, 1), sample_surface(vb, fb, n, 2)
    return 0.5 * (cKDTree(b).query(a)[0].mean() + cKDTree(a).query(b)[0].mean())

"""NumPy restatement of get_mesh_udf_fast's gradient branch (extract_mesh.py:267-304) as csrc/mesh_grad.cu computes it:
the vertex normals, the probe points, the refined vertices, the next indices, and when the shadow raises.  Same operation
order as the kernels; fp32 steps rounded one by one."""
import numpy as np


def _norm(x):
    return np.sqrt((x[..., 0] * x[..., 0] + x[..., 1] * x[..., 1]) + x[..., 2] * x[..., 2])


def _dot(a, b):
    return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def vertex_normals(verts, faces):
    """fp32 [V,3]: per face the unit normal of (v1 - v0) x (v2 - v0) (divided by max(|c|, 1e-300)) times the angle at each
    corner, summed per vertex in (corner, face) order from 0, divided by max(|sum|, 1e-300), rounded to fp32"""
    v = np.asarray(verts, np.float64).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    n = np.zeros((len(v), 3))
    if len(f):
        p = v[f]
        a, b = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
        c = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                      a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
        fn = c / np.maximum(_norm(c), 1e-300)[:, None]
        for k in range(3):
            u, w = p[:, (k + 1) % 3] - p[:, k], p[:, (k + 2) % 3] - p[:, k]
            cosv = _dot(u, w) / np.maximum(_norm(u) * _norm(w), 1e-300)
            np.add.at(n, f[:, k], fn * np.arccos(np.clip(cosv, -1, 1))[:, None])
    return (n / np.maximum(_norm(n), 1e-300)[:, None]).astype(np.float32)


def probes(verts32, normals, eps):
    """(v + fl(eps n), v - fl(eps n)), fp32"""
    e = np.float32(eps)
    o = e * normals
    return verts32 + o, verts32 - o


def refine(verts32, normals, s1, s2, eps):
    """new_verts = (v - (eps s1) n) + (eps s2) n in fp32, each step rounded"""
    e = np.float32(eps)
    s1 = np.asarray(s1, np.float32).reshape(-1, 1)
    s2 = np.asarray(s2, np.float32).reshape(-1, 1)
    with np.errstate(invalid="ignore", over="ignore"):
        return (verts32 - (e * s1) * normals) + (e * s2) * normals


def next_indices(new_verts, N):
    """int64 [7V]: trunc((x + 1) / fl32(2 / (N - 1))) per axis, the flat index and its six clamped neighbours, block-major
    (+x, +y, +z, -x, -y, -z)"""
    voxel = np.float32(2.0 / (N - 1))
    with np.errstate(invalid="ignore", over="ignore"):
        q = ((np.asarray(new_verts, np.float32) - np.float32(-1.0)) / voxel).astype(np.int64)
        i, j, k = q[:, 0], q[:, 1], q[:, 2]
        hi = N - 1
        flat = lambda a, b, c: a * N * N + b * N + c  # noqa: E731
        return np.concatenate([flat(i, j, k), flat(np.minimum(i + 1, hi), j, k), flat(i, np.minimum(j + 1, hi), k),
                               flat(i, j, np.minimum(k + 1, hi)), flat(np.maximum(i - 1, 0), j, k),
                               flat(i, np.maximum(j - 1, 0), k), flat(i, j, np.maximum(k - 1, 0))])


def has_border(faces):
    """whether some edge is used by exactly one face (an empty mesh has none)"""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(f) == 0:
        return False
    e = np.sort(f[:, [0, 1, 1, 2, 2, 0]].reshape(-1, 2), axis=1)
    _, cnt = np.unique(e, axis=0, return_counts=True)
    return bool((cnt == 1).any())


def raises(faces, gradient=True, border_gradients=True, smooth_borders=True):
    """whether get_mesh_udf_fast raises IndexError on this post-processed mesh"""
    return (smooth_borders or (gradient and border_gradients)) and not has_border(faces)


def gradient_branch(verts64, faces, func, eps, N):
    """(normals fp32, new_verts fp32, next_indices int64) of the post-processed mesh; func(points fp32 [P,3]) -> [P]"""
    v32 = np.asarray(verts64, np.float64).astype(np.float32).reshape(-1, 3)
    n = vertex_normals(verts64, faces)
    p1, p2 = probes(v32, n, eps)
    nv = refine(v32, n, func(p1), func(p2), eps)
    return n, nv, next_indices(nv, N)

"""Inputs of the point-cloud evaluation cases (oracle/make_golden_eval.py stores them with the reference's outputs in
tests/golden/eval_<case>.NN.npz) and synthetic meshes for the larger tests and tools/eval_bench.py."""
import numpy as np


def uv_sphere(radius, n_lat, n_lon, center=(0., 0., 0.)):
    """(verts, faces): every latitude ring has n_lon vertices, the pole rings too, so the pole triangles have zero area
    (the protocols' area2 > 0 filter)"""
    th = np.linspace(0, np.pi, n_lat + 1)
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)
    T, P = np.meshgrid(th, ph, indexing="ij")
    v = np.stack([np.sin(T) * np.cos(P), np.sin(T) * np.sin(P), np.cos(T)], -1).reshape(-1, 3) * radius + np.asarray(center)
    f = []
    for i in range(n_lat):
        for j in range(n_lon):
            a, b = i * n_lon + j, i * n_lon + (j + 1) % n_lon
            c, d = a + n_lon, b + n_lon
            f += [(a, c, b), (b, c, d)]
    return v, np.array(f, np.int64)


def grid_patch(n, size, z=0.0, center=(0., 0.)):
    """an open square of n x n quads (2 triangles each) at height z"""
    u = np.linspace(-size / 2, size / 2, n + 1)
    X, Y = np.meshgrid(u + center[0], u + center[1], indexing="ij")
    v = np.stack([X, Y, np.full_like(X, z)], -1).reshape(-1, 3)
    f = []
    for i in range(n):
        for j in range(n):
            a, b, c, d = i * (n + 1) + j, i * (n + 1) + j + 1, (i + 1) * (n + 1) + j, (i + 1) * (n + 1) + j + 1
            f += [(a, c, b), (b, c, d)]
    return v, np.array(f, np.int64)


def open_cylinder(radius, height, n_around, n_up):
    ph = np.linspace(0, 2 * np.pi, n_around, endpoint=False)
    zs = np.linspace(-height / 2, height / 2, n_up + 1)
    Z, P = np.meshgrid(zs, ph, indexing="ij")
    v = np.stack([radius * np.cos(P), radius * np.sin(P), Z], -1).reshape(-1, 3)
    f = []
    for i in range(n_up):
        for j in range(n_around):
            a, b = i * n_around + j, i * n_around + (j + 1) % n_around
            f += [(a, a + n_around, b), (b, a + n_around, b + n_around)]
    return v, np.array(f, np.int64)


def sphere_points(rng, n, radius, center=(0., 0., 0.), noise=0.0):
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return d * (radius + noise * rng.normal(size=(n, 1))) + np.asarray(center)


def torus_points(rng, n, R, r, noise=0.0):
    u, w = rng.uniform(0, 2 * np.pi, n), rng.uniform(0, 2 * np.pi, n)
    rr = r + noise * rng.normal(size=n)
    return np.stack([(R + rr * np.cos(w)) * np.cos(u), (R + rr * np.cos(w)) * np.sin(u), rr * np.sin(w)], -1)


CASES = ["dtu_sphere", "dtu_patch", "dtu_pcd", "deepfashion"]


def case(name):
    """dict: protocol, data, faces (None: point cloud), gt, seed, params, and for DTU obs_mask / bb / res / plane"""
    rng = np.random.default_rng(CASES.index(name) + 11)
    if name == "dtu_sphere":
        # closed mesh in mm; GT partly off-surface and partly below the plane z = 0.5; an ObsMask with holes; a small patch
        # margin so that the in-bound test cuts the sphere at x < -6.3 - 1
        v, f = uv_sphere(8.0, 36, 72, center=(0.0, 0.0, 5.0))
        gt = np.concatenate([sphere_points(rng, 16000, 8.0, (0., 0., 5.), noise=0.15),
                             sphere_points(rng, 1500, 12.5, (0., 0., 5.)), sphere_points(rng, 300, 36.0, (0., 0., 5.))])
        bb = np.array([[-6.3, -9.1, -3.7], [9.3, 9.1, 13.7]])
        res = np.array([[0.7]])
        shape = tuple(int(x) for x in np.floor((bb[1] - bb[0]) / 0.7) + 1)
        obs = (rng.uniform(size=shape) > 0.15).astype(np.uint8)
        obs[:, :, :4] = 0
        return dict(protocol="dtu", data=v, faces=f, gt=gt, obs_mask=obs, bb=bb, res=res, plane=np.array([[0., 0., 1., -0.5]]),
                    seed=1, params=dict(density=0.2, patch=1.0, max_dist=20.0, vis=10.0))
    if name == "dtu_patch":
        # an open patch whose GT extends 35 mm past it: s2d >= max_dist queries
        v, f = grid_patch(12, 20.0, z=1.0)
        u = np.arange(-45.0, 45.0, 0.6)
        X, Y = np.meshgrid(u, u, indexing="ij")
        gt = np.stack([X.ravel(), Y.ravel(), 1.0 + 0.05 * rng.normal(size=X.size)], -1)
        bb = np.array([[-30.0, -30.0, -5.0], [30.0, 30.0, 5.0]])
        obs = np.ones((61, 61, 11), np.uint8)
        obs[25:32, 25:32, :] = 0
        return dict(protocol="dtu", data=v, faces=f, gt=gt, obs_mask=obs, bb=bb, res=np.array([[1.0]]),
                    plane=np.array([[1.0, 0.0, 0.0, 8.0]]), seed=2, params=dict(density=0.2, patch=60.0, max_dist=20.0, vis=10.0))
    if name == "dtu_pcd":
        pcd = torus_points(rng, 20000, 10.0, 3.0, noise=0.1)
        gt = torus_points(rng, 12000, 10.0, 3.0)
        bb = np.array([[-14.0, -14.0, -4.0], [14.0, 14.0, 4.0]])
        obs = (rng.uniform(size=(29, 29, 9)) > 0.1).astype(np.uint8)
        return dict(protocol="dtu", data=pcd, faces=None, gt=gt, obs_mask=obs, bb=bb, res=np.array([[1.0]]),
                    plane=np.array([[0.0, 0.2, 1.0, 1.0]]), seed=3, params=dict(density=0.2, patch=60.0, max_dist=20.0, vis=10.0))
    if name == "deepfashion":
        v, f = open_cylinder(0.06, 0.12, 48, 12)
        gt = np.concatenate([np.stack([0.06 * np.cos(a), 0.06 * np.sin(a), z], -1) for a, z in
                             [(rng.uniform(0, 2 * np.pi, 9000), rng.uniform(-0.08, 0.08, 9000))]]
                            + [rng.uniform(-0.3, 0.3, size=(400, 3))])
        gt[:9000, :2] *= 1 + 0.01 * rng.normal(size=(9000, 1))
        return dict(protocol="deepfashion", data=v, faces=f, gt=gt, seed=4,
                    params=dict(density=0.002, max_dist=0.1, vis=0.01))
    raise KeyError(name)

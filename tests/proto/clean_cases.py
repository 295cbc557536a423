"""Inputs of the mesh-cleaning cases (oracle/make_golden_clean.py stores the reference's outputs for them in
tests/golden/clean_<case>.NN.npz).  Everything is regenerated from seeds, the 1600 x 1200 masks included; the fixtures hold
the SHA-256 of the masks instead of their pixels.  Vertex-view projections within 1e-6 px of a half-integer are screened
out (nudged), so that the result does not depend on the order in which the projection is summed."""
import hashlib

import numpy as np

from tests.proto import eval_cases as E
from tests.proto import mesh_clean as M

H, W = 1200, 1600
SCAN = 24                           # below 83: imgs_idx=None means 49 views
TIE_EPS = 1e-6
CASES = ["sphere", "antialiased", "edges", "kernel31", "all_views"]


def look_at(center, target=(0., 0., 0.), f=1800.0, up=(0., 0., 1.)):
    """world_mat [4, 4] = K [R | -R C] of a camera at `center` looking at `target` (image y down)"""
    C = np.asarray(center, np.float64)
    z = np.asarray(target, np.float64) - C
    z /= np.linalg.norm(z)
    x = np.cross(z, up)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    K = np.array([[f, 0., W / 2 - 0.3], [0., f, H / 2 + 0.2], [0., 0., 1.]])
    P = np.eye(4)
    P[:3, :3], P[:3, 3] = K @ R, K @ (-R @ C)
    return P


def ring(n, dist=600.0, seed=0):
    rng = np.random.default_rng(seed)
    a = np.linspace(0, 2 * np.pi, n, endpoint=False) + rng.uniform(0, 0.2, n)
    el = rng.uniform(0.2, 0.7, n)
    return np.stack([look_at(dist * np.array([np.cos(t) * np.cos(e), np.sin(t) * np.cos(e), np.sin(e)])) for t, e in zip(a, el)])


def silhouette(P, center, radius, soft=None):
    """uint8 [H, W]: the sphere's silhouette, 255 inside; with soft = w a ramp 128 + (radius - d) / w (d = the distance of the
    pixel's ray from the centre), which takes every value around 128 along the rim"""
    inv = np.linalg.inv(P[:3, :3])
    cam = -inv @ P[:3, 3]
    r, c = np.mgrid[0:H, 0:W]
    d = inv @ np.stack([c.ravel(), r.ravel(), np.ones(H * W)])   # direction of the ray through pixel (r, c)
    d /= np.linalg.norm(d, axis=0)
    oc = np.asarray(center) - cam
    along = oc @ d
    dist = np.sqrt(np.maximum(oc @ oc - along ** 2, 0.0)).reshape(H, W)
    if soft is None:
        return np.where(dist <= radius, 255, 0).astype(np.uint8)
    return np.clip(np.round(128 + (radius - dist) / soft), 0, 255).astype(np.uint8)


def junk_sheets(rng, n=3):
    """floating patches around the object, as a UDF reconstruction leaves them"""
    vs, fs, off = [], [], 0
    for k in range(n):
        v, f = E.grid_patch(16, 90.0, z=0.0)
        a = rng.uniform(0, 2 * np.pi)
        Rz = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]])
        v = v @ Rz.T + np.array([140.0 * np.cos(2.1 * k), 140.0 * np.sin(2.1 * k), rng.uniform(-60, 60)])
        vs.append(v)
        fs.append(f + off)
        off += len(v)
    return np.concatenate(vs), np.concatenate(fs)


def screen(verts, mats, rng):
    """nudge vertices whose projection lies within TIE_EPS of a half-integer in some view"""
    verts = verts.copy()
    for _ in range(20):
        bad = M.half_integer_distance(verts, mats) < TIE_EPS
        if not bad.any():
            return verts
        verts[bad] += rng.normal(scale=1e-3, size=(int(bad.sum()), 3))
    raise RuntimeError("could not screen the near-tie projections")


def _sphere_scene(rng, n_views, soft=None, cam_seed=0):
    mats = ring(n_views, seed=cam_seed)
    v, f = E.uv_sphere(100.0, 40, 80, center=(0., 0., 0.))
    jv, jf = junk_sheets(rng)
    verts = np.concatenate([v, jv])
    faces = np.concatenate([f, jf + len(v)])
    verts = verts + rng.normal(scale=0.8, size=verts.shape)          # off the lattice, and partly outside the silhouette
    masks = np.stack([silhouette(P, (0., 0., 0.), 96.0, soft) for P in mats])
    return verts, faces, mats, masks


def _edges_scene(rng):
    """projection corner cases under cameras with P = [I | 0] (q = (x / z, y / z)): columns / rows -1, 0, 1, W - 1, W, W + 1,
    H + 1, the visual-hull border 49 / 50 / 51 px, vertices behind the camera, the camera centre itself (0 / 0)"""
    us = np.array([-2, -1, 0, 1, 2, 48, 49, 50, 51, 700, W - 51, W - 50, W - 49, W - 1, W, W + 1, W + 2])
    vs = np.array([-2, -1, 0, 1, 2, 48, 49, 50, 51, 500, H - 51, H - 50, H - 49, H - 1, H, H + 1, H + 2])
    U, V = np.meshgrid(us, vs, indexing="ij")
    pix = np.stack([U.ravel(), V.ravel()], -1).astype(np.float64)
    front = np.concatenate([pix - 1.0, np.ones((len(pix), 1))], 1)            # rint(q) + 1 = the listed index
    z = rng.uniform(2.0, 5.0, size=(len(pix), 1))
    behind = np.concatenate([-(pix[::7] - 1.0) * 3.0, -3.0 * np.ones((len(pix[::7]), 1))], 1)   # z' < 0, same pixels
    deep = np.concatenate([(pix - 1.0) * z, z], 1)
    verts = np.concatenate([front, deep, behind, np.zeros((2, 3)), np.array([[1e12, 5.0, 1e-9], [np.inf, 0.0, 1.0]])])
    n = len(verts)
    faces = np.stack([np.arange(n - 2), np.arange(1, n - 1), np.arange(2, n)], 1)
    mats = np.stack([np.eye(4), np.eye(4), np.eye(4)])
    masks = np.zeros((3, H, W), np.uint8)
    for k in range(3):                                     # random blobs plus solid borders in view 0
        m = rng.uniform(size=(H // 8 + 1, W // 8 + 1)) < 0.5
        masks[k] = np.kron(m, np.ones((8, 8), bool))[:H, :W] * np.uint8(200 + k)
    masks[0, :3, :], masks[0, -3:, :], masks[0, :, :3], masks[0, :, -3:] = 255, 255, 255, 255
    masks[1, :60, :], masks[1, :, :60] = 0, 0
    return verts, faces, mats, masks


def case(name):
    """dict: verts, faces, mats [V, 4, 4], masks uint8 [V, H, W], imgs_idx (None: all 49), mask_kernel, minimal_vis"""
    rng = np.random.default_rng(CASES.index(name) + 31)
    imgs_idx, kernel, vis = None, 11, 2
    if name == "sphere":
        verts, faces, mats, masks = _sphere_scene(rng, 10)
    elif name == "antialiased":
        verts, faces, mats, masks = _sphere_scene(rng, 8, soft=0.25, cam_seed=1)
        kernel = 1
    elif name == "edges":
        verts, faces, mats, masks = _edges_scene(rng)
        kernel, vis = 10, 0
    elif name == "kernel31":
        verts, faces, mats, masks = _sphere_scene(rng, 9, cam_seed=2)
        kernel = 31
    elif name == "all_views":
        verts, faces, mats, masks = _sphere_scene(rng, 49, cam_seed=3)
    else:
        raise KeyError(name)
    if imgs_idx is None and name != "all_views":
        imgs_idx = list(range(len(mats)))
    if name != "edges":
        verts = screen(verts, mats, rng)
    return dict(verts=verts, faces=faces.astype(np.int64), mats=mats, masks=masks, imgs_idx=imgs_idx, mask_kernel=kernel,
                minimal_vis=vis)


def sha256(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(a)
        h.update(str((a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    return h.hexdigest()

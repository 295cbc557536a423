"""NumPy restatement of camera visibility, orientation and colour of surface points (neuraludf_b200/paint.py,
csrc/udf_paint.cu, DESIGN.md section 1): unit normal lines, candidate ranking, the trace step, the rounds that resolve each
point's view, the orientation and the bilinear image gather, in fp32 with one rounding per operation; plus the projection
matrices as paint.camera_matrices forms them, and analytic test fields with their exact udf and gradient (explicit
operations only, so that NumPy and torch on the device give the same fp64 bits)."""
import numpy as np

f32 = np.float32


def dot3(a, b):
    """(a0 b0 + a1 b1) + a2 b2, rows of [.,3] fp32"""
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


def camera_matrices(intrinsics, poses):
    """(mats fp32 [V,12], centres fp32 [V,3]) of fp32 intrinsics [V,4,4] and c2w poses [V,4,4]: (K inv(pose))[:3] in fp64,
    rounded once; the centre is the pose's translation"""
    K = np.asarray(intrinsics, np.float32).astype(np.float64)
    pose = np.asarray(poses, np.float32).astype(np.float64)
    P = (K @ np.linalg.inv(pose))[:, :3, :]
    return P.reshape(-1, 12).astype(np.float32), np.asarray(poses, np.float32)[:, :3, 3].copy()


def normals(g):
    g = np.asarray(g, f32)
    with np.errstate(all="ignore"):
        L = np.sqrt(dot3(g, g))
        ok = np.isfinite(L) & (L != 0)
        out = np.where(ok[:, None], g / np.where(ok, L, f32(1))[:, None], f32(0))
    return out.astype(f32), int((~ok).sum())


def pixel(mats, k, p, H, W):
    """(u, w, in front and inside) of points p [P,3] in views k [P]"""
    P = np.asarray(mats, f32)[k].reshape(-1, 3, 4)
    x = [dot3(P[:, r, :3], p) + P[:, r, 3] for r in range(3)]
    with np.errstate(all="ignore"):
        u, w = x[0] / x[2], x[1] / x[2]
    ok = (x[2] > 0) & (u >= 0) & (u <= f32(W - 1)) & (w >= 0) & (w <= f32(H - 1))
    return u, w, ok


def towards(centres, k, p):
    """(v, L): the unit direction from p to centres[k] and the distance"""
    d = np.asarray(centres, f32)[k] - p
    L = np.sqrt(dot3(d, d))
    with np.errstate(all="ignore"):
        return d / L[:, None], L


def rank(p, n, mats, centres, H, W, cos_min, K):
    p, n = np.asarray(p, f32), np.asarray(n, f32)
    M, V = len(p), len(centres)
    score = np.full((M, V), -np.inf, np.float64)
    for k in range(V):
        kk = np.full(M, k)
        _, _, ok = pixel(mats, kk, p, H, W)
        v, _ = towards(centres, kk, p)
        a = np.abs(dot3(n, v))
        ok &= a >= f32(cos_min)
        score[ok, k] = a[ok]
    order = np.argsort(-score, axis=1, kind="stable")[:, :K]          # descending, ties to the lower index
    cand = np.where(np.take_along_axis(score, order, 1) > -np.inf, order, -1).astype(np.int32)
    if cand.shape[1] < K:
        cand = np.concatenate([cand, np.full((M, K - cand.shape[1]), -1, np.int32)], 1)
    return cand


def start(p, n, cand, r, view, centres, t_start):
    """round r's pairs (idx, cam, t, q)"""
    idx = np.nonzero((view < 0) & (cand[:, r] >= 0))[0]
    k = cand[idx, r]
    v, _ = towards(centres, k, p[idx])
    with np.errstate(all="ignore"):
        t = f32(t_start) / np.abs(dot3(n[idx], v))
    return idx.astype(np.int32), k.astype(np.int32), t, p[idx] + t[:, None] * v


def trace_step(p, centres, idx, cam, t, u, hit, view):
    """one step; sets view for the visible pairs and returns the active ones (idx, cam, t, q)"""
    u = np.asarray(u, f32)
    go = u >= f32(hit)
    idx, cam, t, u = idx[go], cam[go], t[go], u[go]
    v, L = towards(centres, cam, p[idx])
    t = t + u
    q = p[idx] + t[:, None] * v
    vis = (dot3(q, q) > 1) | (t >= L)
    view[idx[vis]] = cam[vis]
    a = ~vis
    return idx[a], cam[a], t[a], q[a]


def orient(p, n, view, centres):
    out = np.array(n, f32)
    s = np.nonzero(view >= 0)[0]
    if len(s):
        v, _ = towards(centres, view[s], p[s])
        flip = dot3(n[s], v) < 0
        out[s[flip]] = -out[s[flip]]
    return out


def gather(p, view, mats, images, H, W):
    p = np.asarray(p, f32)
    out = np.zeros((len(p), 3), f32)
    s = np.nonzero(view >= 0)[0]
    if not len(s):
        return out
    u, w, ok = pixel(mats, view[s], p[s], H, W)
    s, u, w = s[ok], u[ok], w[ok]
    fu, fw = np.floor(u), np.floor(w)
    a, b = (u - fu)[:, None], (w - fw)[:, None]
    x0, y0 = fu.astype(np.int64), fw.astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    img = np.asarray(images, f32)
    k = view[s]
    c00, c01, c10, c11 = img[k, y0, x0], img[k, y0, x1], img[k, y1, x0], img[k, y1, x1]
    top = c00 + a * (c01 - c00)
    bot = c10 + a * (c11 - c10)
    out[s] = top + b * (bot - top)
    return out


def surface_views(values, p, n, mats, centres, H, W, voxel, candidates=4, cos_min=0.2, start_voxels=2.0, hit=1.0,
                  max_steps=64):
    """paint.surface_views restated: (view int32 [M], oriented normals, info with no_candidate, rounds (traced, visible,
    active after each step), undecided, evaluations).  values(q fp32 [A,3]) -> fp32 [A]"""
    p, n = np.asarray(p, f32), np.asarray(n, f32)
    M = len(p)
    view = np.full(M, -1, np.int32)
    info = dict(no_candidate=0, rounds=[], undecided=0, evaluations=0)
    if M == 0 or len(centres) == 0:
        info["no_candidate"] = M
        return view, n.copy(), info
    cand = rank(p, n, mats, centres, H, W, cos_min, candidates)
    info["no_candidate"] = int((cand[:, 0] < 0).sum())
    t_start, thr = f32(start_voxels * voxel), f32(hit * voxel)
    for r in range(candidates):
        idx, cam, t, q = start(p, n, cand, r, view, centres, t_start)
        traced, active = len(idx), []
        if traced == 0:
            break
        for _ in range(max_steps):
            if len(idx) == 0:
                break
            u = values(q)
            info["evaluations"] += len(idx)
            idx, cam, t, q = trace_step(p, centres, idx, cam, t, u, thr, view)
            active.append(len(idx))
        info["undecided"] += len(idx)
        info["rounds"].append(dict(traced=traced, visible=int((view[cand[:, r] >= 0] == cand[cand[:, r] >= 0, r]).sum()),
                                   active=active))
    return view, orient(p, n, view, centres), info


# ---- analytic fields ------------------------------------------------------------------------------------------------------
def udf_grad(name, p, xp=np):
    """(udf, gradient) fp64 at fp64 points p [P,3], explicit operations only; xp: numpy or torch.
    sphere: | |p| - 0.5 |; nested: spheres of radius 0.3 and 0.6; disc: the disc z = 0, radius 0.6; occluded: that disc
    and the disc z = 0.3, radius 0.25, above its centre"""
    x, y, z = p[:, 0], p[:, 1], p[:, 2]

    def sign(a):
        one = a * 0.0 + 1.0
        return xp.where(a < 0, -one, one)

    def sphere(R):
        r = xp.sqrt((x * x + y * y) + z * z)
        s = sign(r - R)
        return xp.abs(r - R), xp.stack([s * (x / r), s * (y / r), s * (z / r)], 1)

    def disc(R, h):
        rho = xp.sqrt(x * x + y * y)
        dr = xp.clip(rho - R, 0.0, None)
        dz = z - h
        u = xp.sqrt(dr * dr + dz * dz)
        on = u == 0
        d = xp.where(on, 1.0, u)
        rr = xp.where(rho == 0, 1.0, rho)
        return u, xp.stack([xp.where(on, 0.0, (dr * (x / rr)) / d), xp.where(on, 0.0, (dr * (y / rr)) / d),
                            xp.where(on, 0.0, dz / d)], 1)

    def union(a, b):
        pick = a[0] <= b[0]
        return xp.where(pick, a[0], b[0]), xp.where(pick[:, None], a[1], b[1])

    if name == "sphere":
        return sphere(0.5)
    if name == "nested":
        return union(sphere(0.3), sphere(0.6))
    if name == "disc":
        return disc(0.6, 0.0)
    if name == "occluded":
        return union(disc(0.6, 0.0), disc(0.25, 0.3))
    raise KeyError(name)


class Analytic:
    """an analytic field behind fp32 values / value_gradient (fp64, rounded once)"""

    def __init__(self, name):
        self.name = name

    def values(self, p):
        return self.value_gradient(p)[0]

    def value_gradient(self, p):
        with np.errstate(all="ignore"):
            u, g = udf_grad(self.name, np.asarray(p, np.float64))
        return u.astype(f32), g.astype(f32)


def look_at(centre, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)):
    """c2w pose fp32 [4,4] of a pinhole camera at `centre` looking at `target` (OpenCV axes: x right, y down, z forward)"""
    c = np.asarray(centre, np.float64)
    f = np.asarray(target, np.float64) - c
    f /= np.linalg.norm(f)
    up = np.asarray(up, np.float64)
    if abs(float(np.dot(f, up))) > 0.99:
        up = np.array([0.0, 1.0, 0.0])
    r = np.cross(f, up)
    r /= np.linalg.norm(r)
    d = np.cross(f, r)
    pose = np.eye(4)
    pose[:3, 0], pose[:3, 1], pose[:3, 2], pose[:3, 3] = r, d, f, c
    return pose.astype(np.float32)


def intrinsics(H, W, focal):
    K = np.eye(4, dtype=np.float32)
    K[0, 0] = K[1, 1] = focal
    K[0, 2], K[1, 2] = (W - 1) / 2.0, (H - 1) / 2.0
    return K


def cameras(centres, H=64, W=80, focal=60.0):
    """(intrinsics [V,4,4], poses [V,4,4]) fp32 of cameras at `centres` looking at the origin"""
    poses = np.stack([look_at(c) for c in centres])
    return np.stack([intrinsics(H, W, focal)] * len(poses)), poses


def cap_centres(n, radius=2.5, max_polar=np.pi / 4, seed=0):
    """n camera centres on a spherical cap around +z (a DTU-like ring of cameras above the object)"""
    rng = np.random.default_rng(seed)
    th = np.arccos(rng.uniform(np.cos(max_polar), 1.0, n))
    ph = rng.uniform(0, 2 * np.pi, n)
    return radius * np.stack([np.sin(th) * np.cos(ph), np.sin(th) * np.sin(ph), np.cos(th)], 1)


def surface_samples(name, n, seed=0):
    """n fp32 points on the analytic surface with their exact unit normals (fp32, one sign)"""
    rng = np.random.default_rng(seed)
    if name == "sphere" or name == "nested":
        v = rng.normal(size=(n, 3))
        v /= np.linalg.norm(v, axis=1, keepdims=True)
        R = np.where(rng.uniform(size=n) < 0.5, 0.3, 0.6)[:, None] if name == "nested" else 0.5
        return (R * v).astype(f32), v.astype(f32)
    if name in ("disc", "occluded"):
        rho = 0.55 * np.sqrt(rng.uniform(size=n))
        t = rng.uniform(0, 2 * np.pi, n)
        p = np.stack([rho * np.cos(t), rho * np.sin(t), np.zeros(n)], 1)
        return p.astype(f32), np.tile(np.array([[0, 0, 1]], f32), (n, 1))
    raise KeyError(name)

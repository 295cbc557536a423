"""The NumPy restatement of camera visibility, orientation and colour (tests/proto/udf_paint.py) on analytic fields: seen
points face their camera, clear facing candidates are seen and back-facing ones occluded, enclosed and shadowed points
are unseen, open surfaces turn towards the chosen side, and the gather reproduces constant and linear images."""
import numpy as np

from tests.proto import udf_paint as P

H, W = 64, 80
N = 256
VOXEL = 2.0 / (N - 1)


def _setup(centres):
    intr, poses = P.cameras(np.asarray(centres, np.float64), H, W)
    return P.camera_matrices(intr, poses)


def _flip_some(n, seed=0):
    """normal lines with random signs: the orientation must not depend on the sign given"""
    s = np.where(np.random.default_rng(seed).uniform(size=len(n)) < 0.5, -1, 1).astype(np.float32)
    return (n * s[:, None]).astype(np.float32)


def _views(name, p, n, mats, centres, **kw):
    return P.surface_views(P.Analytic(name).values, p, n, mats, centres, H, W, VOXEL, **kw)


def test_camera_matrices_project_the_target_to_the_principal_point():
    mats, centres = _setup(P.cap_centres(5))
    u, w, ok = P.pixel(mats, np.arange(5), np.zeros((5, 3), np.float32), H, W)
    assert ok.all() and np.allclose(u, (W - 1) / 2, atol=1e-4) and np.allclose(w, (H - 1) / 2, atol=1e-4)
    assert np.array_equal(centres, np.asarray(P.cap_centres(5), np.float32))


def test_rank_order_and_ties():
    """equal |n . v| goes to the lower index; cameras behind, outside the image or too oblique are not candidates"""
    p = np.array([[0, 0, 0.5]], np.float32)
    n = np.array([[0, 0, 1]], np.float32)
    centres = [(1.5, 0, -1.0), (1.5, 0, 2.0), (0.0, 0.0, 2.5), (3.0, 0.0, 0.52)]
    mats, c = _setup(centres)
    cand = P.rank(p, n, mats, c, H, W, 0.2, 4)
    assert cand.tolist() == [[2, 0, 1, -1]]                    # camera 3 is at a grazing angle: |n . v| < 0.2
    assert P.rank(p, n, mats, c, H, W, 0.2, 2).tolist() == [[2, 0]]


def test_sphere_seen_points_face_their_camera():
    centres = P.cap_centres(16)
    mats, c = _setup(centres)
    p, n_true = P.surface_samples("sphere", 4000)
    n = _flip_some(n_true)
    view, out, info = _views("sphere", p, n, mats, c)
    seen = view >= 0
    assert seen.sum() > 1000 and (~seen).sum() > 1000             # the upper part is seen, the lower part not
    d = c[view[seen]] - p[seen]
    assert ((d * p[seen]).sum(1) > 0).all()
    assert ((out[seen] * p[seen]).sum(1) > 0).all()
    assert np.array_equal(out[~seen], n[~seen])
    # every point with a candidate that faces it clearly (the true normal . v >= cos_min + 0.05) is seen
    cand = P.rank(p, n, mats, c, H, W, 0.2, 4)
    clear = np.zeros(len(p), bool)
    for r in range(4):
        k = cand[:, r]
        ok = k >= 0
        v, _ = P.towards(c, np.maximum(k, 0), p)
        clear |= ok & ((n_true * v).sum(1) >= 0.25)
    assert clear.sum() > 1000 and seen[clear].all()
    assert info["undecided"] == 0 and info["no_candidate"] == int((cand[:, 0] < 0).sum())
    assert sum(r["visible"] for r in info["rounds"]) == int(seen.sum())


def test_back_facing_candidate_with_equal_score_is_occluded():
    """two cameras mirrored in the tangent plane: the back-facing one (index 0) wins the tie, is traced and occluded; the
    facing one is traced next and seen"""
    p = np.array([[0, 0, 0.5]], np.float32)
    n = np.array([[0, 0, -1]], np.float32)
    mats, c = _setup([(1.5, 0, -1.0), (1.5, 0, 2.0)])
    cand = P.rank(p, n, mats, c, H, W, 0.2, 4)
    assert cand[0, :2].tolist() == [0, 1]
    view, out, info = _views("sphere", p, n, mats, c)
    assert view.tolist() == [1] and out.tolist() == [[0, 0, 1]]
    assert [(r["traced"], r["visible"], r["active"][-1]) for r in info["rounds"]] == [(1, 0, 0), (1, 1, 0)]


def test_nested_spheres_inner_points_unseen():
    mats, c = _setup(P.cap_centres(16))
    p, n = P.surface_samples("nested", 4000)
    view, _, _ = _views("nested", p, n, mats, c)
    inner = np.linalg.norm(p, axis=1) < 0.45
    assert inner.sum() > 1000 and (view[inner] < 0).all()
    assert (view[~inner] >= 0).sum() > 300


def test_open_disc_turns_towards_the_chosen_side():
    mats, c = _setup([(1.5, 0.0, 2.0), (-1.5, 0.0, -2.0)])         # the nearer camera faces a point better
    p, n = P.surface_samples("disc", 3000)
    n = _flip_some(n, 3)
    view, out, _ = _views("disc", p, n, mats, c)
    assert (view >= 0).all()
    assert np.array_equal(np.sign(out[:, 2]), np.sign(c[view, 2]))
    assert (c[view, 2] > 0).sum() > 500 and (c[view, 2] < 0).sum() > 500


def test_disc_under_occluder():
    mats, c = _setup([(0.0, 0.0, 2.5)])
    p, n = P.surface_samples("occluded", 4000)
    view, out, _ = _views("occluded", p, n, mats, c)
    rho = np.linalg.norm(p[:, :2], axis=1)
    edge = 0.25 / (1.0 - 0.3 / 2.5)                          # the occluder's shadow from the camera on z = 0
    under, clear = rho < edge - 0.03, rho > edge + 0.03
    assert under.sum() > 500 and clear.sum() > 500
    assert (view[under] < 0).all() and (view[clear] == 0).all()
    assert (out[clear, 2] > 0).all()


def test_gather_constant_and_ramp_images():
    mats, c = _setup(P.cap_centres(6))
    p, n = P.surface_samples("sphere", 2000)
    view, _, _ = _views("sphere", p, n, mats, c)
    seen = view >= 0
    const = np.broadcast_to(np.array([0.25, 0.5, 0.75], np.float32), (6, H, W, 3)).copy()
    col = P.gather(p, view, mats, const, H, W)
    assert (col[seen] == const[0, 0, 0]).all() and (col[~seen] == 0).all()
    yy, xx = np.meshgrid(np.arange(H, dtype=np.float32), np.arange(W, dtype=np.float32), indexing="ij")
    ramp = np.stack([xx / W, yy / H, (xx + yy) / (W + H)], -1).astype(np.float32)
    ramp = np.broadcast_to(ramp, (6, H, W, 3)).copy()
    col = P.gather(p, view, mats, ramp, H, W)
    u, w, ok = P.pixel(mats, np.maximum(view, 0), p, H, W)
    assert ok[seen].all()
    want = np.stack([u / W, w / H, (u + w) / (W + H)], 1)
    assert np.abs(col[seen] - want[seen]).max() < 1e-5


def test_edge_cases():
    mats, c = _setup(P.cap_centres(3))
    e = np.zeros((0, 3), np.float32)
    view, out, info = _views("sphere", e, e, mats, c)
    assert view.shape == (0,) and out.shape == (0, 3)
    p, n = P.surface_samples("sphere", 50)
    view, out, info = _views("sphere", p, n, np.zeros((0, 12), np.float32), np.zeros((0, 3), np.float32))
    assert (view == -1).all() and np.array_equal(out, n) and info["no_candidate"] == 50
    nz, zero = P.normals(np.array([[0, 0, 0], [3, 0, 4], [np.nan, 0, 1], [np.inf, 0, 0]], np.float32))
    assert zero == 3 and np.array_equal(nz, np.array([[0, 0, 0], [0.6, 0, 0.8], [0, 0, 0], [0, 0, 0]], np.float32))

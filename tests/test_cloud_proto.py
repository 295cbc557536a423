"""The surface point cloud's NumPy restatement (tests/proto/udf_cloud.py) on the analytic fields: every point on the surface
to fp32 rounding (one step lands an exact UDF), coverage of the surface within a voxel, the exact count, seed
determinism, and the edge cases (no surface, dropped rows, the densify round cap)."""
import numpy as np
import pytest
from scipy.spatial import cKDTree

from tests.proto import udf_cloud as U

# fp32 coordinates are within 6e-8 per axis of the point the step computes in exact arithmetic; the step's own roundings
# add less than that again: 1e-6 is an order of magnitude of slack over the rounding
SURFACE_TOL = 1e-6


def _udf64(name, pts):
    return U.udf_grad(name, np.asarray(pts, np.float64))[0]


@pytest.mark.parametrize("steps", [1, 5])
@pytest.mark.parametrize("name", sorted(U.CASES))
def test_points_lie_on_the_surface(name, steps):
    N = U.CASES[name]
    pts, info = U.point_cloud(U.Analytic(name), N, 20000, steps=steps)
    assert info["seeds"] > 4000 and info["filtered"] == info["steps"][-1]     # an exact UDF keeps every projected point
    assert len(pts) == 20000 and info["rounds_used"] >= 1
    assert float(_udf64(name, pts).max()) < SURFACE_TOL


@pytest.mark.parametrize("name", sorted(U.CASES))
def test_coverage_within_a_voxel(name):
    N = U.CASES[name]
    h = 2.0 / (N - 1)
    pts, info = U.point_cloud(U.Analytic(name), N, 30000)
    d, _ = cKDTree(pts.astype(np.float64)).query(U.surface_samples(name, 20000))
    assert float(d.max()) < h, (name, float(d.max()) / h)


def test_count_and_truncation():
    field = U.Analytic("sphere")
    pts, info = U.point_cloud(field, 64, 5000)                 # fewer than the survivors: the first 5000, no rounds
    assert len(pts) == 5000 and info["rounds_used"] == 0 and info["truncated"] == info["filtered"] - 5000
    full, _ = U.point_cloud(field, 64, info["filtered"])
    assert np.array_equal(full[:5000], pts)
    more, info = U.point_cloud(field, 64, 3 * info["filtered"])
    assert len(more) == info["points"] == 3 * info["filtered"] and info["rounds_used"] == 1


def test_same_seed_same_bits():
    field = U.Analytic("cylinder")
    a, _ = U.point_cloud(field, 64, 25000, seed=3)
    b, _ = U.point_cloud(field, 64, 25000, seed=3)
    c, info = U.point_cloud(field, 64, 25000, seed=4)
    n = info["filtered"]
    assert a.view(np.int32).tobytes() == b.view(np.int32).tobytes()
    assert np.array_equal(a[:n], c[:n]) and not np.array_equal(a[n:], c[n:])


def test_hash_and_jitter():
    assert [int(x) for x in U.mix32(np.array([0, 1, 2, 0xDEADBEEF], np.uint64))] == [0, 1753845952, 3507691905, 3861431939]
    assert [int(x) for x in U.cloud_hash(7, 2, np.arange(3), 1)] == [965412113, 896505163, 2789485609]
    pool = np.random.default_rng(0).uniform(-0.5, 0.5, (97, 3)).astype(np.float32)
    voxel = 2.0 / 63
    out = U.resample(pool, 50000, 11, 1, voxel)
    c = (U.cloud_hash(11, 1, np.arange(50000), 0) % np.uint64(97)).astype(np.int64)
    j = out.astype(np.float64) - pool[c]
    assert np.abs(j).max() <= 0.5 * voxel * (1 + 1e-6)
    assert np.bincount(c, minlength=97).min() > 0                          # every pool point is drawn
    assert abs(float(j.mean())) < 0.01 * voxel                             # centred
    assert U.resample(pool, 10, 2 ** 32 + 11, 1, voxel).tobytes() == out[:10].tobytes()   # the seed is taken mod 2^32


class _NoSurface:
    def values(self, p):
        return np.ones(len(p), np.float32)

    def value_gradient(self, p):
        return self.values(p), np.tile(np.float32([1, 0, 0]), (len(p), 1))


def test_no_surface_gives_an_empty_cloud():
    pts, info = U.point_cloud(_NoSurface(), 33, 1000)
    assert pts.shape == (0, 3) and info["seeds"] == 0 and info["rounds_used"] == 0


def test_step_drops_bad_rows():
    nan, inf = np.float32(np.nan), np.float32(np.inf)
    p = np.float32([[0, 0, 0]] * 8 + [[0.99, 0, 0]])
    u = np.float32([0.1, nan, inf, 0.1, 0.1, 0.1, 0.0, 0.1, 0.1])
    g = np.float32([[1, 0, 0], [1, 0, 0], [1, 0, 0], [nan, 0, 0], [0, 0, 0], [1e-30, 0, 0], [0, 1, 0], [0, 3, 4],
                    [-1, 0, 0]])
    q, keep = U.step(p, u, g)
    # finite, NaN u, inf u, NaN g, zero g, |g| underflowing to 0, u = 0 (stays), |g| = 5, leaving the box at x = 1.09
    assert keep.tolist() == [True, False, False, False, False, False, True, True, False]
    assert q.tolist() == [[np.float32(-0.1), 0, 0], [0, 0, 0], [0, np.float32(-0.06), np.float32(-0.08)]]


class _HalfLost:
    """the plane z = 0, but value_gradient is NaN for every point whose fp32 x has its lowest mantissa bit set: about half
    of the jittered points are lost at every step"""

    def values(self, p):
        return np.abs(p[:, 2]).astype(np.float32)

    def value_gradient(self, p):
        u = self.values(p)
        lost = (p[:, 0].view(np.int32) & 1) == 1
        g = np.tile(np.float32([0, 0, 1]), (len(p), 1)) * np.sign(p[:, 2:3] + np.float32(1e-30))
        return np.where(lost, np.float32(np.nan), u), g


def test_round_cap_reports_a_short_cloud():
    pts, info = U.point_cloud(_HalfLost(), 33, 20000, steps=1)
    assert info["rounds_used"] == U.MAX_ROUNDS and 0 < len(pts) < 20000 and info["points"] == len(pts)
    assert all(r["kept"] < r["drawn"] for r in info["rounds"])

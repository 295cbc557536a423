"""The narrow-band culling rule (tests/proto/udf_band.py, the restatement of csrc/mesh_band.cu) on the exactly 1-Lipschitz
analytic fields of the mesh fixtures, including lattices whose blocks are cut short at the last plane: no point is
evaluated twice, every point with udf < 2 voxels is evaluated, and every point left out has udf >= 2 voxels."""
import numpy as np
import pytest

from tests.proto import mesh_cases as C
from tests.proto import udf_band as B

SCHEDULES = [[8, 4, 2, 1], [6, 3, 1], [16, 4, 1]]


def _field(name, N):
    u = B.exact_udf(name, C.lattice(N)).astype(np.float32)
    return u, (lambda idx: u[idx])


def test_exact_fields_match_the_fixture_fields_off_the_degenerate_sets():
    p = C.lattice(50)                                  # even N: no lattice point at the centre or on the axis
    for name in C.CASES:
        assert np.allclose(B.exact_udf(name, p), C.udf(name, p), rtol=0, atol=1e-12)


@pytest.mark.parametrize("N", [33, 50, 65, 129])
@pytest.mark.parametrize("name", sorted(C.CASES))
@pytest.mark.parametrize("strides", SCHEDULES, ids=lambda s: "-".join(map(str, s)))
@pytest.mark.parametrize("lipschitz", [1.0, 2.0])
def test_band_is_exact_on_lipschitz_fields(N, name, strides, lipschitz):
    u, values = _field(name, N)
    tau = np.float32(2 * 2.0 / (N - 1))
    df, levels, _ = B.band(values, N, strides, lipschitz)
    allidx = np.concatenate(levels)
    assert len(np.unique(allidx)) == len(allidx), "a point was evaluated twice"
    ev = np.isfinite(df)
    assert ev.sum() == len(allidx)
    assert np.array_equal(df[ev], u[ev])
    assert ev[u < tau].all(), "a point with udf < 2 voxels was culled"
    assert (u[~ev] >= tau).all()
    if lipschitz == 2.0 and N == 129:
        assert ev.mean() < 0.5                       # the band does cull


def test_sublattice_covers_the_last_plane():
    for N, s in [(50, 8), (33, 8), (10, 4), (2, 1), (5, 16)]:
        c = B.axis_coords(N, s)
        assert c[0] == 0 and c[-1] == N - 1 and (np.diff(c) > 0).all() and (np.diff(c)[:-1] == s).all()
        assert len(B.sublattice(N, s)) == len(c) ** 3


def test_stride_one_schedule_is_the_dense_lattice():
    u, values = _field("sphere", 17)
    df, levels, _ = B.band(values, 17, [1])
    assert np.array_equal(df, u) and len(levels) == 1


def test_nan_corner_keeps_its_block():
    N = 33
    u = np.full(N ** 3, 10.0, np.float32)
    flags, _ = B.block_test(u, N, 8)
    assert not flags.any()
    u[0] = np.nan
    flags, _ = B.block_test(u, N, 8)
    assert flags[0] == 1 and flags.sum() == 1


def test_edge_slope_is_seen():
    N = 33
    u, _ = _field("plane", N)
    _, slope = B.block_test((3.0 * u).astype(np.float32), N, 4)
    assert 2.9 < slope <= 3.0 + 1e-5


def test_default_schedule_rule():
    from neuraludf_b200 import grid
    assert grid.default_strides(17) == [1]
    assert grid.default_strides(128) == [4, 2, 1]
    assert grid.default_strides(512) == [16, 8, 4, 2, 1]
    assert grid.default_strides(1024) == [32, 16, 8, 4, 2, 1]
    for bad in ([4, 2], [4, 3, 1], [2, 2, 1], [0, 1]):
        with pytest.raises(ValueError):
            grid._check_strides(bad)

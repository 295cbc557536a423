"""The block-sparse narrow band (tests/proto/udf_sparse.py, the restatement of grid.udf_band_sparse and
csrc/mesh_sparse.cu) against the dense band of tests/proto/udf_band.py on the analytic fields of the mesh fixtures: the
store reads the dense band's value at every lattice point (+inf where that is +inf, so above 2 voxels wherever the dense
band holds +inf or a value >= 2 voxels), takes the same levels, and its near-surface scan finds the dense scan's
points.  Lattices whose last plane cuts a brick short, and N = 2049 on a small sphere cut by the lattice's corner."""
import numpy as np
import pytest

from tests.proto import mesh_cases as C
from tests.proto import udf_band as B
from tests.proto import udf_sparse as S


def _field(name, N):
    u = B.exact_udf(name, C.lattice(N)).astype(np.float32)
    return u, (lambda idx: u[idx])


@pytest.mark.parametrize("N", [33, 50, 65, 67, 130])
@pytest.mark.parametrize("name", sorted(C.CASES))
@pytest.mark.parametrize("strides", [[16, 8, 4, 2, 1], [16, 4, 1], [6, 3, 1], [4, 2, 1]], ids=lambda s: "-".join(map(str, s)))
def test_store_reads_the_dense_band(N, name, strides):
    u, values = _field(name, N)
    dense, levels, flags = B.band(values, N, strides)
    st, levels_s, flags_s = S.band_sparse(values, N, strides)
    assert all(np.array_equal(a, b) for a, b in zip(levels, levels_s))
    assert all(np.array_equal(a, b) for a, b in zip(flags, flags_s))
    got = st.lookup(np.arange(N ** 3))
    assert np.array_equal(got.view(np.uint32), dense.view(np.uint32)), "the store must give the dense band's bits"
    tau = np.float32(2 * 2.0 / (N - 1))
    assert np.isinf(got[np.isinf(dense)]).all() and (got[~(dense < tau)] >= tau).all()
    assert np.array_equal(st.below(2 * 2.0 / (N - 1)), np.nonzero(dense < 2 * 2.0 / (N - 1))[0])


def test_bricks_straddle_the_last_plane():
    for N in (67, 70, 129, 2049):                 # N - 1 = 66, 69: a partial last brick; 128, 2048: a one-plane brick
        st = S.Store(N, 8)
        last = (N - 1) // S.BRICK
        assert st.nbk == last + 1
        # positions round-trip through flat_index for every point of a corner block that reaches the last plane
        nb = -(-(N - 1) // 8)
        ax = np.arange(8 * (nb - 2), N)
        i, j, k = np.meshgrid(ax, ax, ax, indexing="ij")
        g = ((i * N + j) * N + k).reshape(-1)
        flags = np.zeros((nb, nb, nb), np.uint8)
        flags[-2:, -2:, -2:] = 1                  # the last two blocks of stride 8 per axis
        flags = flags.reshape(-1)
        st.allocate(flags, 8)
        p = st.position(g)
        assert (p >= 0).all() and len(np.unique(p)) == len(p)
        assert np.array_equal(st.flat_index(p), g)
        vals = np.arange(len(g), dtype=np.float32)
        st.store(g, vals)
        assert np.array_equal(st.lookup(g), vals)


def test_2049_small_sphere_at_the_corner():
    """N = 2049, a sphere of radius 0.02 centred near the (+1, +1, +1) corner and cut by the last planes: every lattice
    point with udf < 2 voxels reads its value, every point read as finite reads its value, and a point far away reads +inf."""
    N = 2049
    voxel = 2.0 / (N - 1)
    centre, r = np.array([0.985, 0.97, 0.99]), 0.02

    def values(idx):
        i, j, k = idx // (N * N), (idx // N) % N, idx % N
        p = np.stack([i * voxel - 1.0, j * voxel - 1.0, k * voxel - 1.0], 1)
        return np.abs(np.linalg.norm(p - centre, axis=1) - r).astype(np.float32)

    st, levels, _ = S.band_sparse(values, N, [256, 16, 1])
    assert st.c == 16 and st.nbk == 257 and len(st.keys) > 0
    lo = np.floor((centre - r - 4 * voxel + 1.0) / voxel).astype(np.int64)
    ax = [np.arange(lo[a], N) for a in range(3)]
    i, j, k = np.meshgrid(*ax, indexing="ij")
    g = ((i * N + j) * N + k).reshape(-1)
    u, got = values(g), st.lookup(g)
    tau = np.float32(2 * voxel)
    assert (got[u < tau] == u[u < tau]).all(), "a point with udf < 2 voxels was lost"
    fin = np.isfinite(got)
    assert (got[fin] == u[fin]).all() and (u[~fin] >= tau).all()
    assert np.array_equal(st.below(2 * voxel), np.sort(g[u < tau]))
    far = np.array([[1, 2, 3], [1025, 1030, 1001]])                 # off the stride-16 lattice, far from the sphere
    assert np.isinf(st.lookup((far[:, 0] * N + far[:, 1]) * N + far[:, 2])).all()
    assert sum(len(x) for x in levels) < 2e6                   # a few bricks, not the 8.6 G points of the lattice


def test_coarse_stride_rule():
    assert S.coarse_stride([64, 32, 16, 8, 4, 2, 1]) == 8
    assert S.coarse_stride([16, 4, 1]) == 16
    assert S.coarse_stride([6, 3, 1]) == 6 and S.coarse_stride([1]) == 1
    from neuraludf_b200 import grid
    for s in ([64, 32, 16, 8, 4, 2, 1], [16, 4, 1], [6, 3, 1], [1]):
        assert grid.sparse_coarse_stride(s) == S.coarse_stride(s)


def test_cli_refuses_sparse_with_dense_or_threshold(capsys):
    from neuraludf_b200 import mesh
    for extra in (["--dense"], ["--threshold", "0.005"]):
        with pytest.raises(SystemExit) as e:
            mesh.main(["--ckpt", "x.pth", "--out", "y.ply", "--sparse"] + extra)
        assert e.value.code == 2
        assert "--sparse cannot be combined" in capsys.readouterr().err

"""The block-sparse threshold lattice and the active-cell enumeration from storage positions (tests/proto/iso_sparse.py,
the restatement of grid.iso_band_sparse and csrc/mesh_udf.cu's IsoCells compaction): the store reads iso_band's df at every
lattice point, and the enumeration gives nudf_iso_active's cells of that df -- on random, analytic and non-Lipschitz
fields, NaN corners, values exactly at the level and levels nothing crosses, for small and odd sizes and several
schedules.  Also the CLI's --threshold --band --sparse rules."""
import numpy as np
import pytest
import torch

from tests.proto import iso_band as I
from tests.proto import iso_sparse as S
from tests.proto import udf_band as B

BOX = ([-1.01, -0.9, -1.01], [1.01, 1.01, 0.95])


def _tables(R):
    return [torch.linspace(float(np.float32(BOX[0][a])), float(np.float32(BOX[1][a])), R).numpy() for a in range(3)]


def _field(kind, axes, rng):
    p = I.lattice(axes).astype(np.float64)
    if kind == "random":
        return rng.uniform(-0.05, 0.6, p.shape[0]).astype(np.float32)
    if kind == "steep":                          # 40-Lipschitz: the band misses cells the dense lattice makes active
        return (40.0 * np.abs(p[:, 2] - 0.13) + 0.02 * np.sin(9 * p[:, 0])).astype(np.float32)
    return B.exact_udf(kind, p).astype(np.float32)


def _check(u, axes, strides, level):
    R = len(axes[0])
    level = float(np.float32(level))
    df, _, _, tau = I.band(lambda i: u[i], axes, strides, level)
    st, tau_s = S.band_sparse(lambda i: u[i], axes, strides, level)
    assert tau_s == tau
    g = np.arange(R ** 3, dtype=np.int64)
    assert np.array_equal(st.lookup(g).view(np.int32), df.view(np.int32))        # bit for bit, +inf and NaN included
    want = S.active_cells_scan(df, (R, R, R), level)
    assert np.array_equal(S.active_cells_store(st, level), want)
    assert np.array_equal(S.active_cells_dense(df, (R, R, R), level), want)
    assert np.array_equal(S.active_cells_dense(u, (R, R, R), level), S.active_cells_scan(u, (R, R, R), level))
    return df, want


SCHEDULES = {"16-8-4-2-1": [16, 8, 4, 2, 1], "8-1": [8, 1], "6-3-1": [6, 3, 1], "4-2-1": [4, 2, 1], "1": [1]}


@pytest.mark.parametrize("sched", sorted(SCHEDULES))
@pytest.mark.parametrize("R", [2, 3, 9, 17, 20, 27])
@pytest.mark.parametrize("kind", ["random", "sphere", "cylinder", "steep"])
def test_store_and_enumeration(kind, R, sched):
    rng = np.random.default_rng(R * 7 + len(sched))
    axes = _tables(R)
    u = _field(kind, axes, rng)
    for level in (0.005, 0.02, 0.3):
        _check(u, axes, SCHEDULES[sched], level)


@pytest.mark.parametrize("R", [9, 17, 26])
def test_nan_corners_and_values_at_the_level(R):
    rng = np.random.default_rng(R)
    axes = _tables(R)
    u = _field("sphere", axes, rng)
    level = float(np.float32(0.05))
    u[rng.choice(u.size, 12, replace=False)] = np.nan
    u[rng.choice(u.size, 40, replace=False)] = np.float32(level)                 # v == 0: the <= level side
    for strides in ([8, 4, 2, 1], [4, 1], [1]):
        df, cells = _check(u, axes, strides, level)
        assert cells.size > 0


@pytest.mark.parametrize("level", [-1.0, 5.0])
def test_levels_nothing_crosses(level):
    axes = _tables(17)
    u = _field("sphere", axes, None)
    _, cells = _check(u, axes, [8, 4, 2, 1], level)
    assert cells.size == 0


def test_non_lipschitz_field_is_still_enumerated_exactly():
    """the steep field: the band leaves out points the dense lattice needs, yet the store and the enumeration follow
    iso_band's df exactly"""
    axes = _tables(33)
    u = _field("steep", axes, None)
    level = float(np.float32(1.0))
    df, cells = _check(u, axes, [16, 8, 4, 2, 1], level)
    assert S.active_cells_scan(u, (33, 33, 33), level).size > cells.size


def _cli(args, capsys):
    from neuraludf_b200 import mesh
    with pytest.raises(SystemExit) as e:
        mesh.main(["--ckpt", "x.pth", "--out", "y.ply"] + args)
    return e.value.code, capsys.readouterr().err


def test_cli_threshold_band_sparse_rules(capsys):
    code, err = _cli(["--threshold", "0.005", "--sparse"], capsys)
    assert code == 2 and "--sparse cannot be combined with --threshold" in err
    code, err = _cli(["--threshold", "0.005", "--sparse", "--dense"], capsys)
    assert code == 2 and "--sparse cannot be combined with --dense" in err
    code, err = _cli(["--sparse", "--band"], capsys)
    assert code == 2 and "--band needs --threshold" in err
    if not torch.cuda.is_available():                # the flags pass; the run then needs a device
        with pytest.raises(SystemExit, match="CUDA"):
            from neuraludf_b200 import mesh
            mesh.main(["--ckpt", "x.pth", "--out", "y.ply", "--threshold", "0.005", "--band", "--sparse"])

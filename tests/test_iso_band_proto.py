"""The narrow-band threshold lattice (tests/proto/iso_band.py, the restatement of csrc/mesh_band.cu's table form and
grid.iso_band) on the exactly 1-Lipschitz analytic fields, on cubic and non-cubic boxes: the band equals the dense lattice
below tau and is +inf only at or above it, and the threshold marching cubes of the band is the dense one exactly.  Also: a
case that fails without the L D term, the linspace tables' monotonicity and excursion, and the CLI's --band rules."""
import numpy as np
import pytest
import torch

from tests.proto import iso_band as I
from tests.proto import iso_mc as P
from tests.proto import mesh_cases as C
from tests.proto import udf_band as B

BOXES = {"cube": ([-1.01] * 3, [1.01] * 3), "box": ([-1.01, -0.9, -1.01], [1.01, 1.01, 0.95]),
         "flat": ([-0.8, -1.0, -0.3], [0.9, 1.0, 0.35])}


def _tables(box, R):
    lo, hi = BOXES[box]
    return [torch.linspace(float(np.float32(lo[a])), float(np.float32(hi[a])), R).numpy() for a in range(3)]


def _dense(name, axes):
    return B.exact_udf(name, I.lattice(axes).astype(np.float64)).astype(np.float32)


def _level(level):
    from neuraludf_b200.mesh import _iso_level
    return _iso_level(level)


def _same_mesh(a, b, dims, level):
    va, fa, ia = P.marching_cubes(a, dims, level)
    vb, fb, ib = P.marching_cubes(b, dims, level)
    for k in ("active", "face_keys", "vertex_keys"):
        if not np.array_equal(ia[k], ib[k]):
            return False
    return np.array_equal(fa, fb) and np.array_equal(va, vb)


@pytest.mark.parametrize("level", [0.005, 0.02, 0.06, 5.0, -0.5])
@pytest.mark.parametrize("R", [33, 48])
@pytest.mark.parametrize("box", sorted(BOXES))
@pytest.mark.parametrize("name", sorted(C.CASES))
def test_band_is_exact_on_lipschitz_fields(name, box, R, level):
    from neuraludf_b200 import grid
    axes = _tables(box, R)
    u = _dense(name, axes)
    lv = _level(level)
    df, levels, _, tau = I.band(lambda i: u[i], axes, grid.default_strides(R) if R > 40 else [8, 4, 2, 1], lv)
    allidx = np.concatenate(levels)
    assert len(np.unique(allidx)) == len(allidx), "a point was evaluated twice"
    ev = np.isfinite(df)
    assert np.array_equal(df[ev], u[ev])
    assert ev[u < tau].all(), "a point below tau was culled"
    assert (u[~ev] >= tau).all()
    if level == 5.0:
        assert ev.all()                               # above every value: nothing can be culled
    if 0 < level < 0.1 and R == 48 and box != "flat":
        assert ev.mean() < 0.6                        # the band does cull
    dims = (R, R, R)
    assert _same_mesh(df, u, dims, lv)
    if level == 0.06:                                 # a shell two voxels thick: resolved at both R
        assert len(P.marching_cubes(u, dims, lv)[1]) > 50


@pytest.mark.parametrize("strides", [[6, 3, 1], [16, 4, 1], [2, 1]], ids=lambda s: "-".join(map(str, s)))
def test_other_schedules(strides):
    axes = _tables("box", 50)
    u = _dense("sphere", axes)
    lv = _level(0.02)
    df, _, _, tau = I.band(lambda i: u[i], axes, strides, lv)
    ev = np.isfinite(df)
    assert ev[u < tau].all() and (u[~ev] >= tau).all() and np.array_equal(df[ev], u[ev])
    assert _same_mesh(df, u, (50, 50, 50), lv)


def test_a_threshold_below_the_level_changes_the_mesh(monkeypatch):
    """The comparison above can fail: with tau = level - L D the band culls corners of active cells and the mesh changes.
    With tau = level + L D (iso_cull) it is exact.  tau = level alone would be exact too: every lattice cell lies inside one
    block of each stride, and a block holding a corner at or below the level is never culled (min corner - L r is a lower
    bound on every point of the block), so the L D term is a margin of one cell diagonal on top of that."""
    axes = _tables("box", 33)
    u = _dense("sphere", axes)
    lv = _level(0.02)
    df, _, _, _ = I.band(lambda i: u[i], axes, [8, 4, 2, 1], lv, lipschitz=1.0)
    assert _same_mesh(df, u, (33, 33, 33), lv)
    monkeypatch.setattr(I, "iso_cull", lambda level, lipschitz, h, e: (level - lipschitz * np.sqrt(np.dot(h, h)), 0.0))
    df, _, _, _ = I.band(lambda i: u[i], axes, [8, 4, 2, 1], lv, lipschitz=1.0)
    with np.errstate(invalid="ignore"):
        assert not _same_mesh(df, u, (33, 33, 33), lv)


@pytest.mark.parametrize("box", sorted(BOXES))
def test_linspace_tables_are_monotone_and_the_pad_covers_them(box):
    """torch.linspace's tables (fp32, computed from both ends) on the tested boxes: strictly monotone, so iso_band's
    excursion term is 0; and for any table, every coordinate of a block lies within e of its corner interval."""
    from neuraludf_b200 import grid
    for R in (2, 33, 64, 96, 97, 128, 256, 512, 1024):
        axes = _tables(box, R)
        h, e = I.table_spacing(axes)
        assert e == [0.0, 0.0, 0.0]
        assert all((np.diff(x) > 0).all() for x in axes)
        gh, ge = grid.table_spacing([torch.from_numpy(x) for x in axes])
        assert gh == h and ge == e
    x = np.array([0.0, 0.1, 0.3, 0.29, 0.4, 0.6, 0.58, 0.57, 0.8], np.float32)
    (_, e), = [[v[0] for v in I.table_spacing([x])]]
    assert e == np.float64(np.float32(0.6)) - np.float64(np.float32(0.57))
    for s in (1, 2, 3, 4):
        for lo in range(0, len(x) - 1, s):
            hi = min(lo + s, len(x) - 1)
            a, b = sorted((float(x[lo]), float(x[hi])))
            assert all(a - e <= float(v) <= b + e for v in x[lo:hi + 1])
    assert I.table_spacing([x[::-1]])[1][0] == e                  # a decreasing table: the excursion against its direction


def test_tau_and_pad():
    from neuraludf_b200 import grid
    h, e = [0.01, 0.02, 0.015], [0.0, 1e-7, 0.0]
    tau, pad = grid.iso_cull(0.005, 2.0, h, e)
    assert (tau, pad) == I.iso_cull(0.005, 2.0, h, e)
    d = np.sqrt(0.01 ** 2 + 0.02 ** 2 + 0.015 ** 2)
    assert 0.005 + 2 * d < tau < 0.005 + 2 * d + 1e-7 and 1e-7 < pad < 1.01e-7
    tau, _ = grid.iso_cull(-2 * d, 2.0, h, e)                     # level + L D == 0: the slack still lifts tau above it
    assert tau > 0


def test_argument_errors():
    from neuraludf_b200 import grid
    for bad in (np.nan, np.inf, 1e39):
        with pytest.raises(ValueError):
            grid.iso_band(lambda p: p[:, 0], [-1.0] * 3, [1.0] * 3, 16, bad)
    for bad in (0.0, -1.0, np.inf):
        with pytest.raises(ValueError):
            grid.iso_band(lambda p: p[:, 0], [-1.0] * 3, [1.0] * 3, 16, 0.1, lipschitz=bad)
    with pytest.raises(ValueError):
        grid.iso_band(lambda p: p[:, 0], [-1.0] * 3, [1.0] * 3, 1, 0.1)


def test_cli_band_rules():
    from neuraludf_b200 import mesh
    base = ["--ckpt", "none.pth", "--out", "none.ply"]
    for argv in (["--band"], ["--band", "--lipschitz", "2"], ["--band", "--dense"]):
        with pytest.raises(SystemExit) as ex:
            mesh.main(base + argv)                                  # --band without --threshold
        assert ex.value.code == 2
    for extra in (["--postprocess"], ["--dense"], ["--dist_threshold_ratio", "1"]):
        with pytest.raises(SystemExit) as ex:
            mesh.main(base + ["--threshold", "0.005", "--band"] + extra)
        assert ex.value.code == 2
    # --lipschitz is accepted with --band: parsing passes and the run stops at the device or the missing checkpoint
    with pytest.raises((SystemExit, FileNotFoundError)) as ex:
        mesh.main(base + ["--threshold", "0.005", "--band", "--lipschitz", "3"])
    assert not (isinstance(ex.value, SystemExit) and ex.value.code == 2)

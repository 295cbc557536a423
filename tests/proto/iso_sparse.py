"""NumPy restatement of the block-sparse threshold lattice (grid.iso_band_sparse) and of the active-cell enumeration
from storage positions (mesh.iso_active_cells, csrc/mesh_udf.cu IsoCells): iso_band's level chain
(tests/proto/iso_band.py) run on udf_sparse's store (tests/proto/udf_sparse.py), the table block test reading the store,
and the cells found from the stored points with v <= 0, each emitted by its lowest such corner."""
import numpy as np

from tests.proto import iso_band as I
from tests.proto import iso_mc as P
from tests.proto import udf_band as B
from tests.proto import udf_mc as M
from tests.proto import udf_sparse as U


def band_sparse(values, axes, strides, level, lipschitz=2.0):
    """iso_band's levels into a udf_sparse.Store: (store, tau).  values(flat indices) -> fp32; level: already fp32"""
    N = len(axes[0])
    h, e = I.table_spacing(axes)
    tau, pad = I.iso_cull(level, lipschitz, h, e)
    st = U.Store(N, U.coarse_stride(strides))
    idx = B.sublattice(N, strides[0])
    st.store(idx, values(idx))
    parent = None
    for k, s in enumerate(strides[:-1]):
        flags, _ = I.block_test(st, axes, s, parent, strides[k - 1] if k else 0, h, pad, lipschitz, tau)
        if s == st.c:
            st.allocate(flags, s)
        idx = B.emit(flags, N, s, strides[k + 1])
        st.store(idx, values(idx))
        parent = flags
    return st, tau


def _points(N, g):
    return g // (N * N), (g // N) % N, g % N


def owned_cells(g, value, lookup, dims, level):
    """the cells emitted by the lattice points g (flat) holding `value`: those with v <= 0 emit every active cell holding
    them of which they are the lowest corner with v <= 0 (nudf_iso_active's test on lookup(flat) values); sorted"""
    n0, n1, n2 = dims
    lv = np.float32(level)
    with np.errstate(invalid="ignore"):
        g = g[(np.asarray(value, np.float32) - lv) <= 0]
    i, j, k = g // (n1 * n2), (g // n2) % n1, g % n2
    out = []
    for q, (a, b, c) in enumerate(M.OFF):
        o = np.stack([i - a, j - b, k - c])
        ok = (o >= 0).all(0) & (o[0] < n0 - 1) & (o[1] < n1 - 1) & (o[2] < n2 - 1)
        cell = (o[0] * n1 + o[1]) * n2 + o[2]
        cell = cell[ok]
        v = np.stack([lookup(cell + (x * n1 + y) * n2 + z) for x, y, z in M.OFF]) - lv
        with np.errstate(invalid="ignore"):
            act = (v > 0).any(0) & (v <= 0).any(0) & ~np.isnan(v).any(0) & ~(v[:q] <= 0).any(0)
        out.append(cell[act])
    return np.sort(np.concatenate(out)).astype(np.int64)


def active_cells_store(st, level):
    """the enumeration on a Store: every coarse position and brick slot that holds a lattice point of its own"""
    N = st.N
    m3 = st.mc ** 3
    pos = np.arange(m3 + len(st.bricks), dtype=np.int64)
    g = st.flat_index(pos)
    i, j, k = _points(N, g)
    if len(st.bricks):                           # a slot past N - 1 wraps in the flat index: recompute its point
        q = np.maximum(pos - m3, 0)
        key, loc = st.keys[np.minimum(q // U.BRICK ** 3, len(st.keys) - 1)], q % U.BRICK ** 3
        nbk = st.nbk
        bi = (key // (nbk * nbk)) * U.BRICK + loc // (U.BRICK * U.BRICK)
        bj = ((key // nbk) % nbk) * U.BRICK + (loc // U.BRICK) % U.BRICK
        bk = (key % nbk) * U.BRICK + loc % U.BRICK
        i, j, k = (np.where(pos < m3, a, b) for a, b in ((i, bi), (j, bj), (k, bk)))
    inside = (i < N) & (j < N) & (k < N)
    g = (np.minimum(i, N - 1) * N + np.minimum(j, N - 1)) * N + np.minimum(k, N - 1)
    own = inside & (st.position(g) == pos)
    value = np.concatenate([st.coarse, st.bricks])
    return owned_cells(g[own], value[own], st.lookup, (N, N, N), level)


def active_cells_dense(df, dims, level):
    """the enumeration on a flat array (positions = flat indices)"""
    df = np.asarray(df, np.float32).reshape(-1)
    return owned_cells(np.arange(df.size, dtype=np.int64), df, lambda g: df[g], dims, level)


def active_cells_scan(df, dims, level):
    """nudf_iso_active's cells: every cell scanned"""
    return P.active_cells(P.corner_values(df, level), dims)

"""NumPy restatement of the block-sparse narrow band (grid.SparseBand, grid.udf_band_sparse, csrc/mesh_sparse.cu and the
BrickDf reader of csrc/df_access.cuh): the coarse array of the stride-c lattice, 8^3 bricks behind a dense directory, the
brick allocation from the kept stride-c blocks, and udf_band's level chain (tests/proto/udf_band.py) run on the store."""
import numpy as np

from tests.proto import udf_band as B

BRICK = 8


def coarse_stride(strides):
    big = [s for s in strides if s >= BRICK]
    return big[-1] if big else strides[0]


class Store:
    def __init__(self, N, c):
        self.N, self.c = N, c
        self.mc = -(-(N - 1) // c) + 1
        self.nbk = -(-N // BRICK)
        self.coarse = np.full(self.mc ** 3, np.inf, np.float32)
        self.dir = np.full(self.nbk ** 3, -1, np.int64)
        self.bricks = np.zeros(0, np.float32)
        self.keys = np.zeros(0, np.int64)

    def _coarse_of(self, i):
        return np.where(i == self.N - 1, self.mc - 1, np.where(i % self.c == 0, i // self.c, -1))

    def position(self, g):
        """storage positions of flat indices g: [0, mc^3) coarse, mc^3 + slot * 512 + local, -1 without a brick"""
        g = np.asarray(g, np.int64)
        N = self.N
        i, j, k = g // (N * N), (g // N) % N, g % N
        ci, cj, ck = self._coarse_of(i), self._coarse_of(j), self._coarse_of(k)
        on = (ci >= 0) & (cj >= 0) & (ck >= 0)
        slot = self.dir[((i // BRICK) * self.nbk + j // BRICK) * self.nbk + k // BRICK]
        local = ((i % BRICK) * BRICK + j % BRICK) * BRICK + k % BRICK
        brick = np.where(slot < 0, -1, self.mc ** 3 + slot * BRICK ** 3 + local)
        return np.where(on, (ci * self.mc + cj) * self.mc + ck, brick)

    def lookup(self, g):
        p = self.position(g)
        m3 = self.mc ** 3
        out = np.full(p.shape, np.inf, np.float32)
        c = (p >= 0) & (p < m3)
        out[c] = self.coarse[p[c]]
        b = p >= m3
        out[b] = self.bricks[p[b] - m3]
        return out

    def __getitem__(self, g):                   # B.block_test reads df[flat indices]
        return self.lookup(g)

    def store(self, g, vals):
        p = self.position(g)
        assert (p >= 0).all(), "a value with no storage"
        m3 = self.mc ** 3
        c = p < m3
        self.coarse[p[c]] = vals[c]
        self.bricks[p[~c] - m3] = vals[~c]

    def allocate(self, flags, s):
        """slots for every brick meeting the closed box of a kept block of stride s, ascending brick number"""
        nb, lo, hi = B._blocks(self.N, s)
        kept = np.nonzero(flags)[0]
        b = np.stack([kept // (nb * nb), (kept // nb) % nb, kept % nb], 1)
        marks = np.zeros(self.nbk ** 3, bool)
        blo, bhi = lo[b] // BRICK, hi[b] // BRICK                # [K, 3]
        span = s // BRICK + 2
        for dx in range(span):
            for dy in range(span):
                for dz in range(span):
                    q = blo + np.array([dx, dy, dz])
                    ok = (q <= bhi).all(1)
                    marks[((q[ok, 0] * self.nbk) + q[ok, 1]) * self.nbk + q[ok, 2]] = True
        self.keys = np.nonzero(marks)[0]
        self.dir[:] = -1
        self.dir[self.keys] = np.arange(len(self.keys))
        self.bricks = np.full(len(self.keys) * BRICK ** 3, np.inf, np.float32)

    def flat_index(self, pos):
        pos = np.asarray(pos, np.int64)
        m3, mc, N = self.mc ** 3, self.mc, self.N
        ci, cj, ck = pos // (mc * mc), (pos // mc) % mc, pos % mc
        q = np.maximum(pos - m3, 0)
        keys = self.keys if len(self.keys) else np.zeros(1, np.int64)
        key, l = keys[np.minimum(q // BRICK ** 3, len(keys) - 1)], q % BRICK ** 3
        nbk = self.nbk
        bi = np.where(pos < m3, np.minimum(ci * self.c, N - 1), (key // (nbk * nbk)) * BRICK + l // (BRICK * BRICK))
        bj = np.where(pos < m3, np.minimum(cj * self.c, N - 1), ((key // nbk) % nbk) * BRICK + (l // BRICK) % BRICK)
        bk = np.where(pos < m3, np.minimum(ck * self.c, N - 1), (key % nbk) * BRICK + l % BRICK)
        return (bi * N + bj) * N + bk

    def below(self, thr):
        """sorted flat indices of the stored points with value < thr (fp32 comparison), scanning coarse and bricks only"""
        pos = np.concatenate([np.nonzero(self.coarse < np.float32(thr))[0],
                              np.nonzero(self.bricks < np.float32(thr))[0] + self.mc ** 3])
        return np.sort(self.flat_index(pos))


def band_sparse(values, N, strides, lipschitz=2.0):
    """udf_band's level chain into a Store: (store, per-level emitted indices, per-level kept flags)"""
    c = coarse_stride(strides)
    st = Store(N, c)
    idx = B.sublattice(N, strides[0])
    st.store(idx, values(idx))
    levels, flags_all = [idx], []
    parent = None
    for k, s in enumerate(strides[:-1]):
        flags, _ = B.block_test(st, N, s, parent, strides[k - 1] if k else 0, lipschitz)
        if s == c:
            st.allocate(flags, s)
        idx = B.emit(flags, N, s, strides[k + 1])
        st.store(idx, values(idx))
        levels.append(idx)
        flags_all.append(flags)
        parent = flags
    return st, levels, flags_all

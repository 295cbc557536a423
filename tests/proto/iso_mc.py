"""NumPy restatement of the CUDA threshold marching cubes (nudf_iso_*, neuraludf_b200/csrc/mesh_udf.cu) -- the exact oracle of
its kernels: faces, keys and fp64 vertices must match bit for bit.

It is the MeshUDF construction of tests/proto/udf_mc.py (cell_loops, face_join_bits, loop_triangles) on the corner values
v = f32(f - f32(level)), with no pseudo-signs and no polarity:

  1. active cells: some corner with v > 0, some with v <= 0, none NaN;
  2. per cell, the crossing loops of udf_mc.cell_loops (ambiguous faces by the asymptotic decider, exact ties join the
     face's first diagonal), each triangulated by udf_mc.loop_triangles, then wound the other way: face normals (right-hand
     rule) point from the > level side into the <= level side, towards decreasing values;
  3. vertices keyed as udf_mc's (3 * corner + axis; loop centres 3 * n_points + 4 * cell_position + loop) and numbered by
     ascending key; an edge point sits at t = v_a / (v_a - v_b) from the lower corner, in fp64 from the fp32 v; a loop
     centre at the mean of its edge points, summed in canonical loop order from 0.
"""
import numpy as np

from tests.proto import udf_mc as U


def corner_values(df, level):
    """v = f32(f - f32(level)) of the flat lattice"""
    return (np.asarray(df, np.float32).reshape(-1) - np.float32(level)).astype(np.float32)


def active_cells(v, dims):
    """sorted flat indices (lower corner) of the cells with corners on both sides and no NaN corner"""
    n0, n1, n2 = dims
    g = v.reshape(n0, n1, n2)
    cor = np.stack([g[a:n0 - 1 + a, b:n1 - 1 + b, c:n2 - 1 + c] for a, b, c in U.OFF])
    with np.errstate(invalid="ignore"):
        act = (cor > 0).any(0) & (cor <= 0).any(0) & ~np.isnan(cor).any(0)
    i, j, k = np.nonzero(act)
    return (i * n1 * n2 + j * n2 + k).astype(np.int64)


def _cell(v, cell, base):
    vv = v[cell + base]
    pos_mask = sum(1 << c for c in range(8) if vv[c] > 0)
    return vv, pos_mask


def triangulate(v, dims, cells):
    """[F, 3] int64 vertex keys: cells in order, each cell's triangles in udf_mc's loop / fan order, wound descent"""
    n0, n1, n2 = dims
    base = U.corner_offsets(dims)
    centre0 = 3 * n0 * n1 * n2
    out = []
    for ci, g in enumerate(cells.tolist()):
        vv, pm = _cell(v, g, base)
        for t in U.cell_triangles(pm, U.face_join_bits(vv, pm)):
            row = []
            for e in (t[0], t[2], t[1]):
                row.append(centre0 + 4 * ci + (e - U.CENTRE) if e >= U.CENTRE
                           else 3 * (g + int(base[U.EDGE_CORNERS[e][0]])) + e // 4)
            out.append(row)
    return np.array(out, np.int64).reshape(-1, 3)


def edge_points(v, dims, keys):
    """fp64 lattice-index positions of lattice-edge keys: t = v_a / (v_a - v_b) from the lower corner"""
    n0, n1, n2 = dims
    strides = np.array([n1 * n2, n2, 1], np.int64)
    g, ax = keys // 3, keys % 3
    va = v[g].astype(np.float64)
    vb = v[g + strides[ax]].astype(np.float64)
    t = va / (va - vb)
    x = np.stack([g // (n1 * n2), (g // n2) % n1, g % n2], 1).astype(np.float64)
    x[np.arange(len(keys)), ax] = x[np.arange(len(keys)), ax] + t
    return x


def vertices(v, dims, keys, cells):
    """fp64 positions of the sorted unique keys: edge points, then loop centres"""
    n0, n1, n2 = dims
    centre0 = 3 * n0 * n1 * n2
    base = U.corner_offsets(dims)
    out = np.zeros((len(keys), 3), np.float64)
    ek = keys < centre0
    out[ek] = edge_points(v, dims, keys[ek])
    for r in np.nonzero(~ek)[0]:
        ci, li = int(keys[r] - centre0) >> 2, int(keys[r] - centre0) & 3
        g = int(cells[ci])
        vv, pm = _cell(v, g, base)
        loop, _ = U.canonical_loop(U.cell_loops(pm, U.face_join_bits(vv, pm))[li])
        pts = edge_points(v, dims, np.array([3 * (g + int(base[U.EDGE_CORNERS[e][0]])) + e // 4 for e in loop], np.int64))
        acc = np.zeros(3, np.float64)
        for p in pts:
            acc = acc + p
        out[r] = acc / np.float64(len(loop))
    return out


def marching_cubes(df, dims, level):
    """(verts [V,3] fp64 lattice-index units, faces [F,3] int64, info {active, face_keys, vertex_keys})"""
    dims = tuple(int(d) for d in dims)
    v = corner_values(df, level)
    cells = active_cells(v, dims)
    keys = triangulate(v, dims, cells)
    info = {"active": cells, "face_keys": keys}
    if len(keys) == 0:
        info["vertex_keys"] = np.zeros(0, np.int64)
        return np.zeros((0, 3), np.float64), np.zeros((0, 3), np.int64), info
    uk, inv = np.unique(keys.reshape(-1), return_inverse=True)
    info["vertex_keys"] = uk
    return vertices(v, dims, uk, cells), inv.reshape(-1, 3).astype(np.int64), info


def reference_mapping(verts, resolution, bound_min, bound_max):
    """the runner's extract_geometry mapping (udf_renderer_blending.py:60-62): fp64 vertices, fp32 bounds, b_max - b_min
    formed in fp32, then promoted"""
    b_max_np = np.asarray(bound_max, np.float32)
    b_min_np = np.asarray(bound_min, np.float32)
    return verts / (resolution - 1.0) * (b_max_np - b_min_np)[None, :] + b_min_np[None, :]


# ---------------------------------------------------------------------------------------------------------------
# analytic and seeded test fields: name -> (flat fp32 lattice, dims, level, gradient function of lattice-index points or None)
# ---------------------------------------------------------------------------------------------------------------
def _grid(dims, lo=-1.0, hi=1.0):
    axes = [np.linspace(lo, hi, n) for n in dims]
    return np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3), [(hi - lo) / (n - 1) for n in dims]


def _to_world(lo, h):
    return lambda x: lo + x * np.asarray(h)[None, :]


def case(name):
    if name == "shell":                     # |r - 0.5| at 0.05: two concentric spheres
        dims = (40, 40, 40)
        p, h = _grid(dims)
        r = np.linalg.norm(p, axis=1)
        df = np.abs(r - 0.5)

        def grad(x):
            w = _to_world(-1.0, h)(x)
            rr = np.linalg.norm(w, axis=1, keepdims=True)
            return np.sign(rr - 0.5) * w / rr
        return df.astype(np.float32), dims, 0.05, grad
    if name == "torus":
        dims = (44, 44, 30)
        p, h = _grid(dims)
        R, r0 = 0.55, 0.25

        def sdf_grad(w):
            q = np.linalg.norm(w[:, :2], axis=1)
            a = np.stack([(q - R) * w[:, 0] / q, (q - R) * w[:, 1] / q, w[:, 2]], 1)
            return a / np.linalg.norm(a, axis=1, keepdims=True)
        df = np.sqrt((np.linalg.norm(p[:, :2], axis=1) - R) ** 2 + p[:, 2] ** 2) - r0
        return df.astype(np.float32), dims, 0.0, lambda x: sdf_grad(_to_world(-1.0, h)(x))
    if name == "cut":                       # a sphere of radius 1.3 around (0.4, 0, 0): cut open by the box
        dims = (33, 29, 31)
        p, h = _grid(dims)
        c = np.array([0.4, 0.0, 0.0])
        df = np.linalg.norm(p - c, axis=1) - 1.3

        def grad(x):
            w = _to_world(-1.0, h)(x) - c
            return w / np.linalg.norm(w, axis=1, keepdims=True)
        return df.astype(np.float32), dims, 0.0, grad
    if name.startswith("random"):           # seeded uniform noise: every kind of cell, loops with centre vertices
        seed = int(name[len("random"):] or 0)
        rng = np.random.default_rng(seed)
        dims = (17, 19, 23)
        return rng.uniform(-1, 1, int(np.prod(dims))).astype(np.float32), dims, 0.1 * seed - 0.1, None
    if name == "quantised":                 # values in {-1, 0, 1} at level 0: exact v = 0 corners and decider ties
        rng = np.random.default_rng(5)
        dims = (16, 14, 15)
        return rng.integers(-1, 2, int(np.prod(dims))).astype(np.float32), dims, 0.0, None
    if name == "ties":                      # values in {-2, -1, 1, 2}: a * c == b * d on many ambiguous faces
        rng = np.random.default_rng(9)
        dims = (15, 16, 17)
        return rng.choice(np.float32([-2, -1, 1, 2]), int(np.prod(dims))).astype(np.float32), dims, 0.0, None
    if name == "min":                       # the 2 x 2 x 2 minimum: one cell, corner 7 above the level
        df = np.zeros(8, np.float32)
        df[7] = 1.0
        return df, (2, 2, 2), 0.25, lambda x: np.ones_like(x)     # the values rise towards corner 7
    raise KeyError(name)


CASES = ["shell", "torus", "cut", "random0", "random1", "random2", "random3", "quantised", "ties", "min"]

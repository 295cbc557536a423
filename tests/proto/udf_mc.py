"""NumPy restatement of the CUDA MeshUDF marching cubes (neuraludf_b200/csrc/mesh_udf.cu) -- the exact oracle of its kernels.

Same stages, same float32 operation order, same tie rules, same loop / fan order and the same welding, so the CUDA result
must match it bit for bit in topology (active cells, edge-keyed faces) and to float rounding in positions:

  1. active cells: mean of the 8 corner udf < avg_t and max <= max_t (the reference's thresholds, summed in its corner order);
  2. per-cell pseudo-signs: every corner is compared with the cell's reference corner r (largest udf, ties -> lowest corner
     id) along their displacement d = p_c - p_r: same side when the normals point away from each other along d
     (n_r.d < 0 and n_c.d > 0), else when n_r.n_c >= 0;
  3. global polarity: face-adjacent active cells agree (parity 0) or disagree (parity 1) on the shared corners with udf > 0
     (mixed evidence: no link); union-find with parity by deterministic min-root hooking; each component takes the
     polarity that makes its root cell's corner 0 positive;
  4. per cell, the crossing segments of each face (ambiguous faces: asymptotic decider, exact ties join the face's first
     diagonal), chained into loops from the lowest local edge; each loop triangulated with no chord lying in a cube face
     (loop_triangles), or fanned around a centre vertex of its own when no such triangulation exists;
  5. vertices welded by the global edge key 3 * corner_index + axis, placed at t = u_a / (u_a + u_b) from the lower corner;
     loop centres keyed 3 * n_points + 4 * cell_position + loop, at the mean of the loop's edge points.

Corner ids: c = 4 * a0 + 2 * a1 + a2 (a_i the offset along lattice axis i, axis 0 slowest).  Faces are wound so that their
normal points towards the positive pseudo-side (outwards on a closed surface whose outside is positive, as the reference's
'descent' output).  A missing normal (sparse list without the corner) counts as the zero vector.
"""
import numpy as np

OFF = np.array([[(c >> 2) & 1, (c >> 1) & 1, c & 1] for c in range(8)], np.int64)
# the reference's corner order (avg_cube argument order): its (z, y, x) = our (axis 0, axis 1, axis 2)
LEWINER_ORDER = [0, 1, 3, 2, 4, 5, 7, 6]
# cube faces, corners counter-clockwise seen from outside
FACES = [[0, 1, 3, 2], [4, 6, 7, 5], [0, 4, 5, 1], [2, 3, 7, 6], [0, 2, 6, 4], [1, 5, 7, 3]]


def edge_id(a, b):
    """local edge id 0..11: 4 * axis + the lower corner's position among the 4 edges of that axis"""
    lo, d = min(a, b), a ^ b
    axis = {4: 0, 2: 1, 1: 2}[d]
    rest = [c for c in range(8) if not c & d]
    return 4 * axis + rest.index(lo)


EDGE_CORNERS = [None] * 12
for _a in range(8):
    for _d in (4, 2, 1):
        if not _a & _d:
            EDGE_CORNERS[edge_id(_a, _a | _d)] = (_a, _a | _d)


def thresholds(n2):
    voxel = 2.0 / (n2 - 1)
    return np.float32(1.05 * voxel), np.float32(1.74 * voxel)


def corner_offsets(dims):
    n0, n1, n2 = dims
    return OFF[:, 0] * n1 * n2 + OFF[:, 1] * n2 + OFF[:, 2]


def active_cells(df, dims, avg_t=None, max_t=None):
    """sorted flat lattice indices (of the lower corner) of the active cells"""
    n0, n1, n2 = dims
    if avg_t is None:
        avg_t, max_t = thresholds(n2)
    g = df.reshape(n0, n1, n2).astype(np.float32)
    cor = [g[a:n0 - 1 + a, b:n1 - 1 + b, c:n2 - 1 + c] for a, b, c in OFF]
    s = cor[LEWINER_ORDER[0]]
    for c in LEWINER_ORDER[1:]:
        s = (s + cor[c]).astype(np.float32)
    mean = (s * np.float32(0.125)).astype(np.float32)
    mx = np.max(np.stack(cor), axis=0)
    act = (mean < avg_t) & (mx <= max_t)
    i, j, k = np.nonzero(act)
    return (i * n1 * n2 + j * n2 + k).astype(np.int64)


def _dot(a, b):
    a = a.astype(np.float32)
    b = b.astype(np.float32)
    return ((a[..., 0] * b[..., 0]).astype(np.float32) + (a[..., 1] * b[..., 1]).astype(np.float32)).astype(np.float32) \
        + (a[..., 2] * b[..., 2]).astype(np.float32)


def cell_signs(df, dims, cells, normals, idx=None):
    """uint8 [n]: bit c set = corner c on the negative pseudo-side (before polarity)"""
    co = cells[:, None] + corner_offsets(dims)[None, :]                 # [n, 8]
    u = df[co].astype(np.float32)
    if idx is None:
        g = normals[co].astype(np.float32)
    else:
        pos = np.minimum(np.searchsorted(idx, co), len(idx) - 1)
        g = np.where((idx[pos] == co)[..., None], normals[pos], 0).astype(np.float32)
    r = np.argmax(u, axis=1)                                            # first maximum
    n = len(cells)
    gr = g[np.arange(n), r]                                             # [n, 3]
    d = (OFF[None, :, :] - OFF[r][:, None, :]).astype(np.float32)       # [n, 8, 3]
    pr = _dot(np.broadcast_to(gr[:, None, :], d.shape), d)
    pc = _dot(g, d)
    dd = _dot(np.broadcast_to(gr[:, None, :], g.shape), g)
    same = ((pr < 0) & (pc > 0)) | (dd >= 0)
    same[np.arange(n), r] = True
    neg = ~same
    return (neg.astype(np.int64) << np.arange(8)[None, :]).sum(1).astype(np.uint8), u


def links(df, dims, cells, mask):
    """[n, 3] int64: per + axis, 2 * neighbour position + parity, or -1 (no active neighbour or mixed evidence)"""
    n0, n1, n2 = dims
    strides = [n1 * n2, n2, 1]
    n = len(cells)
    out = np.full((n, 3), -1, np.int64)
    ci = cells // (n1 * n2)
    cj = (cells // n2) % n1
    ck = cells % n2
    lim = [ci, cj, ck]
    co = cells[:, None] + corner_offsets(dims)[None, :]
    u = df[co]
    for ax, bit in enumerate((4, 2, 1)):
        nb = cells + strides[ax]
        pos = np.minimum(np.searchsorted(cells, nb), n - 1)
        ok = (cells[pos] == nb) & (lim[ax] + 1 < dims[ax] - 1)
        agree = np.zeros(n, np.int64)
        disagree = np.zeros(n, np.int64)
        for c in range(8):
            if not c & bit:
                continue
            cn = c ^ bit
            s1 = (mask.astype(np.int64) >> c) & 1
            s2 = (mask[pos].astype(np.int64) >> cn) & 1
            live = u[:, c] > 0
            agree += live & (s1 == s2)
            disagree += live & (s1 != s2)
        par = np.where(disagree == 0, 0, 1)
        good = ok & ((agree == 0) != (disagree == 0))
        out[good, ax] = 2 * pos[good] + par[good]
    return out


def polarity(mask, lk):
    """cell -> (root position, parity to root) by deterministic min-root hooking; returns the flipped masks"""
    n = len(mask)
    par = np.arange(n, dtype=np.int64)
    rel = np.zeros(n, np.int64)
    src = np.repeat(np.arange(n), 3)
    val = lk.reshape(-1)
    keep = val >= 0
    src, dst, p = src[keep], val[keep] >> 1, val[keep] & 1
    big = np.iinfo(np.int64).max
    while True:
        while True:                                                      # pointer jumping to the roots
            pp = par[par]
            if np.array_equal(pp, par):
                break
            rel = rel ^ rel[par]
            par = pp
        rc, rn = par[src], par[dst]
        par_cn = rel[src] ^ rel[dst] ^ p                                  # root(c) vs root(n)
        hook = np.full(n, big, np.int64)
        a = rn < rc
        np.minimum.at(hook, rc[a], (rn[a] << 1) | par_cn[a])
        b = rc < rn
        np.minimum.at(hook, rn[b], (rc[b] << 1) | par_cn[b])
        h = np.nonzero(hook != big)[0]
        if len(h) == 0:
            break
        par[h] = hook[h] >> 1
        rel[h] = hook[h] & 1
    flip = rel ^ (mask[par].astype(np.int64) & 1)
    return np.where(flip == 1, (~mask) & 0xFF, mask).astype(np.uint8), par, rel


_TRI_CACHE = {}


def cell_triangles(pos_mask, face_join):
    """triangles of one cell: local edge ids, or CENTRE + l for the centre vertex of loop l"""
    key = (pos_mask, face_join)
    t = _TRI_CACHE.get(key)
    if t is None:
        t = _TRI_CACHE[key] = [tri for li, lp in enumerate(cell_loops(pos_mask, face_join))
                               for tri in loop_triangles(lp, li)]
    return t


def cell_loops(pos_mask, face_join):
    """the crossing loops of one cell as lists of local edge ids.  pos_mask: bit c = corner c positive; face_join: bit f =
    ambiguous face f joins its positive corners"""
    p = [(pos_mask >> c) & 1 for c in range(8)]
    nxt = [-1] * 12
    for f, q in enumerate(FACES):
        e = [edge_id(q[s], q[(s + 1) % 4]) for s in range(4)]
        ncross = sum(p[q[s]] != p[q[(s + 1) % 4]] for s in range(4))
        if ncross == 2:
            for s in range(4):
                if not p[q[s]] and p[q[(s + 1) % 4]]:
                    a = e[s]
                if p[q[s]] and not p[q[(s + 1) % 4]]:
                    b = e[s]
            nxt[a] = b
        elif ncross == 4:
            join_pos = (face_join >> f) & 1
            for s in range(4):                                           # cut off corner q[s]
                cut = (not p[q[s]]) if join_pos else p[q[s]]
                if not cut:
                    continue
                e_in, e_out = e[(s + 3) % 4], e[s]
                if p[q[s]]:
                    nxt[e_in] = e_out
                else:
                    nxt[e_out] = e_in
    loops, seen = [], [False] * 12
    for s in range(12):
        if nxt[s] < 0 or seen[s]:
            continue
        loop, e = [], s
        while not seen[e]:
            seen[e] = True
            loop.append(e)
            e = nxt[e]
        loops.append(loop)
    return loops


CENTRE = 16


def edge_faces(e):
    """bit f set when local edge e lies on cube face f (FACES order: x=0, x=1, y=0, y=1, z=0, z=1)"""
    lo = EDGE_CORNERS[e][0]
    ax = e // 4
    return sum(1 << (2 * b + ((lo >> (2 - b)) & 1)) for b in range(3) if b != ax)


def loop_triangles(loop, li=0):
    """Triangulation of loop `li` with no chord lying in a cube face (such a chord would also be a chord or a segment of
    the neighbouring cell, making that edge non-manifold).  Dynamic programme over the polygon: cost[i][j] = in-face
    chords of the best triangulation of loop[i..j]; ties take the smallest apex k.  Emitted in pre-order (i, j) ->
    (i, k), (k, j); each triangle (i, k, j) is written (l_i, l_j, l_k), reversed loop order.  When no triangulation is
    free of in-face chords, the loop is fanned around its own centre vertex CENTRE + li: (C, l_{i+1}, l_i).
    The loop is first put in canonical order (from its smallest edge, towards the smaller neighbour) and the winding
    flipped back afterwards, so that a global sign flip, which reverses every loop, gives the same triangles."""
    loop, rev = canonical_loop(loop)
    tris = _loop_triangles(loop, li)
    return [(t[0], t[2], t[1]) for t in tris] if rev else tris


def canonical_loop(loop):
    """(loop starting at its smallest edge and running towards the smaller of its two neighbours, reversed?)"""
    n = len(loop)
    s = loop.index(min(loop))
    loop = loop[s:] + loop[:s]
    if n > 2 and loop[n - 1] < loop[1]:
        return [loop[0]] + loop[:0:-1], True
    return loop, False


def _loop_triangles(loop, li):
    n = len(loop)
    fm = [edge_faces(e) for e in loop]

    def bad(i, j):                                                      # chord (not a loop side) inside one cube face
        return int(j - i > 1 and not (i == 0 and j == n - 1) and (fm[i] & fm[j]) != 0)

    cost = [[0] * n for _ in range(n)]
    apex = [[0] * n for _ in range(n)]
    for span in range(2, n):
        for i in range(0, n - span):
            j = i + span
            best = None
            for k in range(i + 1, j):
                c = cost[i][k] + cost[k][j] + bad(i, k) + bad(k, j)
                if best is None or c < best:
                    best, apex[i][j] = c, k
            cost[i][j] = best
    if n > 2 and cost[0][n - 1] > 0:
        return [(CENTRE + li, loop[(i + 1) % n], loop[i]) for i in range(n)]
    tris, stack = [], [(0, n - 1)]
    while stack:
        i, j = stack.pop()
        if j - i < 2:
            continue
        k = apex[i][j]
        tris.append((loop[i], loop[j], loop[k]))
        stack.append((k, j))
        stack.append((i, k))
    return tris


def face_join_bits(v, pos_mask):
    """bit f set when ambiguous face f connects its positive corners (asymptotic decider; exact ties join q0-q2)"""
    bits = 0
    for f, q in enumerate(FACES):
        p = [(pos_mask >> c) & 1 for c in q]
        if not (p[0] == p[2] and p[1] == p[3] and p[0] != p[1]):
            continue
        a, b, c, d = (np.float32(v[x]) for x in q)
        det = np.float32(np.float32(a * c) - np.float32(b * d))
        if det == 0:
            join_pos = p[0] == 1
        elif p[0]:
            join_pos = det > 0
        else:
            join_pos = det < 0
        bits |= int(join_pos) << f
    return bits


def triangulate(df, dims, cells, mask, u):
    """[F, 3] int64 global edge keys, cells in order, triangles in loop / fan order"""
    n0, n1, n2 = dims
    corner_base = corner_offsets(dims)
    out = []
    for ci in range(len(cells)):
        m = int(mask[ci])
        uu = u[ci]
        pos_mask = 0
        v = np.empty(8, np.float32)
        for c in range(8):
            neg = (m >> c) & 1
            v[c] = -uu[c] if neg else uu[c]
            if v[c] > 0:
                pos_mask |= 1 << c
        if pos_mask == 0 or pos_mask == 0xFF:
            continue
        tris = cell_triangles(pos_mask, face_join_bits(v, pos_mask))
        for t in tris:
            row = []
            for e in t:
                if e >= CENTRE:
                    row.append(3 * n0 * n1 * n2 + 4 * ci + (e - CENTRE))
                else:
                    a, _ = EDGE_CORNERS[e]
                    row.append(3 * (int(cells[ci]) + int(corner_base[a])) + e // 4)
            out.append(row)
    return np.array(out, np.int64).reshape(-1, 3)


def edge_vertices(df, dims, keys):
    """index-space float32 positions of lattice-edge vertex keys"""
    n0, n1, n2 = dims
    strides = np.array([n1 * n2, n2, 1], np.int64)
    g, ax = keys // 3, keys % 3
    ua = df[g].astype(np.float32)
    ub = df[g + strides[ax]].astype(np.float32)
    t = (ua / (ua + ub).astype(np.float32)).astype(np.float32)
    ijk = np.stack([g // (n1 * n2), (g // n2) % n1, g % n2], 1).astype(np.float32)
    ijk[np.arange(len(keys)), ax] = (ijk[np.arange(len(keys)), ax] + t).astype(np.float32)
    return ijk


def vertices(df, dims, keys, cells, mask, u):
    """index-space float32 positions of the welded vertices (keys sorted unique): edge points, then loop centres (the mean
    of the loop's edge points, summed in canonical loop order)"""
    n0, n1, n2 = dims
    c0 = 3 * n0 * n1 * n2
    out = np.zeros((len(keys), 3), np.float32)
    ek = keys < c0
    out[ek] = edge_vertices(df, dims, keys[ek])
    corner_base = corner_offsets(dims)
    for r in np.nonzero(~ek)[0]:
        ci, li = int(keys[r] - c0) >> 2, int(keys[r] - c0) & 3
        m, uu = int(mask[ci]), u[ci]
        v = np.array([-uu[c] if (m >> c) & 1 else uu[c] for c in range(8)], np.float32)
        pos_mask = sum(1 << c for c in range(8) if v[c] > 0)
        loop, _ = canonical_loop(cell_loops(pos_mask, face_join_bits(v, pos_mask))[li])
        ek_loop = np.array([3 * (int(cells[ci]) + int(corner_base[EDGE_CORNERS[e][0]])) + e // 4 for e in loop], np.int64)
        pts = edge_vertices(df, dims, ek_loop)
        acc = pts[0].copy()
        for p in pts[1:]:
            acc = (acc + p).astype(np.float32)
        out[r] = (acc / np.float32(len(loop))).astype(np.float32)
    return out


def marching_cubes(df, dims, normals, idx=None):
    """(verts [V,3] float32 index space, faces [F,3] int64, info dict) -- the whole pipeline"""
    df = np.ascontiguousarray(df, np.float32).reshape(-1)
    cells = active_cells(df, dims)
    info = {"active": cells}
    if len(cells) == 0:
        return np.zeros((0, 3), np.float32), np.zeros((0, 3), np.int64), info
    mask, u = cell_signs(df, dims, cells, normals, idx)
    lk = links(df, dims, cells, mask)
    mask, root, rel = polarity(mask, lk)
    info.update(mask=mask, root=root)
    keys = triangulate(df, dims, cells, mask, u)
    info["face_keys"] = keys
    uk, inv = np.unique(keys.reshape(-1), return_inverse=True)
    return vertices(df, dims, uk, cells, mask, u), inv.reshape(-1, 3).astype(np.int64), info


def to_world(verts, n):
    voxel = np.float32(2.0 / (n - 1))
    return ((verts * voxel).astype(np.float32) - np.float32(1.0)).astype(np.float32)

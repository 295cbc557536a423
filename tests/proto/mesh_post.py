"""NumPy restatement of the mesh post-processing kernels (neuraludf_b200/csrc/mesh_post.cu) and of the torch steps around
them (neuraludf_b200/mesh_post.py): the exact oracle of the device code, same fp64 operation order, same vertex and face
numbering.  The rules it implements restate trimesh's primitives (DESIGN.md §1, "mesh post-processing")."""
import numpy as np

MERGE_TOL_DIGITS = 8            # trimesh tol.merge = 1e-8
NONDEGENERATE_TOL = 1e-8
SMOOTH_LAMBDA = 0.3
SMOOTH_STEPS = 5
MAX_PASSES = 10


def world64(verts_index32, N):
    """fp64(fp32 MC vertex in lattice-index units) * fp64(2 / (N - 1)) - 1, in fp64 (the reference's MC output, `verts - 1`)"""
    return np.asarray(verts_index32, np.float32).astype(np.float64) * (2.0 / (N - 1)) - 1.0


def drop_nonfinite(verts, faces):
    """faces that have a non-finite vertex are dropped (trimesh remove_infinite_values)"""
    ok = np.isfinite(verts).all(1)
    return faces[ok[faces].all(1)] if len(faces) else faces


def merge_keys(verts):
    return np.round(verts * 10.0 ** MERGE_TOL_DIGITS).astype(np.int64)


def merge(verts, faces):
    """(verts, faces, remap): referenced vertices merge when round-half-even(x 1e8) is equal in all three coordinates; the
    merged vertex keeps the coordinates of its lowest-indexed member, merged vertices are numbered in the order of those
    members, unreferenced vertices are dropped.  remap[old] = new index (-1: dropped)."""
    V = verts.shape[0]
    used = np.zeros(V, bool)
    used[faces.reshape(-1)] = True
    ref = np.nonzero(used)[0]
    remap = np.full(V, -1, np.int64)
    if ref.size == 0:
        return verts[:0], faces.reshape(0, 3).astype(np.int64), remap
    _, first, inv = np.unique(merge_keys(verts[ref]), axis=0, return_index=True, return_inverse=True)
    inv = inv.reshape(-1)
    rep = ref[first]                            # np.unique's first occurrence: the lowest member index of each group
    order = np.argsort(rep, kind="stable")
    rank = np.empty_like(order)
    rank[order] = np.arange(order.size)
    remap[ref] = rank[inv]
    return verts[rep[order]], remap[faces], remap


def nondegenerate(verts, faces):
    """a = v1 - v0, b = v2 - v0, c = a x b: keep when |a|, |b|, |c| / |a| and |c| / |b| all exceed 1e-8 (|c| = 2 area);
    |x| = sqrt((x0 x0 + x1 x1) + x2 x2) (trimesh triangles.nondegenerate at tol.merge)"""
    p = verts[faces]
    a, b = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
    c = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                  a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)

    def norm(x):
        return np.sqrt((x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1]) + x[:, 2] * x[:, 2])

    la, lb, lc = norm(a), norm(b), norm(c)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = NONDEGENERATE_TOL
        return (la > t) & (lb > t) & (lc / la > t) & (lc / lb > t)


def first_unique(faces):
    """mask of the first face of each sorted vertex triple (trimesh remove_duplicate_faces, any winding)"""
    if len(faces) == 0:
        return np.zeros(0, bool)
    _, first = np.unique(np.sort(faces, 1), axis=0, return_index=True)
    keep = np.zeros(len(faces), bool)
    keep[first] = True
    return keep


def process(verts, faces):
    """non-finite, merge, duplicate faces, degenerate faces: (verts, faces, counts)"""
    f = drop_nonfinite(verts, faces)
    n_nonfinite = len(faces) - len(f)
    v, f, _ = merge(verts, f)
    keep = first_unique(f)
    n_dup = int((~keep).sum())
    f = f[keep]
    keep = nondegenerate(v, f)
    n_degen = int((~keep).sum())
    return v, f[keep], {"nonfinite": n_nonfinite, "duplicate": n_dup, "degenerate": n_degen}


def boundary(faces, n_verts):
    """(edges [B,2] sorted pairs in ascending key order, dirs [B]: 1 when the face traverses the edge high -> low) of the
    edges used by exactly one face"""
    e = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]], 0).reshape(-1, 2)
    lo, hi = e.min(1), e.max(1)
    code = (lo * n_verts + hi) * 2 + (e[:, 0] > e[:, 1])
    code.sort()
    key = code >> 1
    _, start, cnt = np.unique(key, return_index=True, return_counts=True)
    b = code[start[cnt == 1]]
    k = b >> 1
    return np.stack([k // n_verts, k % n_verts], 1), (b & 1)


def neighbour_csr(edges, n_verts):
    """(rowptr [V+1], cols): each vertex's boundary neighbours in ascending order"""
    src = np.concatenate([edges[:, 0], edges[:, 1]])
    dst = np.concatenate([edges[:, 1], edges[:, 0]])
    order = np.lexsort((dst, src))
    rowptr = np.zeros(n_verts + 1, np.int64)
    np.cumsum(np.bincount(src, minlength=n_verts), out=rowptr[1:])
    return rowptr, dst[order]


def _sqdist(p, q):
    d = p - q
    return (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]


def hole_faces(verts, faces):
    """faces closing every boundary component that is a simple cycle of 3 or 4 vertices (trimesh repair.fill_holes).

    One walk per boundary edge (u, v), u < v: from v away from u over vertices of boundary degree 2, at most 4 vertices;
    the edge owns the hole when the walk returns to u and every other edge of the cycle has a larger key.  The new faces
    traverse the owner edge against its direction in its face.  A quad is split along its shorter diagonal (squared
    lengths, (dx dx + dy dy) + dz dz), on a tie along the one through the smallest vertex index.  Output: in owner-edge
    order, a quad's two faces (d0, d1, d2), (d0, d2, d3) with d0 -- d2 the diagonal."""
    V = verts.shape[0]
    if len(faces) == 0:
        return np.zeros((0, 3), np.int64)
    edges, dirs = boundary(faces, V)
    if len(edges) == 0:
        return np.zeros((0, 3), np.int64)
    rowptr, cols = neighbour_csr(edges, V)
    deg = rowptr[1:] - rowptr[:-1]
    u, v = edges[:, 0], edges[:, 1]
    B = len(u)
    cyc = np.full((B, 4), -1, np.int64)
    cyc[:, 0], cyc[:, 1] = u, v
    length = np.zeros(B, np.int64)
    active = (deg[u] == 2) & (deg[v] == 2)
    prev, cur = u.copy(), v.copy()
    for step in range(3):
        r = rowptr[np.where(active, cur, 0)]
        n0, n1 = cols[np.minimum(r, len(cols) - 1)], cols[np.minimum(r + 1, len(cols) - 1)]
        nxt = np.where(n0 == prev, n1, n0)
        closed = active & (nxt == u) & (step >= 1)
        length[closed] = step + 2
        active &= ~closed
        if step == 2:
            break
        active &= deg[np.where(active, nxt, 0)] == 2
        cyc[active, step + 2] = nxt[active]
        prev, cur = np.where(active, cur, prev), np.where(active, nxt, cur)
    out = []
    for i in np.nonzero(length)[0]:
        L = int(length[i])
        c = [int(x) for x in cyc[i, :L]]
        k0 = c[0] * V + c[1]
        if any(min(c[j], c[(j + 1) % L]) * V + max(c[j], c[(j + 1) % L]) <= k0 for j in range(1, L)):
            continue                            # not the cycle's smallest edge
        if dirs[i] == 0:                        # the face runs u -> v: the new faces run v -> u
            c = [c[0]] + c[:0:-1]
        if L == 3:
            out.append(c)
            continue
        p = verts[c]
        d02, d13 = _sqdist(p[0:1], p[2:3])[0], _sqdist(p[1:2], p[3:4])[0]
        if d13 < d02 or (d13 == d02 and min(c[1], c[3]) < min(c[0], c[2])):
            c = c[1:] + c[:1]
        out += [[c[0], c[1], c[2]], [c[0], c[2], c[3]]]
    return np.asarray(out, np.int64).reshape(-1, 3)


def smooth(verts, faces, steps=SMOOTH_STEPS, lam=SMOOTH_LAMBDA):
    """Jacobi border smoothing (extract_mesh.py:238-265): each pass moves every border vertex to v + lam (mean of its
    border neighbours - v), all from the previous pass's positions; neighbours summed in ascending index order."""
    V = verts.shape[0]
    if len(faces) == 0:
        return verts.copy(), 0
    edges, _ = boundary(faces, V)
    if len(edges) == 0:
        return verts.copy(), 0
    rowptr, cols = neighbour_csr(edges, V)
    deg = rowptr[1:] - rowptr[:-1]
    bv = np.nonzero(deg)[0]
    d = deg[bv]
    v = verts.copy()
    for _ in range(steps):
        s = np.zeros((len(bv), 3))
        for k in range(int(d.max())):
            has = k < d
            nb = cols[np.where(has, rowptr[bv] + k, 0)]
            s = np.where(has[:, None], s + v[nb], s)
        mean = s / d[:, None].astype(np.float64)
        nv = v.copy()
        nv[bv] = v[bv] + lam * (mean - v[bv])
        v = nv
    return v, len(bv)


def postprocess(verts, faces, smooth_borders=True):
    """get_mesh_udf_fast's post-processing after the vertex filter (extract_mesh.py:215-265) under the restated rules:
    (fp64 verts, int64 faces, info)"""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    info = {"input": (len(v), len(f))}
    v, f, c = process(v, f)                         # Trimesh(...) + process, duplicates, degenerate
    info["process"] = c
    holes = hole_faces(v, f)
    info["hole_faces"] = len(holes)
    info["pre_fill"] = (v, f)
    f = np.concatenate([f, holes]) if len(holes) else f
    v, f, _ = merge(v, f)                           # Trimesh(...)
    passes, counts, loop = 0, (0, 0), []
    while counts != (len(v), len(f)) and passes < MAX_PASSES:
        v, f, c = process(v, f)
        loop.append(c)
        counts = (len(v), len(f))
        passes += 1
        v, f, _ = merge(v, f)
    info["loop"], info["passes"] = loop, passes
    info["border_vertices"] = 0
    if smooth_borders:
        v, info["border_vertices"] = smooth(v, f)
    info["output"] = (len(v), len(f))
    return v, f, info


def export_merge(verts, faces):
    """the runner's last Trimesh(...) before export (exp_runner_blending.py:796): one more merge"""
    f = drop_nonfinite(verts, faces)
    v, f, _ = merge(verts, f)
    return v, f


def canonical(verts, faces):
    """vertices sorted lexicographically, each face rotated so that its smallest vertex comes first, faces sorted"""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    order = np.lexsort(v.T[::-1])
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    f = rank[f]
    r = np.argmin(f, 1)
    f = np.stack([f[np.arange(len(f)), (r + k) % 3] for k in range(3)], 1)
    f = f[np.lexsort(f.T[::-1])] if len(f) else f
    return v[order], f

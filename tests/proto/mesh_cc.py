"""NumPy restatement of the connected-component mesh filters (neuraludf_b200/clean.py face_components, keep_largest,
remove_small_components, clean_outliers; csrc/mesh_cc.cu): the exact oracle of the device code.  Components come from
scipy.sparse.csgraph.connected_components, an algorithm independent of the device union-find.  The rules restate
trimesh's face_adjacency, split(only_watertight=False) and submesh (DESIGN.md §1, "connected components"); the crafted
cases below are shared by the tests and oracle/make_golden_cc.py."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from tests.proto import mesh_post as P


def face_adjacency(faces):
    """[P, 2] ascending pairs of trimesh face_adjacency: a sorted edge used by exactly two face slots joins their faces,
    unless the two slots are one face's (a degenerate face such as (a, a, b))"""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    if len(f) == 0:
        return np.zeros((0, 2), np.int64)
    edges = np.sort(f[:, [0, 1, 1, 2, 2, 0]].reshape(-1, 2), axis=1)
    owner = np.repeat(np.arange(len(f), dtype=np.int64), 3)
    _, inv, cnt = np.unique(edges[:, 0] * (int(f.max()) + 1) + edges[:, 1], return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    slots = np.nonzero(cnt[inv] == 2)[0]
    slots = slots[np.argsort(inv[slots], kind="stable")].reshape(-1, 2)
    pairs = np.sort(owner[slots], axis=1)
    return pairs[pairs[:, 0] != pairs[:, 1]]


def face_components(faces):
    """(label [F] int64: the smallest face index of each face's component, paired [F] uint8: in at least one pair)"""
    F = len(np.asarray(faces).reshape(-1, 3))
    pairs = face_adjacency(faces)
    paired = np.zeros(F, np.uint8)
    paired[pairs.reshape(-1)] = 1
    if F == 0:
        return np.zeros(0, np.int64), paired
    g = coo_matrix((np.ones(len(pairs)), (pairs[:, 0], pairs[:, 1])), shape=(F, F))
    _, comp = connected_components(g, directed=False)
    smallest = np.full(comp.max() + 1, F, np.int64)
    np.minimum.at(smallest, comp, np.arange(F, dtype=np.int64))
    return smallest[comp], paired


def submesh(verts, faces, keep):
    """the kept faces in ascending index, over the vertices they reference in ascending index (np.unique)"""
    f = np.asarray(faces, np.int64).reshape(-1, 3)[np.asarray(keep, bool)]
    used = np.unique(f.reshape(-1))
    rank = np.full(len(verts), -1, np.int64)
    rank[used] = np.arange(len(used))
    return np.asarray(verts)[used], rank[f]


def largest_mask(label):
    """faces of the largest component; equal sizes go to the component with the smallest face index"""
    if len(label) == 0:
        return np.zeros(0, bool)
    size = np.bincount(label, minlength=len(label))
    return label == np.argmax(size)


def small_mask(label, paired, faces_num):
    """faces in a pair whose component, counted over paired faces, has at least faces_num faces"""
    p = paired.astype(bool)
    size = np.bincount(label[p], minlength=len(label))
    return p & (size[label] >= faces_num)


def keep_largest(verts, faces):
    return submesh(verts, faces, largest_mask(face_components(faces)[0]))


def remove_small_components(verts, faces, faces_num=500):
    return submesh(verts, faces, small_mask(*face_components(faces), faces_num))


def clean_outliers(verts, faces, faces_num=500, keep_largest=True):
    """trimesh.load's merge (non-finite faces dropped, 1e-8 grid), then keep_largest or remove_small_components"""
    v, f = P.export_merge(np.asarray(verts, np.float64).reshape(-1, 3), np.asarray(faces, np.int64).reshape(-1, 3))
    label, paired = face_components(f)
    return submesh(v, f, largest_mask(label) if keep_largest else small_mask(label, paired, faces_num))


# ---------------------------------------------------------------------------------------------------------------------
# crafted cases: name -> (verts fp64 [V,3], faces int64 [F,3])

def strip(n, x0=0.0, y0=0.0, z=0.0, base=0):
    """n faces over 2 rows of vertices: face i is (i, i + 1, i + 2) with alternating winding"""
    m = n + 2
    v = np.stack([x0 + 0.5 * (np.arange(m) // 2), y0 + (np.arange(m) % 2), np.full(m, z)], 1)
    f = np.array([(i, i + 1, i + 2) if i % 2 == 0 else (i + 1, i, i + 2) for i in range(n)], np.int64).reshape(-1, 3)
    return v, f + base


def grid(nx, ny, x0=0.0, y0=0.0, z=0.0, h=0.1):
    """2 nx ny faces over a (nx + 1) x (ny + 1) vertex grid"""
    xs, ys = np.meshgrid(np.arange(nx + 1), np.arange(ny + 1), indexing="ij")
    v = np.stack([x0 + h * xs.reshape(-1), y0 + h * ys.reshape(-1), np.full(xs.size, z)], 1)
    i = (np.arange(nx)[:, None] * (ny + 1) + np.arange(ny)[None]).reshape(-1)
    f = np.concatenate([np.stack([i, i + ny + 1, i + 1], 1), np.stack([i + 1, i + ny + 1, i + ny + 2], 1)])
    return v, f.astype(np.int64)


def concat(*meshes):
    vs, fs, base = [], [], 0
    for v, f in meshes:
        vs.append(np.asarray(v, np.float64).reshape(-1, 3))
        fs.append(np.asarray(f, np.int64).reshape(-1, 3) + base)
        base += len(vs[-1])
    return np.concatenate(vs), np.concatenate(fs)


def _tri(x, y=0.0, z=0.0):
    return np.array([[x, y, z], [x + 1.0, y, z], [x, y + 1.0, z]]), np.array([[0, 1, 2]])


def _fan(k):
    """k triangles on the edge (0, 1), each with one more triangle hung on its far edge"""
    v = [[0.0, 0.0, 0.0], [1.0, 0.0, 0.0]]
    f = []
    for j in range(k):
        a = 2.0 * np.pi * j / k
        v.append([0.5, np.cos(a), np.sin(a)])
        v.append([1.5, np.cos(a), np.sin(a)])
        f.append([0, 1, 2 + 2 * j] if j % 2 == 0 else [1, 0, 2 + 2 * j])
        f.append([1, 3 + 2 * j, 2 + 2 * j])
    return np.array(v), np.array(f)


def floaters(seed=0):
    """a 24 x 24 sheet in two halves whose seam vertices are duplicated (the load merge joins them), seeded floating strips
    and triangles, a non-finite vertex, unreferenced vertices; faces in a seeded random order"""
    rng = np.random.default_rng(seed)
    a = grid(12, 24, h=0.1)
    b = grid(12, 24, x0=1.2, h=0.1)
    parts = [a, b]
    for _ in range(12):
        n = int(rng.integers(1, 9))
        parts.append(strip(n, x0=float(rng.uniform(-3, 3)), y0=float(rng.uniform(-3, 3)), z=float(rng.uniform(0.5, 2))))
    for _ in range(5):
        parts.append(_tri(float(rng.uniform(-3, 3)), float(rng.uniform(-3, 3)), float(rng.uniform(-2, -0.5))))
    v, f = concat(*parts)
    nan = np.array([[np.nan, 0.0, 0.0]])
    v = np.concatenate([v, nan, rng.uniform(-1, 1, (4, 3))])
    f = np.concatenate([f, [[0, 1, len(v) - 5]]])
    return v, f[rng.permutation(len(f))]


def _cases():
    t = _tri(0.0)
    sq = (np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], np.float64), np.array([[0, 1, 2], [0, 2, 3]]))
    sq2 = (sq[0] + [5.0, 5.0, 0.0], sq[1])
    gv, gf = grid(3, 3)
    emb_v, emb_f = gv, np.concatenate([gf, gf[7:8]])                       # one face duplicated inside a surface
    v_tie, f_tie = concat(sq, strip(2, x0=10.0), sq2)
    return {
        "fan3": _fan(3),
        "fan4": _fan(4),
        "bowtie": (np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [-1, 0, 0], [0, -1, 0]], np.float64),
                   np.array([[0, 1, 2], [0, 3, 4]])),
        "duplicate_isolated": concat((t[0], np.array([[0, 1, 2], [0, 1, 2], [2, 1, 0]])), sq2),
        "duplicate_embedded": (emb_v, emb_f),
        "degenerate": concat((np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0]], np.float64), np.array([[0, 0, 1], [1, 2, 2]])),
                             strip(3, y0=3.0), (np.array([[0, 0, 5], [1, 0, 5], [0, 1, 5]], np.float64),
                                                np.array([[0, 1, 2], [0, 0, 1]]))),
        "isolated": concat(*[_tri(3.0 * i) for i in range(5)]),
        "unreferenced": concat((np.random.default_rng(1).uniform(-1, 1, (3, 3)), np.zeros((0, 3), np.int64)), strip(4),
                               (np.random.default_rng(2).uniform(-1, 1, (2, 3)), np.zeros((0, 3), np.int64)), sq2),
        "empty": (np.zeros((3, 3)), np.zeros((0, 3), np.int64)),
        "one_face": t,
        "tie": (v_tie, f_tie[[4, 0, 2, 5, 1, 3]]),
        "floaters": floaters(),
    }


CASES = sorted(_cases())


def case(name):
    v, f = _cases()[name]
    return np.ascontiguousarray(v, np.float64), np.ascontiguousarray(f, np.int64).reshape(-1, 3)

"""Run the UNMODIFIED reference `get_mesh_udf_fast` (extract_mesh.py:169-354) under a trimesh stub -- test infrastructure.

trimesh is not installed here, so its primitives are restated by the rules of DESIGN.md §1 ("mesh post-processing") and
implemented below independently of tests/proto/mesh_post.py: plain NumPy and dictionaries for the merge and the face
rules, networkx connected components for the holes.  The reference's own control flow (order of steps, the fixed-point
loop, the border smoothing's coo_matrix arithmetic) runs unchanged from the staged `extract_mesh.py` (oracle/make_ref.py).

`fill_holes` also runs trimesh's own recipe (`networkx.cycle_basis` over the boundary graph, 3-cycles as one face, 4-cycles
as faces (c0, c1, c2), (c2, c3, c0)) beside the rule and counts every place where the two differ: a cycle one finds and the
other does not, or a quad split along the other diagonal.  The rule's faces are the ones added.

`run_post` serves `get_udf_normals_grid_fast` from given df / normals, `udf_mc_lewiner` from a given callable (the compiled
reference MC, the device drop-in, or a crafted mesh), maps `.cuda()` to the CPU unless `device` is CUDA, and calls
get_mesh_udf_fast the way Runner.extract_udf_mesh does (exp_runner_blending.py:777-800): gradient=True, eps=0.005, first
with border_gradients and smooth_borders, again without them if that raises; then the runner's last Trimesh(...).
"""
import contextlib
import importlib.util
import os
import sys
import types

import numpy as np
import torch

from oracle import refshim

NX_DISAGREEMENTS = [0]          # fill_holes: places where networkx's cycles / diagonals differ from the rule


def _merge(vertices, faces):
    """non-finite faces dropped, then the merge rule (lowest-indexed member's coordinates, members' order)"""
    v = np.asarray(vertices, np.float64).reshape(-1, 3)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    fin = np.isfinite(v).all(1)
    f = f[fin[f].all(1)] if len(f) else f
    seen, rep = {}, []
    new = np.full(len(v), -1, np.int64)
    for i in sorted(set(f.reshape(-1).tolist())):
        k = tuple(np.round(v[i] * 1e8).astype(np.int64).tolist())
        if k not in seen:
            seen[k] = len(rep)
            rep.append(i)
        new[i] = seen[k]
    return v[np.asarray(rep, np.int64)].reshape(-1, 3), new[f].reshape(-1, 3)


def _norm(x):
    return np.sqrt((x[..., 0] * x[..., 0] + x[..., 1] * x[..., 1]) + x[..., 2] * x[..., 2])


def _edges_sorted(faces):
    return np.sort(np.asarray(faces, np.int64)[:, [0, 1, 1, 2, 2, 0]].reshape(-1, 2), axis=1)


def group_rows(data, require_count=None, digits=None):
    """trimesh.grouping.group_rows for require_count=1: indices of the rows that occur once, in row-value order"""
    assert require_count == 1
    d = np.asarray(data)
    _, first, cnt = np.unique(d, axis=0, return_index=True, return_counts=True)
    return first[cnt == 1]


class Trimesh:
    def __init__(self, vertices=None, faces=None, process=True, **kw):
        self.vertices = np.array(vertices, np.float64).reshape(-1, 3)
        self.faces = np.array(faces, np.int64).reshape(-1, 3)
        if process:
            self.process()

    def process(self, validate=False):
        self.vertices, self.faces = _merge(self.vertices, self.faces)
        return self

    def remove_duplicate_faces(self):
        seen, keep = set(), []
        for i, f in enumerate(self.faces.tolist()):
            k = tuple(sorted(f))
            if k not in seen:
                seen.add(k)
                keep.append(i)
        self.faces = self.faces[np.asarray(keep, np.int64)].reshape(-1, 3)

    def remove_degenerate_faces(self, height=1e-8):
        p = self.vertices[self.faces]
        a, b = p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]
        c = np.stack([a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
                      a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]], 1)
        la, lb, lc = _norm(a), _norm(b), _norm(c)
        with np.errstate(divide="ignore", invalid="ignore"):
            ok = (la > height) & (lb > height) & (lc / la > height) & (lc / lb > height)
        self.faces = self.faces[ok]

    @property
    def edges_sorted(self):
        return _edges_sorted(self.faces)

    def fill_holes(self):
        import networkx as nx
        f = self.faces
        if len(f) == 0:
            return False
        es = _edges_sorted(f)
        directed = f[:, [0, 1, 1, 2, 2, 0]].reshape(-1, 2)
        once = group_rows(es, require_count=1)
        direction = {tuple(es[i]): tuple(directed[i]) for i in once}
        g = nx.Graph()
        g.add_edges_from(es[once].tolist())
        rule = {}                              # frozenset(cycle vertices) -> oriented faces
        for comp in nx.connected_components(g):
            if len(comp) not in (3, 4) or any(g.degree(x) != 2 for x in comp):
                continue
            start = min(comp)
            cyc = [start, min(g.neighbors(start))]
            while len(cyc) < len(comp):
                cyc.append(next(y for y in g.neighbors(cyc[-1]) if y != cyc[-2]))
            ring = [tuple(sorted((cyc[j], cyc[(j + 1) % len(cyc)]))) for j in range(len(cyc))]
            owner = min(ring)
            a, b = direction[owner]                 # the new faces run b -> a
            i = cyc.index(b)
            o = cyc[i:] + cyc[:i]
            if o[1] != a:
                o = [o[0]] + o[:0:-1]
            if len(o) == 3:
                rule[frozenset(o)] = ([o], None)
                continue
            e02, e13 = self.vertices[o[0]] - self.vertices[o[2]], self.vertices[o[1]] - self.vertices[o[3]]
            d02 = (e02[0] * e02[0] + e02[1] * e02[1]) + e02[2] * e02[2]
            d13 = (e13[0] * e13[0] + e13[1] * e13[1]) + e13[2] * e13[2]
            if d13 < d02 or (d13 == d02 and min(o[1], o[3]) < min(o[0], o[2])):
                o = o[1:] + o[:1]
            rule[frozenset(o)] = ([[o[0], o[1], o[2]], [o[0], o[2], o[3]]], frozenset((o[0], o[2])))
        # trimesh's recipe (repair.fill_holes): cycle_basis, 3- and 4-cycles only, quad diagonal c0 -- c2
        found = {}
        if len(f) >= 3 and len(once) >= 3:
            for c in nx.cycle_basis(g):
                if len(c) in (3, 4):
                    found[frozenset(c)] = None if len(c) == 3 else frozenset((c[0], c[2]))
        NX_DISAGREEMENTS[0] += len(set(found) ^ set(rule))
        NX_DISAGREEMENTS[0] += sum(found[k] != rule[k][1] for k in set(found) & set(rule))
        new = [face for k in sorted(rule, key=lambda s: sorted(s)) for face in rule[k][0]]
        if new:
            self.faces = np.concatenate([f, np.asarray(new, np.int64)])
        return True

    # used only for the gradient=True outputs (new_verts, border gradients), which do not reach the exported mesh
    @property
    def face_normals(self):
        p = self.vertices[self.faces]
        n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
        return n / np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-300)

    @property
    def face_angles(self):
        p = self.vertices[self.faces]
        out = []
        for k in range(3):
            u, w = p[:, (k + 1) % 3] - p[:, k], p[:, (k + 2) % 3] - p[:, k]
            cosv = (u * w).sum(1) / np.maximum(np.linalg.norm(u, axis=1) * np.linalg.norm(w, axis=1), 1e-300)
            out.append(np.arccos(np.clip(cosv, -1, 1)))
        return np.stack(out, 1)


def weighted_vertex_normals(vertex_count, faces, face_normals, face_angles, **kw):
    n = np.zeros((vertex_count, 3))
    for k in range(3):
        np.add.at(n, faces[:, k], face_normals * face_angles[:, k:k + 1])
    return n / np.maximum(np.linalg.norm(n, axis=1, keepdims=True), 1e-300)


def trimesh_stub():
    tm = types.ModuleType("trimesh")
    tm.Trimesh = Trimesh
    tm.grouping = types.SimpleNamespace(group_rows=group_rows)
    tm.geometry = types.SimpleNamespace(weighted_vertex_normals=weighted_vertex_normals)
    return tm


def load_extract_mesh():
    """the staged, unmodified extract_mesh.py as a private module, with the trimesh stub and a placeholder custom_mc"""
    path = os.path.join(refshim.REFERENCE_ROOT, "extract_mesh.py")
    if not os.path.isfile(path):
        raise RuntimeError("extract_mesh.py is not staged (oracle/make_ref.py)")
    saved = {k: sys.modules.get(k) for k in ("trimesh", "custom_mc", "custom_mc._marching_cubes_lewiner")}
    cm = types.ModuleType("custom_mc")
    cm.__path__ = []
    cm._marching_cubes_lewiner = types.ModuleType("custom_mc._marching_cubes_lewiner")
    cm._marching_cubes_lewiner.udf_mc_lewiner = None
    sys.modules.update({"trimesh": trimesh_stub(), "custom_mc": cm, "custom_mc._marching_cubes_lewiner": cm._marching_cubes_lewiner})
    try:
        spec = importlib.util.spec_from_file_location("_ref_extract_mesh_post", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        for k, m in saved.items():
            if m is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = m
    return mod


@contextlib.contextmanager
def _cuda_on_cpu():
    orig = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    try:
        yield
    finally:
        torch.Tensor.cuda = orig


class _Recorder(Trimesh):
    """records the first mesh built (the vertex filter's output, extract_mesh.py:215)"""
    first = None

    def __init__(self, vertices=None, faces=None, process=True, **kw):
        if _Recorder.first is None:
            _Recorder.first = (np.array(vertices, np.float64), np.array(faces, np.int64))
        super().__init__(vertices, faces, process, **kw)


def run_post(df, normals, N, mc, func, func_grad=None, dist_threshold_ratio=5.0, device="cpu"):
    """Runner.extract_udf_mesh's call of the unmodified get_mesh_udf_fast (exp_runner_blending.py:777-800, world_space
    False) and its last Trimesh(...).  df [N^3] / normals [N^3,3]: the lattice get_udf_normals_grid_fast would return;
    mc(volume, grads, spacing=...): udf_mc_lewiner; func(xyz [P,3] fp32 tensor) -> [P,1] udf.  Returns a dict with
    `input` (verts, faces after the vertex filter), `verts` / `faces` (the exported mesh), `smoothed` (whether the first
    call succeeded), `fallback` (what the first call raised) and `nx_disagreements`."""
    em = load_extract_mesh()
    em.trimesh.Trimesh = _Recorder
    _Recorder.first = None
    NX_DISAGREEMENTS[0] = 0
    em.udf_mc_lewiner = mc
    dfv = torch.from_numpy(np.asarray(df, np.float32).reshape(N, N, N).copy())
    nrm = torch.from_numpy(np.asarray(normals, np.float32).reshape(N, N, N, 3).copy())
    em.get_udf_normals_grid_fast = lambda func, func_grad, samples, indices, N=N: (dfv.clone(), nrm.clone(), None)
    func_grad = func_grad or (lambda x: torch.zeros(x.shape[0], 1, 3))
    ctx = _cuda_on_cpu() if device == "cpu" else contextlib.nullcontext()
    with ctx:
        try:
            out = em.get_mesh_udf_fast(func, func_grad, samples=None, indices=None, N_MC=N, gradient=True, eps=0.005,
                                       border_gradients=True, smooth_borders=True, dist_threshold_ratio=dist_threshold_ratio)
            smoothed, fallback = True, None
        except Exception as e:                  # the runner's bare `except:` (exp_runner_blending.py:784)
            fallback = "%s: %s" % (type(e).__name__, e)
            _Recorder.first = None
            NX_DISAGREEMENTS[0] = 0
            out = em.get_mesh_udf_fast(func, func_grad, samples=None, indices=None, N_MC=N, gradient=True, eps=0.005,
                                       border_gradients=False, smooth_borders=False, dist_threshold_ratio=dist_threshold_ratio)
            smoothed = False
    pred_mesh = out[2]
    final = Trimesh(pred_mesh.vertices, pred_mesh.faces)
    return {"input": _Recorder.first, "verts": final.vertices, "faces": final.faces, "smoothed": smoothed,
            "nx_disagreements": NX_DISAGREEMENTS[0], "fallback": fallback}

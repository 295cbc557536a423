"""Golden connected-component filters of the reference script -- tests/golden/cc_<case>.00.npz.

    python oracle/make_golden_cc.py      # needs the reference checkout (oracle/ref_clean.py stages its script)

Runs the unmodified clean_outliers of evaluation/clean_dtu_mesh.py (staged by oracle/ref_clean.py) on the crafted cases of
tests/proto/mesh_cc.py, with both keep_largest=True and keep_largest=False.  trimesh is not installed, so the module it
imports is a stub restating the primitives clean_outliers touches, independently of tests/proto/mesh_cc.py:
  load(path)                     the arrays stored under path, merged as trimesh.load does (oracle/ref_post.py's rule:
                                 non-finite faces dropped, 1e-8 merge grid, unreferenced vertices dropped);
  Trimesh.face_adjacency         edge -> face slots in a dictionary; an edge with exactly two slots of two different faces
                                 joins them;
  graph.connected_components     networkx components over the nodes the edges name, of at least min_len nodes, each
                                 sorted, in the order of their smallest node;
  Trimesh.split(False)           every face a node, the components as pieces in that order; a piece keeps its faces in
                                 ascending index over the vertices they reference in ascending index, with no hole filling;
  Trimesh(v, f).export(path)     stores the arrays under path.
Stored per case: the inputs, the exported arrays of keep_largest=True (or the exception it raised) and the exception
clean_mesh_by_faces_num raised for keep_largest=False at faces_num 500 and 2 ("" if it returned).  Its mask is per face but
indexed with vertex ids, and the per-vertex index map is indexed with face ids, so wherever a component passes the size
test it raises IndexError; where none does, np.concatenate of the empty list raises ValueError first.
"""
import os
import sys
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_clean, ref_post  # noqa: E402
from tests.golden_util import save_fixtures  # noqa: E402
from tests.proto import mesh_cc as C  # noqa: E402


FACES_NUMS = (500, 2)            # clean_outliers' default, and a size every crafted piece of two faces or more passes


def _components(edges, nodes, min_len):
    import networkx as nx
    g = nx.Graph()
    g.add_nodes_from(int(n) for n in nodes)
    g.add_edges_from(np.asarray(edges, np.int64).reshape(-1, 2).tolist())
    comps = [np.array(sorted(c), np.int64) for c in nx.connected_components(g) if len(c) >= min_len]
    return sorted(comps, key=lambda c: c[0])


def connected_components(edges, min_len=1, nodes=None, engine=None):
    edges = np.asarray(edges, np.int64).reshape(-1, 2)
    return _components(edges, np.unique(edges) if nodes is None else nodes, min_len)


class Trimesh:
    def __init__(self, vertices=None, faces=None, store=None, process=False, **kw):
        self.vertices = np.array(vertices, np.float64).reshape(-1, 3)
        self.faces = np.array(faces, np.int64).reshape(-1, 3)
        self._store = store

    @property
    def face_adjacency(self):
        slots = {}
        for i, f in enumerate(self.faces.tolist()):
            for a, b in ((f[0], f[1]), (f[1], f[2]), (f[2], f[0])):
                slots.setdefault((min(a, b), max(a, b)), []).append(i)
        pairs = [sorted(s) for s in slots.values() if len(s) == 2 and s[0] != s[1]]
        return np.array(sorted(pairs), np.int64).reshape(-1, 2)

    def split(self, only_watertight=True, **kw):
        assert not only_watertight
        out = []
        for c in _components(self.face_adjacency, range(len(self.faces)), 1):
            f = self.faces[c]
            used = np.unique(f.reshape(-1))
            rank = {int(u): i for i, u in enumerate(used)}
            out.append(Trimesh(self.vertices[used], [[rank[x] for x in r] for r in f.tolist()], self._store))
        return out

    def export(self, path):
        self._store[path] = (np.array(self.vertices), np.array(self.faces))


def trimesh_stub(store):
    tm = types.ModuleType("trimesh")
    tm.load = lambda path, *a, **k: Trimesh(*ref_post._merge(*store[path]), store)
    tm.Trimesh = lambda vertices, faces, *a, **k: Trimesh(vertices, faces, store)
    tm.graph = types.SimpleNamespace(connected_components=connected_components)
    return tm


def run(mod, store, verts, faces, keep_largest, faces_num=500):
    """clean_outliers on the arrays: (exported verts, faces) or the exception as 'Type: message'"""
    store.clear()
    store["in.ply"] = (verts, faces)
    try:
        mod.clean_outliers("in.ply", "out.ply", faces_num=faces_num, keep_largest=keep_largest)
    except Exception as e:
        return "%s: %s" % (type(e).__name__, e)
    return store["out.ply"]


def main():
    store = {}
    mod = ref_clean.load_module(store)
    sys.modules["trimesh"] = mod.trimesh = trimesh_stub(store)
    for name in C.CASES:
        v, f = C.case(name)
        out = dict(in_verts=v, in_faces=f)
        largest = run(mod, store, v, f, True)
        if isinstance(largest, str):
            out["largest_error"] = np.array(largest)
        else:
            out["largest_verts"], out["largest_faces"] = largest
        for n in FACES_NUMS:
            r = run(mod, store, v, f, False, n)
            out["faces_num_error_%d" % n] = np.array(r if isinstance(r, str) else "")
        save_fixtures("cc_" + name, out)
        print(name, len(v), "vertices", len(f), "faces -> largest",
              largest if isinstance(largest, str) else "%d faces" % len(largest[1]),
              "| faces_num:", [str(out["faces_num_error_%d" % n]) for n in FACES_NUMS])


if __name__ == "__main__":
    main()

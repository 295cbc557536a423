"""Golden meshes of the reference's mesh post-processing -- tests/golden/post_<case>.NN.npz.

    python oracle/make_golden_post.py       # needs the staged extract_mesh.py and the compiled reference MC

Each case runs the unmodified get_mesh_udf_fast under oracle/ref_post.py's trimesh stub, the way Runner.extract_udf_mesh
calls it, and stores the mesh after the vertex filter (`in_verts`, `in_faces`: the post-processing's input), the exported
mesh (`out_verts`, `out_faces`), whether the smoothing call succeeded (`smoothed`; the reference falls back to no
smoothing when it raises, as it does for a mesh without border edges) and `nx_disagreements`.

Cases: the five mesh_* fields (tests/proto/mesh_cases.py and the golden scene's network, as oracle/make_golden_mesh.py
meshes them) through the compiled reference MC with dist_threshold_ratio 5, and crafted meshes served as the MC's output
with a zero udf (every face passes the filter):
  holes        a grid with a triangle hole, a quad hole whose shorter diagonal crosses the grid's, a square (equal
               diagonal) hole, and a 5-vertex hole that stays open;
  figure8      two triangle holes that share a vertex: one boundary component through a non-manifold vertex;
  duplicates   faces repeated with the same and with the opposite winding;
  slivers      a repeated vertex index, a vertex merged into another (1e-10 apart), an edge below 1e-8, a height below 1e-8;
  nan          faces on a NaN vertex;
  closed       an octahedron (nothing to fill, nothing to smooth);
  book         three triangles on one edge (a border vertex with three border neighbours) and an isolated triangle, whose
               own boundary is filled with its reverse and then removed as a duplicate inside the loop.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import make_ref_mc, ref_post  # noqa: E402
from tests.golden_util import save_fixtures  # noqa: E402
from tests.proto import mesh_cases as C  # noqa: E402

RATIO = 5.0
CRAFT_N = 8


def _grid(n, h=0.1):
    """an n x n vertex grid in the plane z = 0.05, each cell split along (i, j) -- (i + 1, j + 1)"""
    ij = np.stack(np.meshgrid(np.arange(n), np.arange(n), indexing="ij"), -1).reshape(-1, 2)
    v = np.concatenate([ij * h - 0.5, np.full((len(ij), 1), 0.05)], 1)
    f = []
    for i in range(n - 1):
        for j in range(n - 1):
            a, b, c, d = i * n + j, (i + 1) * n + j, (i + 1) * n + j + 1, i * n + j + 1
            f += [[a, b, c], [a, c, d]]
    return v, np.asarray(f, np.int64)


def _cell(n, i, j):
    return 2 * (i * (n - 1) + j)


def crafted():
    out = {}
    n = 12
    v, f = _grid(n)
    drop = {_cell(n, 1, 1)}                                   # triangle hole
    drop |= {_cell(n, 1, 5), _cell(n, 1, 5) + 1}              # quad hole; its corner (2, 5) pulled out: the other diagonal is shorter
    v[2 * n + 5, :2] += 0.04
    drop |= {_cell(n, 5, 1), _cell(n, 5, 1) + 1}              # square hole: equal diagonals
    drop |= {_cell(n, 5, 6), _cell(n, 5, 6) + 1, _cell(n, 5, 7)}   # a 5-vertex hole
    keep = np.array([i not in drop for i in range(len(f))])
    out["holes"] = (v, f[keep])
    v, f = _grid(8)
    drop = {_cell(8, 2, 2) + 1, _cell(8, 3, 3)}               # touch at vertex (3, 3) only
    out["figure8"] = (v, f[[i not in drop for i in range(len(f))]])
    v, f = _grid(5)
    out["duplicates"] = (v, np.concatenate([f, f[[3]][:, ::-1], np.roll(f[[7]], 1, axis=1), f[[3]], f[[10]][:, [0, 2, 1]]]))
    v, f = _grid(5)
    extra = np.array([[0.123456781, 0.7, 0.3], [0.123456781 + 1e-10, 0.7, 0.3], [0.9, 0.7, 0.3],
                      [0.2, 0.2, 0.6], [0.2 + 5e-9, 0.2, 0.6], [0.4, 0.25, 0.6],
                      [0.1, -0.6, 0.6], [0.3, -0.6, 0.6], [0.5, -0.6 + 4e-9, 0.6]])
    k = len(v)
    v = np.concatenate([v, extra])
    out["slivers"] = (v, np.concatenate([f, [[0, 0, 6]], [[k, k + 1, k + 2]], [[k + 3, k + 4, k + 5]],
                                         [[k + 6, k + 7, k + 8]], [[k, k + 2, k + 5]]]))
    v, f = _grid(6)
    v = np.concatenate([v, [[np.nan, 0.0, 0.0]]])
    out["nan"] = (v, np.concatenate([f, [[len(v) - 1, 0, 1]], [[2, len(v) - 1, 8]]]))
    ov = np.array([[0.3, 0, 0], [-0.3, 0, 0], [0, 0.3, 0], [0, -0.3, 0], [0, 0, 0.3], [0, 0, -0.3]])
    of = np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]])
    out["closed"] = (ov, of)
    bv = np.array([[0, 0, 0], [0, 0.2, 0], [0.2, 0.1, 0], [-0.2, 0.1, 0], [0.05, 0.1, 0.2],
                   [0.5, 0.5, 0.5], [0.6, 0.5, 0.5], [0.5, 0.62, 0.5]])
    out["book"] = (bv, np.array([[0, 1, 2], [1, 0, 3], [0, 1, 4], [5, 6, 7]]))
    return out


def _run_crafted(v, f):
    dummy_df = np.ones(CRAFT_N ** 3, np.float32)
    dummy_n = np.zeros((CRAFT_N ** 3, 3), np.float32)
    mc = lambda volume, grads, spacing=None, **k: (np.asarray(v, np.float64) + 1.0, np.asarray(f, np.int32), None, None)  # noqa: E731
    func = lambda x: torch.zeros(x.shape[0], 1)  # noqa: E731
    return ref_post.run_post(dummy_df, dummy_n, CRAFT_N, mc, func, dist_threshold_ratio=RATIO)


def _save(name, r):
    iv, ifc = r["input"]
    save_fixtures("post_" + name, {"in_verts": iv, "in_faces": ifc, "out_verts": r["verts"], "out_faces": r["faces"],
                                   "smoothed": np.array(r["smoothed"]), "nx_disagreements": np.array(r["nx_disagreements"]),
                                   "ratio": np.array(RATIO)})
    print("%-10s in %6d v %6d f -> out %6d v %6d f  smoothed %s  networkx disagreements %d%s"
          % (name, len(iv), len(ifc), len(r["verts"]), len(r["faces"]), r["smoothed"], r["nx_disagreements"],
             ("  (fallback: %s)" % r["fallback"]) if r.get("fallback") else ""))


def main():
    if not make_ref_mc.verify() and make_ref_mc.stage() is None:
        sys.exit("the compiled reference MC is required (oracle/make_ref_mc.py)")
    ref = make_ref_mc.load()
    from oracle.make_golden_mesh import network_field
    for name in C.CASES:
        df, nrm, N = C.field(name)
        func = lambda x, name=name: torch.from_numpy(C.udf(name, x.numpy().astype(np.float64)).astype(np.float32))[:, None]  # noqa: E731
        _save(name, ref_post.run_post(df, nrm, N, ref.udf_mc_lewiner, func, dist_threshold_ratio=RATIO))
    df, idx, nrm, fn = network_field()
    dense = np.zeros((df.size, 3), np.float32)
    dense[idx] = nrm
    func = lambda x: torch.from_numpy(np.asarray(fn(x.numpy()), np.float32))[:, None]  # noqa: E731
    _save("network", ref_post.run_post(df, dense, 48, ref.udf_mc_lewiner, func, dist_threshold_ratio=RATIO))
    for name, (v, f) in crafted().items():
        _save(name, _run_crafted(v, f))


if __name__ == "__main__":
    main()

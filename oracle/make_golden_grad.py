"""Golden outputs of the reference's gradient branch (extract_mesh.py:267-354) -- tests/golden/grad_<case>.NN.npz.

    python oracle/make_golden_grad.py       # needs the staged extract_mesh.py (oracle/make_ref.py)

Each case runs the unmodified get_mesh_udf_fast on the CPU under oracle/ref_post.py's trimesh stub (through
oracle/ref_grad.py, which keeps the returning call's outputs), the way Runner.extract_udf_mesh calls it (gradient=True,
eps=0.005; border gradients and smoothing, then without them if that raises), with a crafted mesh served as the MC's
output and an analytic torch `func`.  Stored: the mesh the gradient branch saw (`mesh_verts` fp64, `mesh_faces`), the
probe points and func's values there (`p1`, `p2`, `s1`, `s2`: the returning call's two probe calls), `new_verts`,
`next_indices`, `smoothed` (whether the first call returned), `eps` and `N`.

Cases:
  sheet     a grid on the sphere |p| = 0.5 (an open sheet: border edges, smoothed), func = | |p| - 0.5 |;
  closed    a once-subdivided octahedron on the sphere |p| = 0.3 (no border edge: the first call raises), func = | |p| - 0.3 |;
  empty     the sheet with func = 10 everywhere: the vertex filter removes every face (the first call raises, the fallback
            returns an empty mesh);
  lattice   a sheet in the plane x = x0 with its vertices on lattice points, func = |x - x0|: refined vertices land on
            index boundaries;
  network   the post-processing input of tests/golden/post_network (the golden scene's UDF network meshed at 48^3), func
            the CPU oracle's network.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_grad  # noqa: E402
from tests.golden_util import Fixtures, save_fixtures  # noqa: E402

EPS = 0.005
RATIO = 5.0


def _grid_faces(n):
    f = []
    for i in range(n - 1):
        for j in range(n - 1):
            a, b, c, d = i * n + j, (i + 1) * n + j, (i + 1) * n + j + 1, i * n + j + 1
            f += [[a, b, c], [a, c, d]]
    return np.asarray(f, np.int64)


def sphere_sheet(n=12, h=0.3, r=0.5):
    x = np.linspace(-h, h, n)
    xy = np.stack(np.meshgrid(x, x, indexing="ij"), -1).reshape(-1, 2)
    return np.concatenate([xy, np.sqrt(r * r - (xy * xy).sum(1))[:, None]], 1), _grid_faces(n)


def subdivided_octahedron(r=0.3):
    v = [np.array(p, np.float64) for p in ([1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1])]
    faces = [[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]]
    mid = {}

    def m(a, b):
        k = (min(a, b), max(a, b))
        if k not in mid:
            mid[k] = len(v)
            v.append((v[a] + v[b]) / 2)
        return mid[k]

    out = []
    for a, b, c in faces:
        ab, bc, ca = m(a, b), m(b, c), m(c, a)
        out += [[a, ab, ca], [ab, b, bc], [ca, bc, c], [ab, bc, ca]]
    v = np.stack(v)
    return v / np.linalg.norm(v, axis=1, keepdims=True) * r, np.asarray(out, np.int64)


def lattice_sheet(N=32, i0=19, lo=9, n=10):
    voxel = 2.0 / (N - 1)
    jk = np.stack(np.meshgrid(np.arange(lo, lo + n), np.arange(lo, lo + n), indexing="ij"), -1).reshape(-1, 2)
    idx = np.concatenate([np.full((len(jk), 1), i0), jk], 1).astype(np.float32)
    return idx.astype(np.float64) * voxel - 1.0, _grid_faces(n), float(np.float32(i0 * voxel - 1.0))


def _radial(r):
    return lambda x: (torch.linalg.norm(x, dim=1, keepdim=True) - r).abs()


def cases():
    from oracle.make_golden_mesh import network_field
    out = {}
    v, f = sphere_sheet()
    out["sheet"] = (v, f, _radial(0.5), 32)
    v, f = subdivided_octahedron()
    out["closed"] = (v, f, _radial(0.3), 32)
    v, f = sphere_sheet()
    out["empty"] = (v, f, lambda x: torch.full((x.shape[0], 1), 10.0), 32)
    v, f, x0 = lattice_sheet()
    out["lattice"] = (v, f, lambda x: (x[:, :1] - x0).abs(), 32)
    fx = Fixtures("post_network")
    fn = network_field()[3]
    out["network"] = (fx["in_verts"], fx["in_faces"], lambda x: torch.from_numpy(np.asarray(fn(x.numpy()), np.float32))[:, None],
                      48)
    return out


def run_case(v, f, func, N):
    """ref_grad.run_grad on the crafted MC output (v, f) with func, recording func's calls: (its dict, [(input, output)])"""
    calls = []

    def rec(x):
        y = func(x)
        calls.append((x.detach().numpy().copy(), y.detach().reshape(-1).numpy().astype(np.float32)))
        return y

    mc = lambda volume, grads, spacing=None, **k: (np.asarray(v, np.float64) + 1.0, np.asarray(f, np.int32), None, None)  # noqa: E731
    r = ref_grad.run_grad(np.ones(N ** 3, np.float32), np.zeros((N ** 3, 3), np.float32), N, mc, rec,
                          dist_threshold_ratio=RATIO)
    return r, calls


def main():
    for name, (v, f, func, N) in cases().items():
        r, calls = run_case(v, f, func, N)
        (p1, s1), (p2, s2) = calls[-4:-2] if r["smoothed"] else calls[-2:]
        mv, mf = r["mesh"]
        save_fixtures("grad_" + name, {"mesh_verts": mv, "mesh_faces": mf, "p1": p1, "p2": p2, "s1": s1, "s2": s2,
                                       "new_verts": r["new_verts"], "next_indices": r["next_indices"],
                                       "smoothed": np.array(r["smoothed"]), "eps": np.array(EPS), "N": np.array(N)})
        print("%-8s mesh %5d v %5d f  smoothed %-5s  %s" % (name, len(mv), len(mf), r["smoothed"], r["fallback"] or ""))


if __name__ == "__main__":
    main()

"""Golden meshes of the reference's MeshUDF marching cubes -- tests/golden/mesh_<case>.NN.npz.

    python oracle/make_golden_mesh.py       # needs the compiled reference MC (oracle/make_ref_mc.py)

Cases (tests/proto/mesh_cases.py): an analytic sphere (r = 0.5, N = 64), an open square patch at z = 0.1 (N = 64, off the
lattice), the plane z = 0 at N = 65 (exact zeros on the lattice), an open cylinder (garment-like), and the golden scene's
UDF network at N = 48 with df and normals from the CPU oracle (stored: they cannot be regenerated analytically without the
oracle's own rounding).  For each case the reference's raw `udf_mc_lewiner` output (world coordinates, 'descent') and its
faces after the vertex filter of extract_mesh.py:205-214 are stored.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import make_ref_mc  # noqa: E402
from oracle import oracle_torch as O  # noqa: E402
from tests.golden_util import save_fixtures  # noqa: E402
from tests.proto import mesh_cases as C  # noqa: E402

NET_N = 48


def network_field(N=NET_N):
    """(df [N^3] fp32, idx [M] int64, normals [M,3] fp32, udf_fn) of the golden scene's UDF network on the CPU oracle:
    udf on the lattice, normals -normalize(g / (|g| + 1e-5)) where udf < 2 voxels (extract_mesh.py:77-98)."""
    cfg = O.udf_cfg()
    p = O.make_udf_params(cfg, seed=0)
    pts = torch.from_numpy(C.lattice(N)).float()

    def udf_fn(x):
        with torch.no_grad():
            return torch.cat([O.udf_mlp(p, cfg, x[i:i + 65536])[:, 0] for i in range(0, x.shape[0], 65536)])

    df = udf_fn(pts)
    voxel = 2.0 / (N - 1)
    idx = torch.nonzero(df < 2 * voxel).reshape(-1)
    g = O.udf_gradient_autograd(p, cfg, pts[idx], create_graph=False).detach()
    g = g / (torch.linalg.norm(g, ord=2, dim=-1, keepdim=True) + 1e-5)
    nrm = -torch.nn.functional.normalize(g, dim=1)
    return df.numpy(), idx.numpy(), nrm.numpy().astype(np.float32), lambda v: udf_fn(torch.from_numpy(v).float()).numpy()


def reference_mesh(ref, df, nrm_dense, N):
    voxel = 2.0 / (N - 1)
    v, f, _, _ = ref.udf_mc_lewiner(df.reshape(N, N, N), nrm_dense.reshape(N, N, N, 3), spacing=[voxel] * 3)
    return (v - 1).astype(np.float64), np.ascontiguousarray(f, np.int64)


def main():
    if not make_ref_mc.verify() and make_ref_mc.stage() is None:
        sys.exit("the compiled reference MC is required (oracle/make_ref_mc.py)")
    ref = make_ref_mc.load()
    for name in C.CASES:
        df, nrm, N = C.field(name)
        v, f = reference_mesh(ref, df, nrm, N)
        ff = C.vertex_filter(v, f, C.udf(name, v), N)
        save_fixtures("mesh_" + name, {"ref_verts": v, "ref_faces": f, "ref_faces_filtered": ff})
        print(name, len(v), len(f), len(ff), C.mesh_stats(v, ff))
    df, idx, nrm, fn = network_field()
    dense = np.zeros((df.size, 3), np.float32)
    dense[idx] = nrm
    v, f = reference_mesh(ref, df, dense, NET_N)
    ff = C.vertex_filter(v, f, fn(v), NET_N)
    save_fixtures("mesh_network", {"df": df, "idx": idx, "normals": nrm, "ref_verts": v, "ref_faces": f,
                                   "ref_faces_filtered": ff})
    print("network", len(v), len(f), len(ff), C.mesh_stats(v, ff))


if __name__ == "__main__":
    main()

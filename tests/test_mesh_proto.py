"""CPU checks of the MeshUDF marching cubes restated in NumPy (tests/proto/udf_mc.py, the exact oracle of
csrc/mesh_udf.cu): loop construction on random sign grids, and the prototype against the reference's compiled Cython MC
on the golden meshes (tests/golden/mesh_*.npz, oracle/make_golden_mesh.py)."""
import numpy as np
import pytest
import torch

from tests.golden_util import Fixtures
from tests.proto import mesh_cases as C
from tests.proto import udf_mc as P


def _sign_grid_mesh(sign, u):
    """triangulate every cell of a lattice with GLOBAL signs (bit set = negative corner) -> face keys"""
    n = sign.shape[0]
    dims = (n, n, n)
    i, j, k = np.meshgrid(*[np.arange(n - 1)] * 3, indexing="ij")
    cells = (i * n * n + j * n + k).reshape(-1)
    co = cells[:, None] + P.corner_offsets(dims)[None, :]
    neg = sign.reshape(-1)[co] < 0
    mask = (neg.astype(np.int64) << np.arange(8)).sum(1).astype(np.uint8)
    return P.triangulate(u.reshape(-1), dims, cells, mask, u.reshape(-1)[co])


def _directed_edges(f):
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


def _canon(f):
    """rotate each triangle so that its smallest key comes first (keeps the winding)"""
    r = np.argmin(f, axis=1)
    return np.stack([f[np.arange(len(f)), (r + s) % 3] for s in range(3)], 1)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_random_sign_grid_is_closed_two_manifold_and_flip_reverses_winding(seed):
    rng = np.random.default_rng(seed)
    n = 16
    sign = np.where(rng.random((n, n, n)) < 0.5, -1.0, 1.0)
    sign[[0, -1], :, :] = sign[:, [0, -1], :] = sign[:, :, [0, -1]] = 1.0    # keep the surface off the grid border
    u = rng.uniform(0.05, 1.0, (n, n, n)).astype(np.float32)
    f = _sign_grid_mesh(sign, u)
    assert len(f) > 1000
    e = _directed_edges(f)
    und, cnt = np.unique(np.sort(e, 1), axis=0, return_counts=True)
    assert np.all(cnt == 2)                                                 # every edge used exactly twice ...
    assert len(np.unique(e, axis=0)) == len(e)                              # ... once in each direction
    g = _sign_grid_mesh(-sign, u)
    a = _canon(f)
    b = _canon(g[:, ::-1])
    assert np.array_equal(np.unique(a, axis=0), np.unique(b, axis=0))      # same triangles, reversed winding


def test_no_chord_lies_in_a_cube_face():
    """Over every sign pattern and every ambiguous-face decision, no triangle edge other than a loop segment joins two
    vertices on one cube face: such an edge would also belong to the neighbouring cell (non-manifold)."""
    centres = 0
    for pm in range(1, 255):
        for fj in range(64):
            loops = P.cell_loops(pm, fj)
            side = {frozenset((lp[i], lp[(i + 1) % len(lp)])) for lp in loops for i in range(len(lp))}
            tris = P.cell_triangles(pm, fj)
            fanned = [any(P.CENTRE + li in t for t in tris) for li in range(len(loops))]
            assert len(tris) == sum(len(lp) if c else len(lp) - 2 for lp, c in zip(loops, fanned))
            for t in tris:
                for a, b in ((t[0], t[1]), (t[1], t[2]), (t[2], t[0])):
                    if a >= P.CENTRE or b >= P.CENTRE or frozenset((a, b)) in side:
                        continue
                    assert not P.edge_faces(a) & P.edge_faces(b), (pm, fj, a, b)
            centres += sum(1 for t in tris if t[0] >= P.CENTRE)
    assert centres > 0                                                       # the centre fan is exercised


def _proto(name):
    fx = Fixtures("mesh_" + name)
    if name == "network":
        from oracle import oracle_torch as O
        cfg = O.udf_cfg()
        p = O.make_udf_params(cfg, seed=0)
        N, df, idx, nrm = 48, fx["df"], fx["idx"], fx["normals"]

        def ufn(v):
            with torch.no_grad():
                return O.udf_mlp(p, cfg, torch.from_numpy(v).float())[:, 0].numpy()
    else:
        df, nrm, N = C.field(name)
        idx = None

        def ufn(v):
            return C.udf(name, v)
    v, f, info = P.marching_cubes(df, (N, N, N), nrm, idx)
    vw = P.to_world(v, N).astype(np.float64)
    return fx, N, vw, f, C.vertex_filter(vw, f, ufn(vw), N)


def test_sphere_matches_reference():
    fx, N, v, f, _ = _proto("sphere")
    voxel = 2.0 / (N - 1)
    st = C.mesh_stats(v, f)
    assert st["boundary"] == 0 and st["nonmanifold"] == 0 and st["euler"] == 2
    assert st["same_direction"] == 0                                          # consistent winding
    from scipy.spatial import cKDTree
    d, _ = cKDTree(v).query(fx["ref_verts"])
    assert np.mean(d < 1e-4 * voxel) >= 0.99                                 # measured: 1.0
    assert np.abs(np.linalg.norm(v, axis=1) - 0.5).max() < 0.05 * voxel     # measured: 0.0076 voxel
    c = v[f].mean(1)
    nf = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    assert np.all((nf * c).sum(1) > 0)                                      # outwards, as the reference's 'descent'


# (chamfer / voxel, area ratio to the reference, max boundary edges) bounds; measured on the prototype beside them.
# Two samplings of the SAME mesh already give a Chamfer of ~0.2 voxel (20k samples per side).
BOUNDS = {
    "patch": (0.35, (0.95, 1.03), 160),       # measured 0.12, 0.982, 128 (reference: 130)
    "cylinder": (0.35, (0.93, 1.03), 400),    # measured 0.19, 0.958, 328 (reference: 189)
    "network": (0.35, (0.98, 1.02), 10),      # measured 0.16, 1.000, 0   (reference: 0)
}


@pytest.mark.parametrize("name", sorted(BOUNDS))
def test_filtered_mesh_against_reference(name):
    fx, N, v, _, ff = _proto(name)
    voxel = 2.0 / (N - 1)
    rv, rff = fx["ref_verts"], fx["ref_faces_filtered"]
    cd_max, (lo, hi), nb = BOUNDS[name]
    st, rst = C.mesh_stats(v, ff), C.mesh_stats(rv, rff)
    assert C.chamfer(v, ff, rv, rff) / voxel < cd_max
    assert lo < st["area"] / rst["area"] < hi
    assert st["boundary"] <= nb and st["nonmanifold"] == 0


def test_zero_plane_is_finite_and_covers_the_plane():
    """The plane z = 0 through lattice points (exact zeros).  Known deviation from the reference (one sheet, area 4.0):
    the cells on BOTH sides of the plane emit it, so the mesh is two coincident sheets of opposite winding.  Each sheet
    covers the plane within 2 % and the total area is twice the plane's."""
    _, N, v, f, _ = _proto("plane")
    assert np.isfinite(v).all() and len(f) > 0
    assert np.abs(v[:, 2]).max() < 1e-6
    nf = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    up = 0.5 * np.clip(nf[:, 2], 0, None).sum()                               # the sheet facing +z
    down = 0.5 * np.clip(-nf[:, 2], 0, None).sum()                            # the sheet facing -z
    assert abs(up / 4.0 - 1.0) < 0.02 and abs(down / 4.0 - 1.0) < 0.02       # measured: 4.0 each
    assert abs(C.mesh_stats(v, f)["area"] / 8.0 - 1.0) < 0.02                 # measured: 8.0 = two sheets


def test_reference_mc_manifest():
    from oracle import make_ref_mc
    if not make_ref_mc.available():
        pytest.skip("reference MC not built here (needs the reference checkout and Cython)")
    assert make_ref_mc.verify()
    ref = make_ref_mc.load()
    df, nrm, N = C.field("sphere")
    v, f, n, val = ref.udf_mc_lewiner(df.reshape(N, N, N), nrm.reshape(N, N, N, 3))
    assert len(f) == len(Fixtures("mesh_sphere")["ref_faces"])

"""Connected-component mesh filters on the device (neuraludf_b200/clean.py, csrc/mesh_cc.cu): labels and pairing against
the NumPy restatement (tests/proto/mesh_cc.py, scipy components) exactly, on the crafted cases, the C5 network's band
meshes with seeded floating patches, a 2 M-face strip in random face order, 2 M isolated triangles and many equal-size
pieces; clean_outliers in both branches bit for bit; determinism; no host synchronisation in the labelling; the CLI."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.proto import mesh_cc as C

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch.device("cuda", 0)


@pytest.fixture(scope="module")
def c5(golden):
    _dev()
    from tests.gpu_util import build_modules
    return build_modules(golden, "cuda")[0]


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.int64) if a.dtype == np.float64 else a


def _same_mesh(dev_out, proto_out):
    (dv, df), (pv, pf) = dev_out, proto_out
    assert dv.dtype == torch.float64 and df.dtype == torch.int64
    assert np.array_equal(df.cpu().numpy(), pf)
    assert np.array_equal(_bits(dv.cpu().numpy()), _bits(pv))


def _check(verts, faces, dev, faces_nums=(1, 2, 500)):
    """labels, pairing and every filter against the restatement; returns the device labels"""
    from neuraludf_b200 import clean as CL
    v = torch.from_numpy(np.asarray(verts, np.float64)).to(dev)
    f = torch.from_numpy(np.asarray(faces, np.int64)).to(dev)
    label, paired = CL.face_components(f, v)
    pl, pp = C.face_components(faces)
    assert np.array_equal(label.cpu().numpy(), pl) and np.array_equal(paired.cpu().numpy(), pp)
    _same_mesh(CL.keep_largest(v, f), C.keep_largest(verts, faces))
    _same_mesh(CL.clean_outliers(v, f, keep_largest=True), C.clean_outliers(verts, faces, keep_largest=True))
    for n in faces_nums:
        _same_mesh(CL.remove_small_components(v, f, n), C.remove_small_components(verts, faces, n))
        _same_mesh(CL.clean_outliers(v, f, faces_num=n, keep_largest=False),
                   C.clean_outliers(verts, faces, faces_num=n, keep_largest=False))
    return label, paired


@pytest.mark.parametrize("name", C.CASES)
def test_crafted_cases(name):
    dev = _dev()
    v, f = C.case(name)
    _check(v, f, dev)
    from neuraludf_b200 import clean as CL
    if len(f):                                  # the vertex count alone (verts=None) gives the same labels
        label, _ = CL.face_components(torch.from_numpy(f).to(dev))
        assert np.array_equal(label.cpu().numpy(), C.face_components(f)[0])


def _with_floaters(verts, faces, seed):
    """a band mesh plus seeded strips and triangles floating outside it, faces in a seeded random order"""
    rng = np.random.default_rng(seed)
    parts = [(verts, faces)]
    for _ in range(40):
        n = int(rng.integers(1, 600))
        parts.append(C.strip(n, x0=float(rng.uniform(1.5, 3.0)), y0=float(rng.uniform(-3, 3)), z=float(rng.uniform(-3, 3))))
    for _ in range(20):
        parts.append((rng.uniform(-3, -1.5, (3, 3)), np.array([[0, 1, 2]])))
    v, f = C.concat(*parts)
    return v, f[rng.permutation(len(f))]


@pytest.mark.parametrize("N", [256, 512])
def test_band_meshes_with_floaters(c5, N):
    dev = _dev()
    from neuraludf_b200 import clean as CL
    from neuraludf_b200 import grid, mesh
    voxel = 2.0 / (N - 1)
    df, _ = grid.udf_band(c5, N)
    vi, faces = mesh._mc_lattice(c5, N, df, 0, 1 << 21)
    v64 = vi.double() * voxel - 1.0
    vd = c5.udf_values(v64.float()).reshape(-1)
    faces = faces[vd[faces].max(dim=1).values < voxel * 5.0]
    v, f = _with_floaters(v64.cpu().numpy(), faces.cpu().numpy(), seed=N)
    label, paired = _check(v, f, dev, faces_nums=(500,))
    vt, ft = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
    l2, p2 = CL.face_components(ft, vt)
    assert torch.equal(label, l2) and torch.equal(paired, p2)
    a, b = CL.clean_outliers(vt, ft), CL.clean_outliers(vt, ft)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    n_comp = int((label == torch.arange(label.numel(), device=dev)).sum())
    print("C5 band %d^3 + floaters: %d faces, %d components, %d unpaired, largest %d faces"
          % (N, f.shape[0], n_comp, int((paired == 0).sum()), a[1].shape[0]))


def test_permuted_strip():
    """2 M faces in one strip, face order permuted: deep union-find trees"""
    dev = _dev()
    rng = np.random.default_rng(7)
    v, f = C.strip(2_000_000)
    f = f[rng.permutation(len(f))]
    label, paired = _check(v, f, dev, faces_nums=(500, 2_000_001))
    assert int(label.max()) == 0 and bool(paired.all())


def test_isolated_triangles():
    dev = _dev()
    n = 2_000_000
    rng = np.random.default_rng(8)
    v = rng.uniform(-1, 1, (3 * n, 3))
    f = np.arange(3 * n, dtype=np.int64).reshape(n, 3)[rng.permutation(n)]
    label, paired = _check(v, f, dev, faces_nums=(1,))
    assert torch.equal(label, torch.arange(n, device=dev)) and not bool(paired.any())


def test_equal_size_pieces():
    """100 000 strips of 4 faces in random face order: every piece ties, the one holding face 0 is kept"""
    dev = _dev()
    rng = np.random.default_rng(9)
    k = 100_000
    base = C.strip(4)
    v = np.concatenate([base[0] + [3.0 * (i % 300), 3.0 * (i // 300), 0.0] for i in range(k)])
    f = (base[1][None] + 6 * np.arange(k)[:, None, None]).reshape(-1, 3)
    f = f[rng.permutation(len(f))]
    label, _ = _check(v, f, dev, faces_nums=(4, 5))
    assert int((label == torch.arange(label.numel(), device=dev)).sum()) == k


def test_labelling_has_no_host_sync():
    dev = _dev()
    from neuraludf_b200 import clean as CL
    v, f = C.case("floaters")
    vt, ft = torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        keys, key_face = CL._edge_keys(vt, ft)
        label, paired = CL._label_faces(keys, key_face, ft.shape[0])
        keep = CL._largest(label)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert np.array_equal(label.cpu().numpy(), C.face_components(f)[0])
    assert np.array_equal(keep.cpu().numpy(), C.largest_mask(C.face_components(f)[0]))


def test_cli(tmp_path):
    """--outliers on a scan: clean_ and visualhull_ unchanged, final_ = clean_outliers of visualhull_; and on a mesh alone"""
    _dev()
    import cv2
    from neuraludf_b200 import evaluate as E
    from tests.proto import clean_cases as CC
    c = CC.case("sphere")
    scan_dir = tmp_path / "dtu" / ("scan%d" % CC.SCAN)
    os.makedirs(scan_dir / "mask")
    np.savez(str(scan_dir / "cameras.npz"), **{"world_mat_%d" % i: m for i, m in enumerate(c["mats"])})
    for i, m in enumerate(c["masks"]):
        assert cv2.imwrite(str(scan_dir / "mask" / ("%03d.png" % i)), m)
    mesh = str(tmp_path / "mesh.ply")
    E.write_ply_mesh(mesh, c["verts"], c["faces"])
    base = [sys.executable, "-m", "neuraludf_b200.clean", "--mesh", mesh, "--dtu_dir", str(tmp_path / "dtu"), "--scan",
            str(CC.SCAN), "--mask_kernel", str(c["mask_kernel"]), "--minimal_vis", str(c["minimal_vis"]),
            "--imgs_idx"] + [str(i) for i in c["imgs_idx"]]
    run = lambda cmd: subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    outs = {}
    for tag, extra in (("plain", []), ("largest", ["--outliers", "largest"]),
                       ("faces", ["--outliers", "faces", "--faces_num", "50"])):
        r = run(base + ["--out_dir", str(tmp_path / tag)] + extra)
        assert r.returncode == 0, r.stderr[-3000:]
        outs[tag] = sorted(os.listdir(tmp_path / tag))
        for stem in ("clean", "visualhull"):
            name = "%s_%03d.ply" % (stem, CC.SCAN)
            assert open(tmp_path / tag / name, "rb").read() == open(tmp_path / "plain" / name, "rb").read()
    final = "final_%03d.ply" % CC.SCAN
    assert final not in outs["plain"] and final in outs["largest"] and final in outs["faces"]
    hv, hf = E.read_ply(str(tmp_path / "plain" / ("visualhull_%03d.ply" % CC.SCAN)))
    for tag, kw in (("largest", dict(keep_largest=True)), ("faces", dict(keep_largest=False, faces_num=50))):
        v, f = E.read_ply(str(tmp_path / tag / final))
        pv, pf = C.clean_outliers(hv, hf.astype(np.int64), **kw)
        assert np.array_equal(f, pf) and np.array_equal(v, pv)
    # on a mesh alone, as for DeepFashion3D
    fv, ff = C.case("floaters")
    alone = str(tmp_path / "garment.ply")
    E.write_ply_mesh(alone, fv, ff)
    for mode, kw in (("largest", dict(keep_largest=True)), ("faces", dict(keep_largest=False, faces_num=3))):
        out = str(tmp_path / ("alone_%s.ply" % mode))
        r = run([sys.executable, "-m", "neuraludf_b200.clean", "--mesh", alone, "--outliers", mode, "--faces_num", "3",
                 "--out", out])
        assert r.returncode == 0, r.stderr[-3000:]
        v, f = E.read_ply(out)
        pv, pf = C.clean_outliers(*E.read_ply(alone), **kw)
        assert np.array_equal(f, pf) and np.array_equal(v, pv)
    r = run([sys.executable, "-m", "neuraludf_b200.clean", "--mesh", alone])
    assert r.returncode != 0 and "--outliers" in r.stderr

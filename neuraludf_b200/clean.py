"""Mask and visual-hull cleaning of a DTU mesh on the device: the protocol of the reference's
evaluation/clean_dtu_mesh.py without trimesh.

A DTU mesh is cleaned in two passes before evaluation (clean_dtu_mesh.py:194-220):
  mask pass         a vertex is kept when more than `minimal_vis` views see it inside its mask dilated by an ellipse of
                    `mask_kernel` (clean_points_by_mask, :36-68);
  visual-hull pass  a vertex of the first pass's mesh is kept when fewer than 5 views see it, 50 px or more inside the
                    image, outside its mask dilated by an ellipse of `mask_kernel + 20` (clean_points_by_visualhull, :71-105);
each followed by the face filter of clean_mesh_faces_by_{mask,visualhull} (:108-155).  The dilation and the per-vertex vote
are CUDA (csrc/mesh_clean.cu); the face filter and compaction are torch.  tests/proto/mesh_clean.py restates all of it in
NumPy.  The projection runs in one fixed fp64 order (`count_views`); NumPy's matmul may sum in another, which can move a
vertex whose projection lies within rounding of a half-integer pixel to the neighbouring pixel.

Images are any H x W (the reference requires 1600 x 1200 and gives the same result there).  What trimesh does on load and
export (merging vertices, dropping unreferenced ones) is not reproduced: the outputs are the script's arrays.

The script's clean_outliers (:158-191) is here too: `clean_outliers` merges as trimesh.load does, then keeps the largest
connected piece of faces (`keep_largest`) or drops the pieces of fewer than faces_num faces (`remove_small_components`).
The face labelling is CUDA (csrc/mesh_cc.cu); sizes, selection and compaction are torch.  tests/proto/mesh_cc.py restates
it with scipy's connected components.  CLI:

    python -m neuraludf_b200.clean --mesh M.ply --dtu_dir D --scan N [--out_dir O] [--mask_kernel 11] [--minimal_vis 2]
                                   [--imgs_idx I ...] [--outliers {largest,faces} [--faces_num 500]]
    python -m neuraludf_b200.clean --mesh M.ply --outliers {largest,faces} [--faces_num 500] [--out PATH]

With --scan, --outliers also writes final_<scan>.ply, clean_outliers of the visual-hull result; clean_<scan>.ply and
visualhull_<scan>.ply are the same as without it.  Without --dtu_dir / --scan, only clean_outliers runs, on --mesh.
"""
import argparse
import ctypes
import glob
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from neuraludf_b200 import _lib
from neuraludf_b200._lib import check, ptr

# the script's main block and visual-hull constants (clean_dtu_mesh.py:95, 105, 198, 213-217)
MASK_KERNEL, MINIMAL_VIS, HULL_KERNEL_EXTRA, HULL_BORDER, HULL_MAX_OUTSIDE = 11, 2, 20, 50, 5
MAX_KERNEL = 255
FACES_NUM = 500                 # clean_outliers' default (clean_dtu_mesh.py:180)


def ellipse_element(k):
    """OpenCV's MORPH_ELLIPSE structuring element of size k x k as uint8 [k, k]: with r = c = k // 2, row i is set on
    columns [max(c - dx, 0), min(c + dx + 1, k)) where dx = round_half_even(c * sqrt((r^2 - (i - r)^2) / r^2)) and
    |i - r| <= r, empty otherwise; k = 1 is the single pixel."""
    k = int(k)
    if k < 1:
        raise ValueError("kernel size must be positive")
    el = np.zeros((k, k), np.uint8)
    if k == 1:
        el[0, 0] = 1
        return el
    r = c = k // 2
    inv_r2 = 1.0 / float(r * r)
    for i in range(k):
        dy = i - r
        if abs(dy) <= r:
            dx = int(np.rint(c * np.sqrt((r * r - dy * dy) * inv_r2)))
            el[i, max(c - dx, 0):min(c + dx + 1, k)] = 1
    return el


def element_rows(element):
    """(lo, hi) int32 [kh]: the set columns [lo[i], hi[i]) of every row of a 0/1 element (lo == hi: empty row).  Raises
    unless every row is a single interval."""
    el = np.asarray(element) != 0
    if el.ndim != 2 or min(el.shape) < 1 or max(el.shape) > MAX_KERNEL:
        raise ValueError("structuring element must be 2-D with sides in [1, %d]" % MAX_KERNEL)
    lo, hi = np.zeros(el.shape[0], np.int32), np.zeros(el.shape[0], np.int32)
    for i, row in enumerate(el):
        cols = np.nonzero(row)[0]
        if len(cols):
            if cols[-1] - cols[0] + 1 != len(cols):
                raise ValueError("row %d of the structuring element is not one interval" % i)
            lo[i], hi[i] = cols[0], cols[-1] + 1
    return lo, hi


def _device_of(*xs):
    for x in xs:
        if torch.is_tensor(x) and x.is_cuda:
            return x.device
    if not torch.cuda.is_available():
        raise RuntimeError("mesh cleaning runs on a CUDA device")
    return torch.device("cuda", torch.cuda.current_device())


def _masks(masks, dev):
    m = torch.as_tensor(masks).to(dev)
    if m.dtype != torch.uint8 or m.dim() != 3:
        raise ValueError("masks must be uint8 [views, height, width] (channel 0 of each mask image)")
    return m.contiguous()


def _mats(world_mats, dev):
    m = torch.as_tensor(world_mats).to(dev).to(torch.float64)
    if m.dim() != 3 or m.shape[1] not in (3, 4) or m.shape[2] != 4:
        raise ValueError("world_mats must be [views, 3 or 4, 4]")
    return m[:, :3, :].contiguous()


def _points(verts, dev):
    return torch.as_tensor(verts).to(dev).to(torch.float64).reshape(-1, 3).contiguous()


@torch.no_grad()
def dilate_masks(masks, kernel=MASK_KERNEL, below=False):
    """Bit-packed thresholds of the grayscale dilation of masks uint8 [V, H, W] (cv2.dilate with its default border and
    anchor): int32 [V, H, ceil(W / 32)] holding uint32 words, bit b of word w set where column 32 w + b of the dilated mask
    is > 128 (below=False, the mask pass) or < 128 (below=True, the visual-hull pass).  kernel: an ellipse size or a 0/1
    element whose rows are single intervals."""
    dev = _device_of(masks)
    m = _masks(masks, dev)
    el = ellipse_element(kernel) if np.ndim(kernel) == 0 else np.asarray(kernel)
    lo, hi = element_rows(el)
    kh, kw = el.shape
    V, H, W = m.shape
    out = torch.empty(V, H, -(-W // 32), dtype=torch.int32, device=dev)
    c_lo, c_hi = (ctypes.c_int32 * kh)(*lo.tolist()), (ctypes.c_int32 * kh)(*hi.tolist())
    check(_lib.lib().nudf_cl_dilate(ptr(m), V, H, W, c_lo, c_hi, kh, kw, kw // 2, kh // 2, int(bool(below)), ptr(out),
                                    _lib.stream_ptr()), "nudf_cl_dilate")
    return out


def unpack_masks(packed, width):
    """bool [V, H, width] of dilate_masks' packed words"""
    bits = (packed.to(torch.int64)[..., None] >> torch.arange(32, device=packed.device)) & 1
    return bits.reshape(*packed.shape[:-1], -1)[..., :width].bool()


@torch.no_grad()
def count_views(verts, world_mats, packed, height, width, border=0):
    """int32 [N]: the number of views whose packed mask (from dilate_masks) counts each vertex -- the accumulated sum of
    clean_points_by_mask (border=0) or clean_points_by_visualhull (border=50).  A view counts a vertex when its projection
    u = rint(s0 / s2) + 1, v = rint(s1 / s2) + 1, s = P[:3, :3] p + P[:3, 3] in fp64 with each row summed as
    ((P0 x + P1 y) + P2 z) + P3, has border <= u <= width - border and border <= v <= height - border, and the mask padded
    by a ring of ones is set at row v, column u (so with border 0 a projection onto pixel -1 counts)."""
    dev = _device_of(verts, packed)
    p, mats = _points(verts, dev), _mats(world_mats, dev)
    packed = packed.to(dev).contiguous()
    if packed.shape != (mats.shape[0], height, -(-width // 32)):
        raise ValueError("packed masks must be [views, height, ceil(width / 32)] with one view per matrix")
    counts = torch.zeros(p.shape[0], dtype=torch.int32, device=dev)
    check(_lib.lib().nudf_cl_vote(ptr(p), p.shape[0], ptr(mats), mats.shape[0], ptr(packed), int(height), int(width),
                                  int(border), ptr(counts), _lib.stream_ptr()), "nudf_cl_vote")
    return counts


def _pass(verts, world_mats, masks, kernel, below, border):
    dev = _device_of(verts, masks)
    m = _masks(masks, dev)
    packed = dilate_masks(m, kernel, below=below)
    return count_views(verts, world_mats, packed, m.shape[1], m.shape[2], border), packed


def points_in_masks(verts, world_mats, masks, kernel=MASK_KERNEL, minimal_vis=0):
    """clean_points_by_mask: bool [N], the vertices that more than minimal_vis views see inside their mask dilated by an
    ellipse of `kernel` (> 128 after dilation).  masks uint8 [V, H, W], world_mats [V, 3 or 4, 4]."""
    return _pass(verts, world_mats, masks, kernel, False, 0)[0] > minimal_vis


def points_in_visual_hull(verts, world_mats, masks, kernel=MASK_KERNEL + HULL_KERNEL_EXTRA, border=HULL_BORDER,
                          max_outside=HULL_MAX_OUTSIDE):
    """clean_points_by_visualhull: bool [N], the vertices that fewer than max_outside views see, at least `border` pixels
    inside the image, outside their mask dilated by an ellipse of `kernel` (< 128 after dilation)."""
    return _pass(verts, world_mats, masks, kernel, True, border)[0] < max_outside


@torch.no_grad()
def clean_mesh(verts, faces, keep):
    """The face filter of clean_mesh_faces_by_*: (verts[keep], faces) where a face survives when all three of its vertices
    are kept and is re-indexed by the rank of each vertex among the kept ones.  Kept vertices keep their order, including
    kept vertices no face references."""
    keep = torch.as_tensor(keep).to(torch.bool).reshape(-1)
    verts = torch.as_tensor(verts)
    faces = torch.as_tensor(faces).to(keep.device).to(torch.int64).reshape(-1, 3)
    if keep.numel() != verts.shape[0]:
        raise ValueError("keep must have one entry per vertex")
    if faces.numel() and (int(faces.min()) < 0 or int(faces.max()) >= keep.numel()):
        raise ValueError("face index out of range")
    rank = torch.cumsum(keep.to(torch.int64), 0) - 1
    fk = faces[keep[faces].all(dim=1)]
    return verts[keep.to(verts.device)], rank[fk]


@torch.no_grad()
def clean_dtu_mesh(verts, faces, world_mats, masks, mask_kernel=MASK_KERNEL, minimal_vis=MINIMAL_VIS):
    """The script's main block for one scan: the mask pass (kernel mask_kernel, more than minimal_vis views) on the mesh,
    then the visual-hull pass (kernel mask_kernel + 20) on its result.  Returns ((verts, faces, info), (verts, faces, info)),
    the arrays written to clean_%03d.ply and visualhull_%03d.ply; info holds the per-vertex view `counts`, the `keep` mask
    and the `packed` dilated masks of the pass.  Inputs may be device tensors (e.g. udf_mesh output in world space)."""
    dev = _device_of(verts, faces, masks)
    m = _masks(masks, dev)
    mats = _mats(world_mats, dev)
    if mats.shape[0] != m.shape[0]:
        raise ValueError("one world matrix per mask")
    verts = torch.as_tensor(verts).to(dev)
    faces = torch.as_tensor(faces).to(dev)
    stages = []
    for kernel, below, border in ((mask_kernel, False, 0), (mask_kernel + HULL_KERNEL_EXTRA, True, HULL_BORDER)):
        counts, packed = _pass(verts, mats, m, kernel, below, border)
        keep = counts < HULL_MAX_OUTSIDE if below else counts > minimal_vis
        verts, faces = clean_mesh(verts, faces, keep)
        stages.append((verts, faces, dict(counts=counts, keep=keep, packed=packed)))
    return tuple(stages)


def _faces(faces, n_verts, dev):
    f = torch.as_tensor(faces).to(dev).to(torch.int64).reshape(-1, 3).contiguous()
    if f.numel() and (int(f.min()) < 0 or int(f.max()) >= n_verts):
        raise ValueError("face index out of range")
    return f


def _label_faces(keys, key_face, n_faces):
    """csrc/mesh_cc.cu on sorted edge keys and their faces: (label int64 [F], paired uint8 [F]); no host synchronisation"""
    dev = keys.device
    label = torch.empty(n_faces, dtype=torch.int64, device=dev)
    paired = torch.empty(n_faces, dtype=torch.uint8, device=dev)
    check(_lib.lib().nudf_cc_label(ptr(keys), ptr(key_face), keys.numel(), n_faces, ptr(label), ptr(paired),
                                   _lib.stream_ptr()), "nudf_cc_label")
    return label, paired


def _edge_keys(verts, faces):
    """(ascending edge keys lo * V + hi of every face slot, the face of each key): nudf_mp_faces' edge codes, sorted"""
    from neuraludf_b200.mesh_post import _face_pass
    if faces.shape[0] == 0:
        e = torch.empty(0, dtype=torch.int64, device=faces.device)
        return e, e
    codes = _face_pass(verts, faces, None)[2]
    keys, order = torch.sort(codes.reshape(-1) >> 1)
    return keys, order // 3


@torch.no_grad()
def face_components(faces, verts=None):
    """Connected components of the faces under trimesh's face_adjacency: (label int64 [F], the smallest face index of each
    face's component; paired uint8 [F], 1 when the face shares an edge used by exactly two face slots with another face).
    An edge used by one face, or by three or more, joins nothing, and a degenerate face (a, a, b) pairs only with itself,
    which is dropped.  verts: the fp64 [V, 3] the faces index (default: zeros over max(faces) + 1 vertices; only the
    vertex count matters)."""
    dev = _device_of(faces, verts)
    if verts is None:
        f = torch.as_tensor(faces).to(dev)
        verts = torch.zeros(int(f.max()) + 1 if f.numel() else 0, 3, dtype=torch.float64, device=dev)
    verts = _points(verts, dev)
    f = _faces(faces, verts.shape[0], dev)
    keys, key_face = _edge_keys(verts, f)
    return _label_faces(keys, key_face, f.shape[0])


def _sizes(label, count):
    """int64 [F]: at each root, the number of its component's faces where `count` (int64 0/1) is set; 0 elsewhere.  A
    scatter-add rather than torch.bincount, which reads its input's maximum on the host."""
    return torch.zeros_like(label).index_add_(0, label, count)


def _largest(label):
    """faces of the largest component: equal sizes go to the smallest face index (scipy's component order, np.argmax's
    first maximum)"""
    if label.numel() == 0:
        return torch.zeros(0, dtype=torch.bool, device=label.device)
    return label == torch.argmax(_sizes(label, torch.ones_like(label)))


def _at_least(label, paired, faces_num):
    """faces in a pair whose component, counted over the paired faces, has at least faces_num faces"""
    p = paired.bool()
    return p & (_sizes(label, p.to(torch.int64))[label] >= faces_num)


def _submesh(verts, faces, keep):
    """the kept faces in ascending index over the vertices they reference, in ascending index (trimesh submesh)"""
    f = faces[keep]
    used = torch.zeros(verts.shape[0], dtype=torch.bool, device=verts.device)
    used[f.reshape(-1)] = True
    rank = torch.cumsum(used.to(torch.int64), 0) - 1
    return verts[used], rank[f]


def _filter(verts, faces, keep_largest, faces_num):
    dev = _device_of(verts, faces)
    v = _points(verts, dev)
    f = _faces(faces, v.shape[0], dev)
    label, paired = _label_faces(*_edge_keys(v, f), f.shape[0])
    return _submesh(v, f, _largest(label) if keep_largest else _at_least(label, paired, faces_num))


@torch.no_grad()
def keep_largest(verts, faces):
    """trimesh's split(only_watertight=False) followed by the piece with the most faces (clean_outliers, keep_largest=True):
    (fp64 verts, int64 faces).  Every face is a node, so an isolated face is a piece of one face; equal sizes go to the
    piece holding the smallest face index.  The pieces' holes are not filled."""
    return _filter(verts, faces, True, 0)


@torch.no_grad()
def remove_small_components(verts, faces, faces_num=FACES_NUM):
    """What clean_mesh_by_faces_num means to do (the reference's indexing cannot run): keep the faces of every component of
    face_adjacency with at least faces_num faces, counted over the faces in a pair; a face in no pair is dropped."""
    return _filter(verts, faces, False, faces_num)


@torch.no_grad()
def clean_outliers(verts, faces, faces_num=FACES_NUM, keep_largest=True):
    """clean_outliers of clean_dtu_mesh.py: the merge trimesh.load applies (non-finite faces dropped, vertices on one 1e-8
    grid point merged, unreferenced ones dropped), then keep_largest (keep_largest=True) or remove_small_components."""
    from neuraludf_b200.mesh_post import export_merge
    dev = _device_of(verts, faces)
    v = _points(verts, dev)
    v, f = export_merge(v, _faces(faces, v.shape[0], dev))
    return _filter(v, f, keep_largest, faces_num)


def load_dtu_scan(dtu_dir, scan, imgs_idx=None):
    """(world_mats float64 [V, 4, 4], masks uint8 [V, H, W]) of views imgs_idx (default: all 49 views of scans below 83,
    64 above) of <dtu_dir>/scan<scan>: `world_mat_i` of cameras.npz and channel 0 of cv2.imread of the i-th file of
    sorted(mask/*.png), as the script reads them."""
    import cv2
    root = os.path.join(dtu_dir, "scan%d" % scan)
    cams = np.load(os.path.join(root, "cameras.npz"))
    paths = sorted(glob.glob(os.path.join(root, "mask", "*.png")))
    if imgs_idx is None:
        imgs_idx = range(49 if scan < 83 else 64)
    imgs_idx = [int(i) for i in imgs_idx]
    if any(i < 0 or i >= len(paths) for i in imgs_idx):
        raise ValueError("%s has %d masks; views %s requested" % (root, len(paths), imgs_idx))

    def read(i):
        img = cv2.imread(paths[i])
        if img is None:
            raise ValueError("cannot read mask %s" % paths[i])
        return np.ascontiguousarray(img[:, :, 0])

    with ThreadPoolExecutor(max(1, min(8, os.cpu_count() or 1))) as ex:
        masks = list(ex.map(read, imgs_idx))
    if len({m.shape for m in masks}) > 1:
        raise ValueError("the masks of %s differ in size" % root)
    mats = np.stack([np.asarray(cams["world_mat_%d" % i], dtype=np.float64) for i in imgs_idx])
    return mats, np.stack(masks) if masks else np.zeros((0, 0, 0), np.uint8)


def main(argv=None):
    from neuraludf_b200.evaluate import read_ply, write_ply_mesh
    ap = argparse.ArgumentParser(prog="python -m neuraludf_b200.clean", description=__doc__.split("\n\n")[0])
    ap.add_argument("--mesh", required=True, help="mesh to clean, PLY in the scan's world coordinates")
    ap.add_argument("--dtu_dir", default=None, help="directory holding scan<N>/cameras.npz and scan<N>/mask/*.png")
    ap.add_argument("--scan", type=int, default=None)
    ap.add_argument("--out_dir", default=None, help="where clean_<scan>.ply and visualhull_<scan>.ply go (default: beside --mesh)")
    ap.add_argument("--mask_kernel", type=int, default=MASK_KERNEL)
    ap.add_argument("--minimal_vis", type=int, default=MINIMAL_VIS)
    ap.add_argument("--imgs_idx", type=int, nargs="*", default=None, help="views to use (default: all of the scan's)")
    ap.add_argument("--outliers", choices=("largest", "faces"), default=None,
                    help="clean_outliers after the visual-hull pass (written to final_<scan>.ply), or on --mesh alone without "
                         "--dtu_dir / --scan: keep the largest piece, or drop the pieces of fewer than --faces_num faces")
    ap.add_argument("--faces_num", type=int, default=FACES_NUM)
    ap.add_argument("--out", default=None, help="output of --outliers on --mesh alone (default: final_<mesh name> beside it)")
    a = ap.parse_args(argv)
    if (a.dtu_dir is None) != (a.scan is None):
        ap.error("--dtu_dir and --scan go together")
    if a.dtu_dir is None and a.outliers is None:
        ap.error("--dtu_dir and --scan are required unless --outliers cleans --mesh alone")
    if a.dtu_dir is not None and a.out is not None:
        ap.error("--out is for --outliers on --mesh alone; with --dtu_dir the outputs go to --out_dir")
    verts, faces = read_ply(a.mesh)
    if faces is None:
        raise SystemExit("%s has no faces" % a.mesh)

    def outliers(v, f, path):
        v, f = clean_outliers(v, f, faces_num=a.faces_num, keep_largest=a.outliers == "largest")
        write_ply_mesh(path, v, f)
        print("%s: %d vertices, %d faces" % (path, v.shape[0], f.shape[0]))
        return v, f

    if a.dtu_dir is None:
        head, tail = os.path.split(os.path.abspath(a.mesh))
        return outliers(verts, faces, a.out if a.out is not None else os.path.join(head, "final_" + tail))
    mats, masks = load_dtu_scan(a.dtu_dir, a.scan, a.imgs_idx)
    out_dir = a.out_dir if a.out_dir is not None else os.path.dirname(os.path.abspath(a.mesh))
    os.makedirs(out_dir, exist_ok=True)
    stages = clean_dtu_mesh(verts, faces, mats, masks, mask_kernel=a.mask_kernel, minimal_vis=a.minimal_vis)
    for name, (v, f, _) in zip(("clean", "visualhull"), stages):
        path = os.path.join(out_dir, "%s_%03d.ply" % (name, a.scan))
        write_ply_mesh(path, v, f)
        print("%s: %d vertices, %d faces" % (path, v.shape[0], f.shape[0]))
    if a.outliers is not None:
        v, f, _ = stages[1]
        return stages + (outliers(v, f, os.path.join(out_dir, "final_%03d.ply" % a.scan)),)
    return stages


if __name__ == "__main__":
    main()

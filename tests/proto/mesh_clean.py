"""NumPy restatement of the DTU mesh-cleaning protocol (evaluation/clean_dtu_mesh.py:36-155 and its main block :194-220), for
any image size: the exact oracle of neuraludf_b200/clean.py.  The projection is the script's own np.matmul call; the
dilation follows the definition of cv2.dilate (max over the element, anchor at its centre, pixels outside the image not
contributing) with each element row's window max taken from a range-max table, and is held to cv2.dilate by
tests/test_clean_proto.py."""
import numpy as np

from neuraludf_b200.clean import element_rows, ellipse_element


def dilate(img, kernel):
    """uint8 [H, W] grayscale dilation by an ellipse of size `kernel` or a 0/1 element with single-interval rows"""
    el = ellipse_element(kernel) if np.ndim(kernel) == 0 else np.asarray(kernel)
    kh, kw = el.shape
    H, W = img.shape
    pad = np.zeros((H + kh - 1, W + kw - 1), np.uint8)           # pad[r, c] = img[r - kh // 2, c - kw // 2]
    pad[kh // 2:kh // 2 + H, kw // 2:kw // 2 + W] = img
    levels = [pad]                                               # levels[p][r, c] = max(pad[r, c:c + 2^p])
    out = np.zeros((H, W), np.uint8)
    for i, (lo, hi) in enumerate(zip(*element_rows(el))):
        n = int(hi - lo)
        if n <= 0:
            continue
        p = n.bit_length() - 1
        while len(levels) <= p:
            prev, s = levels[-1], 1 << (len(levels) - 1)
            nxt = prev.copy()
            nxt[:, :-s] = np.maximum(prev[:, :-s], prev[:, s:])
            levels.append(nxt)
        M = levels[p]
        a, b = int(lo), int(hi) - (1 << p)
        out = np.maximum(out, np.maximum(M[i:i + H, a:a + W], M[i:i + H, b:b + W]))
    return out


def threshold(dilated, below):
    """the script's `> 128` (mask pass) or `< 128` (visual-hull pass)"""
    return dilated < 128 if below else dilated > 128


def pack(bits):
    """bool [..., W] -> uint32 [..., ceil(W / 32)], bit b of word w = column 32 w + b"""
    W = bits.shape[-1]
    Wp = -(-W // 32)
    padded = np.zeros(bits.shape[:-1] + (Wp * 32,), np.uint8)
    padded[..., :W] = bits
    return np.packbits(padded, axis=-1, bitorder="little").view("<u4")


def project(points, P):
    """the script's pixel indices (u, v) = round(P p / z') + 1 as int32 (clean_dtu_mesh.py:47-49)"""
    with np.errstate(divide="ignore", invalid="ignore"):
        pts_image = np.matmul(P[None, :3, :3], points[:, :, None]).squeeze() + P[None, :3, 3]
        pts_image = pts_image / pts_image[:, 2:]
        pts_image = np.round(pts_image).astype(np.int32) + 1
    return pts_image[:, 0], pts_image[:, 1]


def count_views(points, mats, bits, border):
    """the accumulated counts of clean_points_by_mask (border 0) / clean_points_by_visualhull (border 50); bits: the
    thresholded dilated masks bool [V, H, W]"""
    points = np.asarray(points, np.float64).reshape(-1, 3)
    counts = np.zeros(len(points), np.int64)
    if len(points) == 0:
        return counts
    _, H, W = bits.shape
    for P, m in zip(mats, bits):
        u, v = project(points, np.asarray(P, np.float64))
        padded = np.ones((H + 2, W + 2), bool)
        padded[1:-1, 1:-1] = m
        in_range = (u >= border) & (u <= W - border) & (v >= border) & (v <= H - border)
        counts += padded[v.clip(0, H + 1), u.clip(0, W + 1)] & in_range
    return counts


def clean_mesh(verts, faces, keep):
    """clean_mesh_faces_by_*'s face filter (:113-122)"""
    indexes = (np.ones(len(verts)) * -1).astype(np.int64)
    indexes[np.where(keep)] = np.arange(len(np.where(keep)[0]))
    faces_mask = keep[faces[:, 0]] & keep[faces[:, 1]] & keep[faces[:, 2]]
    new_faces = faces[np.where(faces_mask)]
    for k in range(3):
        new_faces[:, k] = indexes[new_faces[:, k]]
    return verts[np.where(keep)], new_faces


def run_pass(verts, mats, masks, kernel, below, border):
    """(counts, thresholded dilated masks bool [V, H, W]) of one pass"""
    bits = np.stack([threshold(dilate(m, kernel), below) for m in masks])
    return count_views(verts, mats, bits, border), bits


def clean_dtu_mesh(verts, faces, mats, masks, mask_kernel=11, minimal_vis=2):
    """the main block's two stages: [(verts, faces, counts, keep, bits)] * 2"""
    out = []
    for kernel, below, border in ((mask_kernel, False, 0), (mask_kernel + 20, True, 50)):
        counts, bits = run_pass(verts, mats, masks, kernel, below, border)
        keep = counts < 5 if below else counts > minimal_vis
        verts, faces = clean_mesh(verts, faces, keep)
        out.append((verts, faces, counts, keep, bits))
    return out


def half_integer_distance(points, mats):
    """[N]: over all views and both image axes, the smallest distance of the projection P p / z' to a half-integer (the only
    place where the projection's summation order can change a result); NaN projections are ignored"""
    points = np.asarray(points, np.float64).reshape(-1, 3)
    best = np.full(len(points), np.inf)
    with np.errstate(divide="ignore", invalid="ignore"):
        for P in mats:
            P = np.asarray(P, np.float64)
            s = np.matmul(P[None, :3, :3], points[:, :, None])[:, :, 0] + P[None, :3, 3]
            q = s[:, :2] / s[:, 2:]
            d = np.abs(q - np.floor(q) - 0.5).min(axis=1)
            best = np.fmin(best, d)
    return best

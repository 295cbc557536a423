"""Chamfer evaluation of a reconstruction on the device: the DTU and DeepFashion3D protocols of the reference's
evaluation/eval_dtu_python.py and eval_deepfashion_python.py, without open3d.

Stages (each on the device, fp64; kernels in csrc/eval_pc.cu, NumPy restatement in tests/proto/eval_pc.py):
  `sample_mesh`       the scripts' per-triangle surface sampling, bit-identical, vertices first;
  `downsample`        the scripts' greedy radius downsampling in a given (or seeded) shuffle order -- the reference shuffles
                      with an unseeded generator, here the permutation is an input, so a run is reproducible;
  `nearest_distance`  exact nearest distance, +inf where it is >= max_dist (no output of the protocols depends on such a
                      distance's value).
`eval_dtu` / `eval_deepfashion` run a whole protocol and return its metrics; `read_ply` / `write_ply_points` are the PLY I/O the
runner's meshes and the data need.  CLI:

    python -m neuraludf_b200.evaluate {dtu,deepfashion} --data M.ply --gt G.ply [--scan N --dataset_dir D] [--mode mesh|pcd]
                                      [--seed S] [--vis_out_dir V] [--log L]
"""
import argparse
import ctypes
import os
import sys

import numpy as np
import torch

from neuraludf_b200 import _lib
from neuraludf_b200._lib import check, ptr

# the scripts' defaults (eval_dtu_python.py:190-193, eval_deepfashion_python.py:52-55) and F-score thresholds
DTU_DEFAULTS = dict(density=0.2, patch=60.0, max_dist=20.0, visualize_threshold=10.0, thresholds=(1.0, 2.0))
DEEPFASHION_DEFAULTS = dict(density=0.002, max_dist=0.1, visualize_threshold=0.01, thresholds=(0.001, 0.002))
LEAF = 32                          # targets per leaf of the nearest-distance tree (csrc/eval_pc.cu)


def _device(t):
    if t.device.type != "cuda":
        raise ValueError("point-cloud evaluation runs on a CUDA device (got a tensor on %s)" % t.device)
    return t.device


def _points(x, dev=None):
    t = torch.as_tensor(x)
    if dev is not None:
        t = t.to(dev)
    t = t.to(torch.float64).reshape(-1, 3).contiguous()
    return t


def _host3(vals, ctype):
    return (ctype * 3)(*vals)


@torch.no_grad()
def sample_mesh(verts, faces, density):
    """The scripts' surface sampling (eval_dtu_python.py:56-75): [V + S, 3] fp64 -- the vertices, then the samples of every
    triangle with area2 > 0 in triangle order."""
    verts = _points(verts)
    dev = _device(verts)
    faces = torch.as_tensor(faces).to(dev).to(torch.int64).reshape(-1, 3).contiguous()
    if faces.numel() and (int(faces.min()) < 0 or int(faces.max()) >= verts.shape[0]):
        raise ValueError("face index out of range")
    L, st = _lib.lib(), _lib.stream_ptr()
    nf = faces.shape[0]
    counts = torch.zeros(nf, dtype=torch.int64, device=dev)
    check(L.nudf_pc_sample_count(ptr(verts), verts.shape[0], ptr(faces), nf, float(density), ptr(counts), st),
          "nudf_pc_sample_count")
    csum = torch.cumsum(counts, 0)
    n = int(csum[-1]) if nf else 0
    out = torch.empty(verts.shape[0] + n, 3, dtype=torch.float64, device=dev)
    out[:verts.shape[0]] = verts
    if n:
        samples = out[verts.shape[0]:]
        check(L.nudf_pc_sample_emit(ptr(verts), verts.shape[0], ptr(faces), nf, float(density), ptr((csum - counts).contiguous()),
                                    ptr(samples), st), "nudf_pc_sample_emit")
    return out


def seeded_permutation(n, seed):
    """The shuffle order of `np.random.default_rng(seed).shuffle(points, axis=0)`: points[perm]."""
    return np.random.default_rng(seed).permutation(n)


@torch.no_grad()
def downsample(points, radius, perm=None, seed=None):
    """The scripts' greedy radius downsampling (eval_dtu_python.py:85-98) of points in the order points[perm].

    perm: explicit permutation, else drawn from `seed` as the scripts' shuffle would (default seed 0).  Returns
    (kept points [K,3] in shuffled order, info) with info `perm`, `kept_index` (positions in the shuffled order), `rounds`
    (parallel rounds of the independent-set computation) and `edges` (lower-rank pairs within radius)."""
    points = _points(points)
    dev = _device(points)
    n = points.shape[0]
    if perm is None:
        perm = seeded_permutation(n, 0 if seed is None else seed)
    perm = torch.as_tensor(perm).to(dev).to(torch.int64).reshape(-1)
    if perm.numel() != n:
        raise ValueError("perm must have one entry per point")
    info = {"perm": perm, "rounds": 0, "edges": 0}
    sp = points[perm].contiguous()
    if n == 0:
        info["kept_index"] = torch.zeros(0, dtype=torch.int64, device=dev)
        return sp, info
    if not radius > 0:
        raise ValueError("radius must be positive")
    if not bool(torch.isfinite(sp).all()):
        raise ValueError("points must be finite")
    L, st = _lib.lib(), _lib.stream_ptr()
    cell = float(radius) * (1.0 + 1e-6)
    lo_t, hi_t = sp.min(0).values.tolist(), sp.max(0).values.tolist()
    dims = [int(np.floor((h - l) / cell)) + 1 for l, h in zip(lo_t, hi_t)]
    if dims[0] * dims[1] * dims[2] >= 1 << 62:
        raise ValueError("the cloud spans too many radius cells for 64-bit keys")
    lo, dm = _host3(lo_t, ctypes.c_double), _host3(dims, ctypes.c_int64)
    keys = torch.empty(n, dtype=torch.int64, device=dev)
    check(L.nudf_pc_cell_keys(ptr(sp), n, lo, cell, dm, ptr(keys), st), "nudf_pc_cell_keys")
    skeys, order = torch.sort(keys, stable=True)
    ps = sp[order].contiguous()
    cells, ccount = torch.unique_consecutive(skeys, return_counts=True)
    cstart = torch.zeros(cells.numel() + 1, dtype=torch.int64, device=dev)
    cstart[1:] = torch.cumsum(ccount, 0)
    args = (ptr(ps), ptr(order), ptr(skeys), n, ptr(cells), ptr(cstart), cells.numel(), lo, cell, dm, float(radius))
    counts = torch.empty(n, dtype=torch.int32, device=dev)
    check(L.nudf_pc_radius_count(*args, ptr(counts), st), "nudf_pc_radius_count")
    off = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    off[1:] = torch.cumsum(counts, 0)
    n_edges = int(off[-1])
    nbr = torch.empty(max(n_edges, 1), dtype=torch.int32, device=dev)
    check(L.nudf_pc_radius_emit(*args, ptr(off), ptr(nbr), st), "nudf_pc_radius_emit")
    state = torch.empty(n, dtype=torch.uint8, device=dev)
    flag = torch.empty(1, dtype=torch.int32, device=dev)
    rounds = ctypes.c_int32(0)
    check(L.nudf_pc_greedy_mis(ptr(off), ptr(nbr), n, ptr(state), ptr(flag), ctypes.byref(rounds), st), "nudf_pc_greedy_mis")
    kept = torch.nonzero(state == 1).reshape(-1)
    info.update(kept_index=kept, rounds=int(rounds.value), edges=n_edges)
    return sp[kept], info


class NearestIndex:
    """The targets of `nearest_distance`, Morton-sorted into 32-point leaves under an AABB tree; reusable across queries."""

    @torch.no_grad()
    def __init__(self, targets):
        t = _points(targets)
        self.dev = _device(t)
        self.n = t.shape[0]
        if self.n == 0:
            return
        if not bool(torch.isfinite(t).all()):
            raise ValueError("targets must be finite")
        L, st = _lib.lib(), _lib.stream_ptr()
        lo, hi = t.min(0).values, t.max(0).values
        ext = float((hi - lo).max())
        self.lo = _host3(lo.tolist(), ctypes.c_double)
        self.scale = 2097151.0 / ext if ext > 0 else 0.0
        codes = torch.empty(self.n, dtype=torch.int64, device=self.dev)
        check(L.nudf_pc_morton(ptr(t), self.n, self.lo, self.scale, ptr(codes), st), "nudf_pc_morton")
        order = torch.sort(codes, stable=True).indices
        self.targets = t[order].contiguous()
        self.n_leaves = 1 << max(0, int(np.ceil(np.log2(-(-self.n // LEAF)))))
        while self.n_leaves * LEAF < self.n:
            self.n_leaves <<= 1
        self.boxes = torch.empty(2 * self.n_leaves - 1, 6, dtype=torch.float64, device=self.dev)
        check(L.nudf_pc_bvh_build(ptr(self.targets), self.n, self.n_leaves, ptr(self.boxes), st), "nudf_pc_bvh_build")

    @torch.no_grad()
    def query(self, queries, max_dist=float("inf")):
        q = _points(queries, self.dev)
        out = torch.full((q.shape[0],), float("inf"), dtype=torch.float64, device=self.dev)
        if q.shape[0] == 0 or self.n == 0:
            return out
        if not max_dist > 0:
            raise ValueError("max_dist must be positive")
        L, st = _lib.lib(), _lib.stream_ptr()
        codes = torch.empty(q.shape[0], dtype=torch.int64, device=self.dev)
        check(L.nudf_pc_morton(ptr(q), q.shape[0], self.lo, self.scale, ptr(codes), st), "nudf_pc_morton")
        qorder = torch.sort(codes, stable=True).indices.contiguous()
        check(L.nudf_pc_nearest(ptr(q), q.shape[0], ptr(qorder), ptr(self.targets), self.n, ptr(self.boxes), self.n_leaves,
                                float(max_dist), ptr(out), st), "nudf_pc_nearest")
        return out


def nearest_distance(queries, targets, max_dist=float("inf")):
    """[Q] fp64: exact distance from every query to its nearest target (the KD-tree's sqrt((dx^2 + dy^2) + dz^2)) where it is
    below max_dist, +inf elsewhere (and everywhere when there are no targets)."""
    return NearestIndex(targets).query(queries, max_dist)


def _metrics(d2s, s2d, max_dist, thresholds):
    """means over d < max_dist, over_all, precision / recall / F-score at the thresholds (eval_dtu_python.py:303-348)"""
    mean_d2s = float(d2s[d2s < max_dist].mean()) if d2s.numel() else float("nan")
    mean_s2d = float(s2d[s2d < max_dist].mean()) if s2d.numel() else float("nan")
    out = {"mean_d2gt": mean_d2s, "mean_gt2d": mean_s2d, "over_all": (mean_d2s + mean_s2d) / 2}
    for k, t in enumerate(thresholds, 1):
        p = int((d2s < t).sum()) / d2s.numel() if d2s.numel() else float("nan")
        r = int((s2d < t).sum()) / s2d.numel() if s2d.numel() else float("nan")
        out["precision_%d" % k], out["recall_%d" % k] = p, r
        out["fscore_%d" % k] = 2 * p * r / (p + r + 1e-6)
    return out


_RED, _GREEN, _BLUE, _WHITE = (1., 0., 0.), (0., 1., 0.), (0., 0., 1.), (1., 1., 1.)


def _error_colors(d, vis, max_dist, dev):
    """R * alpha + W * (1 - alpha), alpha = min(d, vis) / vis; green where d >= max_dist"""
    R = torch.tensor([_RED], dtype=torch.float64, device=dev)
    W = torch.tensor([_WHITE], dtype=torch.float64, device=dev)
    alpha = (d.clamp(max=vis) / vis)[:, None]
    c = R * alpha + W * (1 - alpha)
    c[d >= max_dist] = torch.tensor(_GREEN, dtype=torch.float64, device=dev)
    return c


def _blue(n, dev):
    return torch.tensor([_BLUE], dtype=torch.float64, device=dev).repeat(n, 1)


def _cloud(data, faces, density, dev):
    data = _points(data, dev)
    return data if faces is None else sample_mesh(data, faces, density)


@torch.no_grad()
def eval_dtu(data, faces, gt, obs_mask, bb, res, plane, density=0.2, patch=60.0, max_dist=20.0, visualize_threshold=10.0,
             thresholds=(1.0, 2.0), perm=None, seed=None, colors=False, device=None):
    """The DTU protocol (eval_dtu_python.py:40-175 and the metrics of its main block).

    data / faces: mesh vertices [V,3] and faces [F,3] (faces None: data is a point cloud, `--mode pcd`); gt: the STL cloud;
    obs_mask [X,Y,Z], bb [2,3], res, plane [4]: the scan's ObsMask / BB / Res and ground plane P.  Tensors may already be on
    the device.  Returns a dict: mean_d2gt, mean_gt2d, over_all, precision_k / recall_k / fscore_k (k = 1, 2 for the two
    thresholds), the counts n_points, n_down, n_in, n_in_obs, n_gt, n_gt_above, downsample_rounds, and with colors=True the
    vis clouds data_down / data_color and gt / gt_color of vis_XXX_d2gt.ply / vis_XXX_gt2d.ply."""
    dev = torch.device(device) if device is not None else (data.device if torch.is_tensor(data) and data.is_cuda
                                                           else torch.device("cuda", torch.cuda.current_device()))
    pcd = _cloud(data, faces, density, dev)
    down, dinfo = downsample(pcd, density, perm=perm, seed=seed)
    # in-bound test against BB cast to fp32, its margins computed in fp32 as NumPy does (eval_dtu_python.py:104-107)
    BB = np.asarray(torch.as_tensor(bb).cpu().numpy(), dtype=np.float32).reshape(2, 3)
    lo = torch.from_numpy((BB[:1] - patch).astype(np.float64)).to(dev)
    hi = torch.from_numpy((BB[1:] + patch * 2).astype(np.float64)).to(dev)
    inbound = ((down >= lo) & (down < hi)).all(dim=1)
    data_in = down[inbound]
    res = float(np.asarray(torch.as_tensor(res).cpu().numpy(), dtype=np.float64).reshape(-1)[0])
    bb0 = torch.from_numpy(BB[:1].astype(np.float64)).to(dev)
    grid = torch.round((data_in - bb0) / res).to(torch.int32)           # np.around: half to even
    obs = torch.as_tensor(obs_mask).to(dev)
    shape = torch.tensor(list(obs.shape), dtype=torch.int32, device=dev)
    grid_inbound = ((grid >= 0) & (grid < shape)).all(dim=1)
    gi = grid[grid_inbound].long()
    in_obs = obs[gi[:, 0], gi[:, 1], gi[:, 2]] != 0
    data_in_obs = data_in[grid_inbound][in_obs]
    stl = _points(gt, dev)
    d2s = nearest_distance(data_in_obs, stl, max_dist)
    # ground plane (eval_dtu_python.py:130-134): ((P0 x + P1 y) + P2 z) + P3 > 0, one rounding per operation
    P = [float(v) for v in np.asarray(torch.as_tensor(plane).cpu().numpy(), dtype=np.float64).reshape(4)]
    s = stl[:, 0] * P[0]
    s = s + stl[:, 1] * P[1]
    s = s + stl[:, 2] * P[2]
    above = (s + P[3]) > 0
    s2d = nearest_distance(stl[above], data_in, max_dist)
    out = _metrics(d2s, s2d, max_dist, thresholds)
    out.update(n_points=pcd.shape[0], n_down=down.shape[0], n_in=data_in.shape[0], n_in_obs=data_in_obs.shape[0],
               n_gt=stl.shape[0], n_gt_above=int(above.sum()), downsample_rounds=dinfo["rounds"])
    if colors:
        dc = _blue(down.shape[0], dev)
        idx = torch.nonzero(inbound).reshape(-1)[grid_inbound][in_obs]
        dc[idx] = _error_colors(d2s, visualize_threshold, max_dist, dev)
        gc = _blue(stl.shape[0], dev)
        gc[torch.nonzero(above).reshape(-1)] = _error_colors(s2d, visualize_threshold, max_dist, dev)
        out.update(data_down=down, data_color=dc, gt=stl, gt_color=gc)
    out["stages"] = dict(data_pcd=pcd, downsample=dinfo, inbound=inbound, grid_inbound=grid_inbound, in_obs=in_obs, above=above,
                          dist_d2s=d2s, dist_s2d=s2d)
    return out


@torch.no_grad()
def eval_deepfashion(data, faces, gt, density=0.002, max_dist=0.1, visualize_threshold=0.01, thresholds=(0.001, 0.002),
                     perm=None, seed=None, colors=False, device=None):
    """The DeepFashion3D protocol (eval_deepfashion_python.py:87-198): no mask and no plane, data_down <-> all of the GT.
    Arguments and result as `eval_dtu` (counts n_points, n_down, n_gt)."""
    dev = torch.device(device) if device is not None else (data.device if torch.is_tensor(data) and data.is_cuda
                                                           else torch.device("cuda", torch.cuda.current_device()))
    pcd = _cloud(data, faces, density, dev)
    down, dinfo = downsample(pcd, density, perm=perm, seed=seed)
    stl = _points(gt, dev)
    d2s = nearest_distance(down, stl, max_dist)
    s2d = nearest_distance(stl, down, max_dist)
    out = _metrics(d2s, s2d, max_dist, thresholds)
    out.update(n_points=pcd.shape[0], n_down=down.shape[0], n_gt=stl.shape[0], downsample_rounds=dinfo["rounds"])
    if colors:
        out.update(data_down=down, data_color=_error_colors(d2s, visualize_threshold, max_dist, dev), gt=stl,
                   gt_color=_error_colors(s2d, visualize_threshold, max_dist, dev))
    out["stages"] = dict(data_pcd=pcd, downsample=dinfo, dist_d2s=d2s, dist_s2d=s2d)
    return out


# ---- PLY -------------------------------------------------------------------------------------------------------------------
_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
              "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4",
              "double": "f8", "float64": "f8"}


def _parse_header(f):
    if f.readline().strip() != b"ply":
        raise ValueError("not a PLY file")
    fmt, elements = None, []
    while True:
        line = f.readline()
        if not line:
            raise ValueError("PLY header has no end_header")
        tok = line.decode("ascii", "replace").split()
        if not tok or tok[0] in ("comment", "obj_info"):
            continue
        if tok[0] == "end_header":
            break
        if tok[0] == "format":
            if tok[1] not in ("ascii", "binary_little_endian") or tok[2] != "1.0":
                raise ValueError("unsupported PLY format %s %s (ascii and binary_little_endian 1.0 only)" % (tok[1], tok[2]))
            fmt = tok[1]
        elif tok[0] == "element":
            elements.append((tok[1], int(tok[2]), []))
        elif tok[0] == "property":
            if tok[1] == "list":
                elements[-1][2].append((tok[4], _PLY_TYPES[tok[2]], _PLY_TYPES[tok[3]]))
            else:
                elements[-1][2].append((tok[2], _PLY_TYPES[tok[1]], None))
    if fmt is None:
        raise ValueError("PLY header has no format line")
    return fmt, elements


def _read_binary_element(buf, pos, count, props):
    """(dict name -> array, new pos); list properties of one common length take a fast path, others are parsed row by row"""
    if all(p[2] is None for p in props):
        dt = np.dtype([(n, "<" + t) for n, t, _ in props])
        a = np.frombuffer(buf, dt, count, pos)
        return {n: a[n] for n, _, _ in props}, pos + count * dt.itemsize
    if count:
        # assume every list has the length of the first row's, then verify
        fields, p = [], pos
        for n, t, lt in props:
            if lt is None:
                fields.append((n, "<" + t))
                p += np.dtype(t).itemsize
            else:
                k = int(np.frombuffer(buf, "<" + t, 1, p)[0])
                fields += [(n + "#n", "<" + t), (n, "<" + lt, (k,))]
                p += np.dtype(t).itemsize + k * np.dtype(lt).itemsize
        dt = np.dtype(fields)
        if pos + count * dt.itemsize <= len(buf):
            a = np.frombuffer(buf, dt, count, pos)
            if all((a[n + "#n"] == dt[n].shape[0]).all() for n, _, lt in props if lt is not None):
                return {n: a[n] for n, _, _ in props}, pos + count * dt.itemsize
    out = {n: [] for n, _, _ in props}
    for _ in range(count):
        for n, t, lt in props:
            if lt is None:
                out[n].append(np.frombuffer(buf, "<" + t, 1, pos)[0])
                pos += np.dtype(t).itemsize
            else:
                k = int(np.frombuffer(buf, "<" + t, 1, pos)[0])
                pos += np.dtype(t).itemsize
                out[n].append(np.frombuffer(buf, "<" + lt, k, pos))
                pos += k * np.dtype(lt).itemsize
    return {n: (v if lt is not None else np.array(v)) for (n, _, lt), v in zip(props, out.values())}, pos


def _read_ascii_element(lines, count, props):
    rows = [lines.pop() for _ in range(count)]
    if all(p[2] is None for p in props):
        a = np.array(" ".join(rows).split(), dtype=np.float64).reshape(count, len(props)) if count else np.zeros((0, len(props)))
        return {n: a[:, i] for i, (n, _, _) in enumerate(props)}
    out = {n: [] for n, _, _ in props}
    for r in rows:
        tok, i = r.split(), 0
        for n, _, lt in props:
            if lt is None:
                out[n].append(float(tok[i]))
                i += 1
            else:
                k = int(float(tok[i]))
                out[n].append(np.array(tok[i + 1:i + 1 + k], dtype=np.int64))
                i += 1 + k
    return out


def read_ply(path):
    """(vertices [V,3] fp64, faces [F,3] int64 or None) of a PLY file: ascii or binary_little_endian 1.0, vertex x / y / z
    of any scalar type (other vertex properties skipped), faces as a list property (vertex_indices or vertex_index).
    Other elements are skipped; faces must be triangles."""
    with open(path, "rb") as f:
        fmt, elements = _parse_header(f)
        body = f.read()
    data, pos = {}, 0
    if fmt == "ascii":
        lines = [l for l in body.decode("ascii").splitlines() if l.strip()][::-1]
    for name, count, props in elements:
        if fmt == "ascii":
            data[name] = _read_ascii_element(lines, count, props)
        else:
            data[name], pos = _read_binary_element(body, pos, count, props)
    if "vertex" not in data or not all(k in data["vertex"] for k in "xyz"):
        raise ValueError("PLY file has no vertex x / y / z")
    v = data["vertex"]
    verts = np.stack([np.asarray(v[k], dtype=np.float64) for k in "xyz"], axis=1).reshape(-1, 3)
    faces = None
    if "face" in data:
        fd = data["face"]
        key = "vertex_indices" if "vertex_indices" in fd else ("vertex_index" if "vertex_index" in fd else None)
        if key is None:
            raise ValueError("PLY face element has no vertex_indices list")
        lst = fd[key]
        if isinstance(lst, np.ndarray) and lst.ndim == 2:
            faces = lst.astype(np.int64)
        else:
            if any(len(x) != 3 for x in lst):
                raise ValueError("only triangle faces are supported")
            faces = np.array(lst, dtype=np.int64).reshape(-1, 3)
        if faces.ndim != 2 or (faces.shape[0] and faces.shape[1] != 3):
            raise ValueError("only triangle faces are supported")
        faces = faces.reshape(-1, 3)
    return verts, faces


def write_ply_points(path, points, colors=None, ascii=False):
    """A point cloud as PLY: double x / y / z and, with colors in [0,1], uchar red / green / blue (round(255 c))."""
    pts = np.ascontiguousarray(torch.as_tensor(points).detach().cpu().numpy(), dtype=np.float64).reshape(-1, 3)
    head = ["ply", "format %s 1.0" % ("ascii" if ascii else "binary_little_endian"), "element vertex %d" % len(pts),
            "property double x", "property double y", "property double z"]
    fields = [("x", "<f8"), ("y", "<f8"), ("z", "<f8")]
    rgb = None
    if colors is not None:
        c = np.asarray(torch.as_tensor(colors).detach().cpu().numpy(), dtype=np.float64).reshape(-1, 3)
        if len(c) != len(pts):
            raise ValueError("colors must have one row per point")
        rgb = np.clip(np.round(c * 255.0), 0, 255).astype(np.uint8)
        head += ["property uchar red", "property uchar green", "property uchar blue"]
        fields += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    head.append("end_header")
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode("ascii"))
        if ascii:
            for i in range(len(pts)):
                row = ["%r" % float(x) for x in pts[i]] + ([str(int(x)) for x in rgb[i]] if rgb is not None else [])
                f.write((" ".join(row) + "\n").encode("ascii"))
        else:
            a = np.empty(len(pts), dtype=np.dtype(fields))
            a["x"], a["y"], a["z"] = pts[:, 0], pts[:, 1], pts[:, 2]
            if rgb is not None:
                a["red"], a["green"], a["blue"] = rgb[:, 0], rgb[:, 1], rgb[:, 2]
            f.write(a.tobytes())


def read_ply_colors(path):
    """The red / green / blue vertex properties of a PLY point cloud as uint8 [V,3] (None when absent)."""
    with open(path, "rb") as f:
        fmt, elements = _parse_header(f)
        body = f.read()
    name, count, props = elements[0]
    if fmt == "ascii":
        d = _read_ascii_element([l for l in body.decode("ascii").splitlines() if l.strip()][::-1], count, props)
    else:
        d = _read_binary_element(body, 0, count, props)[0]
    if not all(k in d for k in ("red", "green", "blue")):
        return None
    return np.stack([np.asarray(d[k]).astype(np.uint8) for k in ("red", "green", "blue")], axis=1)


# ---- CLI -------------------------------------------------------------------------------------------------------------------
def _result_lines(r):
    return ["over_all: %s; mean_d2gt: %s; mean_gt2d: %s." % (r["over_all"], r["mean_d2gt"], r["mean_gt2d"]),
            "precision_1mm: %s;  recall_1mm: %s;  fscore_1mm: %s" % (r["precision_1"], r["recall_1"], r["fscore_1"]),
            "precision_2mm: %s;  recall_2mm: %s;  fscore_2mm: %s" % (r["precision_2"], r["recall_2"], r["fscore_2"])]


def format_log(r, stem, digits):
    """the main block's log (eval_dtu_python.py:359-369: 3 digits, eval_deepfashion_python.py:205-215: 6 digits)"""
    rd = lambda k: np.round(np.float64(r[k]), digits)  # noqa: E731
    return (f"over_all {rd('over_all')} mean_d2gt {rd('mean_d2gt')} mean_gt2d {rd('mean_gt2d')} \n"
            f"precision_1mm {rd('precision_1')} recall_1mm {rd('recall_1')} fscore_1mm {rd('fscore_1')} \n"
            f"precision_2mm {rd('precision_2')} recall_2mm {rd('recall_2')} fscore_2mm {rd('fscore_2')} \n"
            f"[{stem}] \n")


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m neuraludf_b200.evaluate", description=__doc__.split("\n\n")[0])
    ap.add_argument("protocol", choices=["dtu", "deepfashion"])
    ap.add_argument("--data", required=True, help="reconstructed mesh (or point cloud with --mode pcd), PLY")
    ap.add_argument("--gt", required=True, help="ground-truth point cloud, PLY")
    ap.add_argument("--scan", type=int, default=1)
    ap.add_argument("--mode", default="mesh", choices=["mesh", "pcd"])
    ap.add_argument("--dataset_dir", default=".", help="DTU: the directory holding ObsMask/ObsMask<scan>_10.mat and Plane<scan>.mat")
    ap.add_argument("--vis_out_dir", default=None, help="write vis_<scan>_d2gt.ply / vis_<scan>_gt2d.ply there")
    ap.add_argument("--downsample_density", type=float, default=None)
    ap.add_argument("--patch_size", type=float, default=60.0)
    ap.add_argument("--max_dist", type=float, default=None)
    ap.add_argument("--visualize_threshold", type=float, default=None)
    ap.add_argument("--seed", type=int, default=0, help="seed of the shuffle before downsampling")
    ap.add_argument("--log", default=None, help="log file (default: eval_result.txt beside --data)")
    a = ap.parse_args(argv)
    dflt = DTU_DEFAULTS if a.protocol == "dtu" else DEEPFASHION_DEFAULTS
    density = dflt["density"] if a.downsample_density is None else a.downsample_density
    max_dist = dflt["max_dist"] if a.max_dist is None else a.max_dist
    vis = dflt["visualize_threshold"] if a.visualize_threshold is None else a.visualize_threshold
    verts, faces = read_ply(a.data)
    if a.mode == "mesh" and faces is None:
        sys.exit("--mode mesh needs a PLY with faces: %s" % a.data)
    faces = faces if a.mode == "mesh" else None
    gt, _ = read_ply(a.gt)
    kw = dict(density=density, max_dist=max_dist, visualize_threshold=vis, seed=a.seed, colors=a.vis_out_dir is not None)
    if a.protocol == "dtu":
        from scipy.io import loadmat
        m = loadmat(os.path.join(a.dataset_dir, "ObsMask", "ObsMask%d_10.mat" % a.scan))
        plane = loadmat(os.path.join(a.dataset_dir, "ObsMask", "Plane%d.mat" % a.scan))["P"]
        r = eval_dtu(verts, faces, gt, m["ObsMask"], m["BB"], m["Res"], plane, patch=a.patch_size, **kw)
    else:
        r = eval_deepfashion(verts, faces, gt, **kw)
    if a.vis_out_dir is not None:
        os.makedirs(a.vis_out_dir, exist_ok=True)
        write_ply_points(os.path.join(a.vis_out_dir, f"vis_{a.scan:03}_d2gt.ply"), r["data_down"], r["data_color"])
        write_ply_points(os.path.join(a.vis_out_dir, f"vis_{a.scan:03}_gt2d.ply"), r["gt"], r["gt_color"])
    for line in _result_lines(r):
        print(line)
    stem = os.path.splitext(os.path.basename(a.data))[0]
    log = a.log if a.log is not None else os.path.join(os.path.dirname(os.path.abspath(a.data)), "eval_result.txt")
    with open(log, "w+") as f:
        f.write(format_log(r, stem, 3 if a.protocol == "dtu" else 6))
    return r


if __name__ == "__main__":
    main()

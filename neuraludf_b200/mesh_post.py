"""The runner's mesh post-processing on the device: what get_mesh_udf_fast does after the vertex filter
(extract_mesh.py:215-265) and what the runner's last `trimesh.Trimesh(...)` does before export (exp_runner_blending.py:796).

trimesh's primitives are restated as rules (DESIGN.md §1, "mesh post-processing"), all geometry in fp64:
  non-finite   faces with a non-finite vertex are dropped;
  merge        referenced vertices with equal round-half-even(x 1e8) in all three coordinates become one, which keeps the
               coordinates of the lowest-indexed member; merged vertices are numbered in the order of those members and
               unreferenced vertices are dropped;
  duplicates   faces with the same sorted vertex triple, whatever their winding: the first in face order stays;
  degenerate   a = v1 - v0, b = v2 - v0: a face stays when |a|, |b|, |a x b| / |a| and |a x b| / |b| all exceed 1e-8;
  holes        a boundary component (edges used by one face) that is a simple cycle of 3 or 4 vertices gets one or two
               faces, which traverse the boundary against the existing faces (the cycle's smallest edge decides);
  smoothing    5 Jacobi steps v + 0.3 (mean of the border neighbours - v) over the border vertices.
The kernels are in csrc/mesh_post.cu; sorting, unique and compaction run in torch.  tests/proto/mesh_post.py restates
the whole of it in NumPy, bit for bit.
"""
import torch

from neuraludf_b200 import _lib
from neuraludf_b200._lib import check, ptr

MERGE_SCALE = 1e8               # trimesh tol.merge = 1e-8
SMOOTH_LAMBDA = 0.3
SMOOTH_STEPS = 5
MAX_PASSES = 10


def _i64(*shape, dev):
    return torch.empty(*shape, dtype=torch.int64, device=dev)


def drop_nonfinite(verts, faces):
    """the faces whose three vertices are finite"""
    if faces.shape[0] == 0:
        return faces
    ok = torch.isfinite(verts).all(1)
    return faces[ok[faces].all(1)]


def merge_remap(verts, faces):
    """(merged verts, remap [V] int64: new index or -1 for an unreferenced vertex) of the merge rule"""
    dev = verts.device
    V = verts.shape[0]
    used = torch.zeros(V, dtype=torch.bool, device=dev)
    used[faces.reshape(-1)] = True
    ref = torch.nonzero(used).reshape(-1)
    remap = torch.full((V,), -1, dtype=torch.int64, device=dev)
    if ref.numel() == 0:
        return verts[:0], remap
    x = verts[ref] * MERGE_SCALE
    if not bool((x.abs() < 2.0 ** 62).all()):
        raise ValueError("vertex coordinates too large for the 1e-8 merge grid")
    keys = torch.round(x).to(torch.int64)                       # half to even, as np.round
    _, inv = torch.unique(keys, dim=0, return_inverse=True)
    n = int(inv.max()) + 1
    rep = torch.full((n,), V, dtype=torch.int64, device=dev).scatter_reduce(0, inv, ref, "amin")
    rep_sorted, order = torch.sort(rep)
    rank = torch.empty_like(order)
    rank[order] = torch.arange(n, device=dev)
    remap[ref] = rank[inv]
    return verts[rep_sorted], remap


def _face_pass(verts, faces, remap):
    """csrc/mesh_post.cu face pass: (remapped faces, sorted triples, edge codes [F,3], nondegenerate [F] bool)"""
    dev = verts.device
    F = faces.shape[0]
    out, srt, codes = _i64(F, 3, dev=dev), _i64(F, 3, dev=dev), _i64(F, 3, dev=dev)
    nondeg = torch.empty(F, dtype=torch.uint8, device=dev)
    check(_lib.lib().nudf_mp_faces(ptr(verts), verts.shape[0], ptr(faces), F, ptr(remap), ptr(out), ptr(srt), ptr(codes),
                                   ptr(nondeg), _lib.stream_ptr()), "nudf_mp_faces")
    return out, srt, codes, nondeg.bool()


def _first_unique(srt):
    """mask of the first face of each sorted triple"""
    F = srt.shape[0]
    _, inv = torch.unique(srt, dim=0, return_inverse=True)
    ar = torch.arange(F, device=srt.device)
    first = torch.full((int(inv.max()) + 1,), F, dtype=torch.int64, device=srt.device).scatter_reduce(0, inv, ar, "amin")
    keep = torch.zeros(F, dtype=torch.bool, device=srt.device)
    keep[first] = True
    return keep


def process(verts, faces):
    """non-finite, merge, duplicates, degenerate: (verts, faces, edge codes of the kept faces, counts)"""
    dev = verts.device
    f = drop_nonfinite(verts, faces)
    counts = {"nonfinite": int(faces.shape[0] - f.shape[0]), "duplicate": 0, "degenerate": 0}
    v, remap = merge_remap(verts, f)
    if f.shape[0] == 0:
        return v, f.reshape(0, 3), _i64(0, 3, dev=dev), counts
    f = f.contiguous()
    f, srt, codes, nondeg = _face_pass(v, f, remap)
    keep = _first_unique(srt)
    counts["duplicate"] = int(f.shape[0] - int(keep.sum()))
    f, codes, nondeg = f[keep], codes[keep], nondeg[keep]
    counts["degenerate"] = int(f.shape[0] - int(nondeg.sum()))
    return v, f[nondeg], codes[nondeg], counts


def _compact(verts, faces):
    """merge that can only drop unreferenced vertices (the coordinates are merged already)"""
    v, remap = merge_remap(verts, faces)
    return v, remap[faces]


def _codes(verts, faces):
    _, _, codes, _ = _face_pass(verts, faces.contiguous(), None)
    return codes


def boundary(codes, n_verts):
    """(edges [B,2] ascending, dirs [B] uint8, rowptr [V+1], cols) of the edges used by one face, from their edge codes"""
    dev = codes.device
    c, _ = torch.sort(codes.reshape(-1))
    key = c >> 1
    _, cnt = torch.unique_consecutive(key, return_counts=True)
    start = torch.cumsum(cnt, 0) - cnt
    b = c[start[cnt == 1]]
    k = b >> 1
    edges = torch.stack([k // n_verts, k % n_verts], 1).contiguous()
    dirs = (b & 1).to(torch.uint8).contiguous()
    src = torch.cat([edges[:, 0], edges[:, 1]])
    dst = torch.cat([edges[:, 1], edges[:, 0]])
    order = torch.argsort(src * n_verts + dst)
    rowptr = torch.zeros(n_verts + 1, dtype=torch.int64, device=dev)
    rowptr[1:] = torch.cumsum(torch.bincount(src, minlength=n_verts), 0)
    return edges, dirs, rowptr, dst[order].contiguous()


def hole_faces(verts, codes):
    """the faces that close the 3- and 4-vertex holes (csrc/mesh_post.cu holes), in boundary edge order"""
    dev = verts.device
    V = verts.shape[0]
    edges, dirs, rowptr, cols = boundary(codes, V)
    B = edges.shape[0]
    if B == 0:
        return _i64(0, 3, dev=dev)
    L, st = _lib.lib(), _lib.stream_ptr()
    counts = torch.empty(B, dtype=torch.int32, device=dev)
    check(L.nudf_mp_hole_count(ptr(edges), B, ptr(rowptr), ptr(cols), V, ptr(counts), st), "nudf_mp_hole_count")
    csum = torch.cumsum(counts, 0, dtype=torch.int64)
    n = int(csum[-1])
    out = _i64(n, 3, dev=dev)
    if n:
        offsets = (csum - counts).contiguous()
        check(L.nudf_mp_hole_emit(ptr(verts), ptr(edges), ptr(dirs), B, ptr(rowptr), ptr(cols), V, ptr(offsets), ptr(out), st),
              "nudf_mp_hole_emit")
    return out


def smooth_border_vertices(verts, codes, steps=SMOOTH_STEPS, lam=SMOOTH_LAMBDA):
    """(verts, border vertex count): `steps` Jacobi steps over the border vertices (csrc/mesh_post.cu smoothing)"""
    V = verts.shape[0]
    _, _, rowptr, cols = boundary(codes, V)
    border = torch.nonzero(rowptr[1:] > rowptr[:-1]).reshape(-1).contiguous()
    nb = border.numel()
    a = verts.clone()
    if nb == 0:
        return a, 0
    b = verts.clone()
    L, st = _lib.lib(), _lib.stream_ptr()
    for _ in range(steps):
        check(L.nudf_mp_smooth_step(ptr(a), ptr(b), ptr(border), nb, ptr(rowptr), ptr(cols), lam, st), "nudf_mp_smooth_step")
        a, b = b, a
    return a, nb


@torch.no_grad()
def postprocess(verts64, faces, smooth_borders=True):
    """get_mesh_udf_fast's post-processing (extract_mesh.py:215-265) on the device: (fp64 verts, int64 faces, info).

    verts64 [V,3] and faces [F,3] are the mesh after the vertex filter, on a CUDA device; the vertices are used as fp64.
    The steps follow the reference: Trimesh(...) and process (non-finite, merge), duplicates, degenerate, fill_holes once;
    then at most 10 passes of process / duplicates / degenerate / Trimesh(...) until (V, F) stops changing; then, with
    `smooth_borders`, the border smoothing.  info: `input`, `process` (faces each rule removed), `hole_faces`, `loop`
    (the same per pass), `passes`, `border_vertices`, `output` ((V, F) pairs and counts), `ms` (CUDA-event milliseconds of
    the first process, the hole filling, the loop and the smoothing)."""
    if verts64.device.type != "cuda":
        raise ValueError("postprocess runs on a CUDA device (verts are on %s)" % verts64.device)
    v = verts64.to(torch.float64).reshape(-1, 3).contiguous()
    f = faces.to(device=v.device, dtype=torch.int64).reshape(-1, 3).contiguous()
    info = {"input": (v.shape[0], f.shape[0])}
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    ev[0].record()
    v, f, codes, info["process"] = process(v, f)
    ev[1].record()
    holes = hole_faces(v, codes) if f.shape[0] else _i64(0, 3, dev=v.device)
    info["hole_faces"] = int(holes.shape[0])
    f = torch.cat([f, holes]) if holes.shape[0] else f
    ev[2].record()
    v, f = _compact(v, f)
    passes, counts, loop = 0, (0, 0), []
    while counts != (v.shape[0], f.shape[0]) and passes < MAX_PASSES:
        v, f, _, c = process(v, f)
        loop.append(c)
        counts = (v.shape[0], f.shape[0])
        passes += 1
        v, f = _compact(v, f)
    info["loop"], info["passes"], info["border_vertices"] = loop, passes, 0
    ev[3].record()
    if smooth_borders and f.shape[0]:
        v, info["border_vertices"] = smooth_border_vertices(v, _codes(v, f))
    ev[4].record()
    info["output"] = (v.shape[0], f.shape[0])
    torch.cuda.synchronize(v.device)
    info["ms"] = dict(zip(("process", "holes", "loop", "smooth"), (ev[i].elapsed_time(ev[i + 1]) for i in range(4))))
    return v, f, info


@torch.no_grad()
def export_merge(verts, faces):
    """the runner's last Trimesh(...) before export (exp_runner_blending.py:796): non-finite, then one more merge"""
    v = verts.to(torch.float64).reshape(-1, 3).contiguous()
    f = drop_nonfinite(v, faces.to(device=v.device, dtype=torch.int64).reshape(-1, 3))
    v2, remap = merge_remap(v, f)
    return v2, remap[f]

"""Oriented normals and colours of surface points and mesh vertices, on the device.

A UDF's gradient gives each surface point a normal *line*: the field grows away from the surface on both sides, so the
sign means nothing.  The only orientation that means something for an open surface is towards the cameras that see the
point, and seeing is also what colouring from the images needs.  `surface_views` decides it by sphere tracing the UDF
from the point towards its best-facing cameras (DESIGN.md section 1 states the algorithm):
1. `rank_candidates`: the cameras the point projects in front of and inside, with |n . v| >= cos_min, best facing first.
2. Round r traces the r-th candidate of the points still unresolved: the ray q(t) = p + t v starts one tangent-plane
   distance of `start` voxels off the surface, t0 = start h / |n . v|, and steps t <- t + u(q(t)).  A udf below `hit`
   voxels means the ray met the surface (occluded); leaving the unit sphere or reaching the camera means it did not
   (visible).  The first visible candidate is the point's view.
3. `orient_normals` turns each seen point's normal towards its view; unseen points keep theirs.
`point_colors` gives the colour of the view's image at the point (`mode="image"`) or of the colour network seen from that
camera (`mode="network"`).  The kernels are csrc/udf_paint.cu's; tests/proto/udf_paint.py restates them in NumPy.
"""
import torch

from neuraludf_b200 import _lib
from neuraludf_b200._lib import check, ptr


def _cuda(t, what, dtype, cols=None):
    ok = isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and t.is_contiguous()
    if ok and cols is not None:
        ok = t.dim() == 2 and t.shape[1] == cols
    elif ok:
        ok = t.dim() == 1
    if not ok:
        raise ValueError("%s must be a contiguous %s CUDA tensor [%s]" % (what, dtype, "n" if cols is None else "n,%d" % cols))
    return t


def _cameras(mats, centres):
    _cuda(mats, "mats", torch.float32, 12)
    _cuda(centres, "centres", torch.float32, 3)
    V = mats.shape[0]
    if centres.shape[0] != V:
        raise ValueError("mats and centres must hold one row per camera")
    if V > _lib.PT_MAX_VIEWS:
        raise ValueError("at most %d cameras (got %d)" % (_lib.PT_MAX_VIEWS, V))
    return V


def _same_rows(a, b, what):
    if a.shape[0] != b.shape[0]:
        raise ValueError("%s must hold one row per point" % what)


def camera_matrices(intrinsics, poses, device=None):
    """(mats fp32 [V,12], centres fp32 [V,3]) on the device of fp32 intrinsics [V,4,4] and c2w poses [V,4,4] (render.Scan's
    intrinsics_all / pose_all): the pixel projection (K inv(pose))[:3] formed in fp64 and rounded to fp32 once, and the
    camera centre, the pose's translation."""
    K = torch.as_tensor(intrinsics).detach().to("cpu", torch.float32).double()
    pose = torch.as_tensor(poses).detach().to("cpu", torch.float32)
    dev = device if device is not None else torch.as_tensor(poses).device
    P = (K @ torch.linalg.inv(pose.double()))[:, :3, :].reshape(-1, 12).float()
    return P.contiguous().to(dev), pose[:, :3, 3].contiguous().to(dev)


def scan_cameras(scan):
    """camera_matrices of a render.Scan, with its image size (mats, centres, H, W)"""
    mats, centres = camera_matrices(scan.intrinsics_all, scan.pose_all, scan.device)
    return mats, centres, scan.H, scan.W


def unit_normals(g):
    """g / |g| of g fp32 [M,3] (nudf_pt_normals), 0 where |g| is 0 or not finite"""
    _cuda(g, "g", torch.float32, 3)
    out = torch.empty_like(g)
    check(_lib.lib().nudf_pt_normals(ptr(g), g.shape[0], ptr(out), _lib.stream_ptr()), "nudf_pt_normals")
    return out


@torch.no_grad()
def point_normals(field, points, max_batch=1 << 20, info=None):
    """unit normal lines fp32 [M,3] of points [M,3]: the unit gradient of field.value_gradient (one fused evaluation per
    batch), 0 where the gradient is 0 or not finite (where the udf evaluates to exactly 0, DESIGN.md section 8).
    info: `zero`, the count of such points."""
    _cuda(points, "points", torch.float32, 3)
    out = torch.empty_like(points)
    for head in range(0, points.shape[0], int(max_batch)):
        _, g = field.value_gradient(points[head:head + max_batch])
        out[head:head + max_batch] = unit_normals(g.reshape(-1, 3).float().contiguous())
    if info is not None:
        info["zero"] = int((out == 0).all(1).sum())
    return out


def rank_candidates(points, normals, mats, centres, H, W, cos_min=0.2, candidates=4):
    """int32 [M, candidates] (nudf_pt_rank): the cameras each point projects in front of and inside [0,W-1] x [0,H-1],
    with |n . v| >= cos_min (v the unit direction to the camera), by |n . v| descending, ties to the lower index; -1 pads"""
    _cuda(points, "points", torch.float32, 3)
    _cuda(normals, "normals", torch.float32, 3)
    _same_rows(points, normals, "normals")
    V = _cameras(mats, centres)
    K = int(candidates)
    if not 1 <= K <= _lib.PT_MAX_CAND:
        raise ValueError("candidates must lie in [1, %d]" % _lib.PT_MAX_CAND)
    M = points.shape[0]
    cand = torch.full((M, K), -1, dtype=torch.int32, device=points.device)
    check(_lib.lib().nudf_pt_rank(ptr(points), ptr(normals), M, ptr(mats), ptr(centres), V, int(H), int(W), float(cos_min),
                                  K, ptr(cand), _lib.stream_ptr()), "nudf_pt_rank")
    return cand


def _pairs(n, dev):
    return (torch.empty(n, dtype=torch.int32, device=dev), torch.empty(n, dtype=torch.int32, device=dev),
            torch.empty(n, dtype=torch.float32, device=dev), torch.empty(n, 3, dtype=torch.float32, device=dev))


def start_pairs(points, normals, cand, r, view, centres, t_start):
    """round r's pairs (idx, cam int32 [A], t fp32 [A], q fp32 [A,3]; nudf_pt_start_*): every point with view < 0 and
    k = cand[i, r] >= 0, in order, at t0 = fp32(t_start) / |n . v| and q = p + t0 v"""
    L, st, dev = _lib.lib(), _lib.stream_ptr(), points.device
    M, K = cand.shape
    args = (ptr(points), ptr(normals), ptr(cand), K, int(r), ptr(view), M, ptr(centres), float(t_start))
    if M == 0:
        return _pairs(0, dev)
    counts = _lib.seg_counts(M, dev)
    check(L.nudf_pt_start_count(*args, ptr(counts), st), "nudf_pt_start_count")
    csum = torch.cumsum(counts, 0, dtype=torch.int64)
    out = _pairs(int(csum[-1].item()), dev)
    if out[0].shape[0] == 0:
        return out
    check(L.nudf_pt_start_emit(*args, ptr(csum - counts), *(ptr(a) for a in out), st), "nudf_pt_start_emit")
    return out


def trace_step(points, centres, pairs, u, hit, view):
    """one trace step (nudf_pt_trace_*) of pairs (idx, cam, t, q) with u fp32 [A], the udf at their q: occluded pairs
    (u < fp32(hit), or NaN) are dropped; the others take t <- t + u, and those that leave the unit sphere or reach the
    camera are dropped with view[idx] = cam; returns the pairs still active, in order"""
    return _trace(points, centres, pairs, lambda q: u, hit, view, max(pairs[0].shape[0], 1))


def _trace(points, centres, pairs, values, hit, view, max_batch):
    """one trace step of every pair, the udf taken from values(q) over batches of max_batch (_lib.compact_batches)"""
    L, st, dev = _lib.lib(), _lib.stream_ptr(), points.device
    out = _pairs(pairs[0].shape[0], dev)

    def batch(lo, hi):
        idx, cam, t, q = (a[lo:hi] for a in pairs)
        u = values(q).reshape(-1).float().contiguous()
        if u.shape[0] != hi - lo:
            raise ValueError("u must hold one value per pair")

        def launch(counts, offsets=None):      # holds u until both passes are enqueued
            args = (ptr(points), ptr(centres), ptr(idx), ptr(cam), ptr(t), ptr(u), hi - lo, float(hit))
            if offsets is None:
                check(L.nudf_pt_trace_count(*args, ptr(counts), st), "nudf_pt_trace_count")
            else:
                check(L.nudf_pt_trace_emit(*args, ptr(offsets), ptr(view), *(ptr(a) for a in out), st),
                      "nudf_pt_trace_emit")
        return launch

    n = _lib.compact_batches(pairs[0].shape[0], max_batch, dev, batch)
    return tuple(a[:n] for a in out)


def orient_normals(points, normals, view, centres):
    """normals turned towards their view's camera (nudf_pt_orient): -n where view >= 0 and n . v < 0, else n"""
    out = torch.empty_like(normals)
    check(_lib.lib().nudf_pt_orient(ptr(points), ptr(normals), ptr(view), points.shape[0], ptr(centres), ptr(out),
                                    _lib.stream_ptr()), "nudf_pt_orient")
    return out


@torch.no_grad()
def surface_views(field, points, normals, mats, centres, H, W, voxel, *, candidates=4, cos_min=0.2, start=2.0, hit=1.0,
                  max_steps=64, max_batch=1 << 20, info=None):
    """(view int32 [M], oriented normals fp32 [M,3]): the first of each point's `candidates` best-facing cameras that sees
    it (-1 if none), and its normal line turned towards that camera (kept as given where view is -1).

    field: anything with udf_values(points [A,3]) -> [A] (a UDFNetwork); points, normals: fp32 [M,3] CUDA, in the network's
    frame, the normals unit lines (point_normals); mats, centres: camera_matrices' (at most 64 cameras); H, W: the image
    size; voxel: the length h of start = start h and hit = hit h.  Round r traces the r-th candidate of the unresolved
    points (module docstring); a pair still active after max_steps udf evaluations counts as occluded.  The udf is
    evaluated over batches of max_batch pairs; the results do not depend on it.  The active counts are the only host reads.
    info (a dict, filled when given): no_candidate (points with no candidate camera), rounds (per round: traced pairs and
    visible ones, and the pairs still active after each step), undecided (pairs still active at max_steps), evaluations (udf evaluations in all), seen, and ms,
    CUDA-event milliseconds of the rank, trace and orient stages."""
    _cuda(points, "points", torch.float32, 3)
    _cuda(normals, "normals", torch.float32, 3)
    _same_rows(points, normals, "normals")
    V = _cameras(mats, centres)
    K, max_steps, max_batch = int(candidates), int(max_steps), int(max_batch)
    if max_steps < 1 or max_batch < 1:
        raise ValueError("max_steps and max_batch must be >= 1")
    M, dev = points.shape[0], points.device
    view = torch.full((M,), -1, dtype=torch.int32, device=dev)
    events = []

    def mark():
        events.append(torch.cuda.Event(enable_timing=True))
        events[-1].record()

    mark()
    cand = rank_candidates(points, normals, mats, centres, H, W, cos_min, K)
    mark()
    t_start, thr = float(start) * float(voxel), float(hit) * float(voxel)
    rounds, undecided, evaluations = [], 0, 0
    for r in range(K if V and M else 0):
        pairs = start_pairs(points, normals, cand, r, view, centres, t_start)
        traced, active = pairs[0].shape[0], []
        if traced == 0:
            break
        for _ in range(max_steps):
            if pairs[0].shape[0] == 0:
                break
            evaluations += pairs[0].shape[0]
            pairs = _trace(points, centres, pairs, field.udf_values, thr, view, max_batch)
            active.append(pairs[0].shape[0])
        undecided += pairs[0].shape[0]
        rounds.append((traced, active))
    mark()
    out = orient_normals(points, normals, view, centres)
    mark()
    if info is not None:
        torch.cuda.synchronize(dev)
        ms = [a.elapsed_time(b) for a, b in zip(events, events[1:])]
        seen = [int(((view == cand[:, r]) & (cand[:, r] >= 0)).sum()) for r in range(len(rounds))]
        info.update(no_candidate=int((cand[:, 0] < 0).sum()) if M else 0,
                    rounds=[dict(traced=t, visible=s, active=a) for (t, a), s in zip(rounds, seen)], undecided=undecided,
                    evaluations=evaluations, seen=int((view >= 0).sum()), ms=dict(zip(["rank", "trace", "orient"], ms)))
    return view, out


def gather_colors(points, view, mats, images):
    """fp32 [M,3] in the images' channel order (nudf_pt_gather): the bilinear sample of images[view] (fp32 [V,H,W,3]) at
    the point's pixel, pixel centres on the integers; 0 where view is -1"""
    _cuda(points, "points", torch.float32, 3)
    _cuda(view, "view", torch.int32)
    _same_rows(points, view, "view")
    if not (isinstance(images, torch.Tensor) and images.is_cuda and images.dtype == torch.float32 and images.dim() == 4
            and images.shape[3] == 3 and images.is_contiguous()):
        raise ValueError("images must be a contiguous float32 CUDA tensor [V,H,W,3]")
    _cuda(mats, "mats", torch.float32, 12)
    V, H, W = images.shape[:3]
    if mats.shape[0] != V or V > _lib.PT_MAX_VIEWS:
        raise ValueError("images and mats must hold one entry per camera, at most %d" % _lib.PT_MAX_VIEWS)
    out = torch.empty_like(points)
    check(_lib.lib().nudf_pt_gather(ptr(points), ptr(view), points.shape[0], ptr(mats), ptr(images), V, H, W, ptr(out),
                                    _lib.stream_ptr()), "nudf_pt_gather")
    return out


def view_directions(points, view, normals, centres):
    """the direction the colour network is asked about: normalize(p - c_view), the ray direction of the camera that sees
    p, and -n where view is -1"""
    c = centres[view.clamp(min=0).long()]
    d = torch.nn.functional.normalize(points - c, dim=1)
    return torch.where((view >= 0)[:, None], d, -normals)


@torch.no_grad()
def point_colors(points, view, normals, mode, *, images=None, mats=None, centres=None, udf_network=None,
                 color_network=None, max_batch=1 << 20):
    """RGB in [0,1] fp32 [M,3] of the points (channels reversed from the dataset's BGR).

    mode "image": gather_colors of `images` (render.Scan.images, fp32 [V,H,W,3] BGR / 256) through `mats`; 0 where view
    is -1.  mode "network": the colour network's colour (ResidualRenderingNetwork.forward's second output) at p, with the
    feature of udf_network.value_feature_gradient(p) and the direction view_directions(points, view, normals, centres),
    in batches of max_batch points: the colour the renderer's network gives that sample seen from that camera."""
    _cuda(points, "points", torch.float32, 3)
    _cuda(view, "view", torch.int32)
    _same_rows(points, view, "view")
    if mode == "image":
        if images is None or mats is None:
            raise ValueError('mode "image" needs images and mats')
        bgr = gather_colors(points, view, mats, images)
    elif mode == "network":
        if udf_network is None or color_network is None or centres is None:
            raise ValueError('mode "network" needs udf_network, color_network and centres')
        _cuda(normals, "normals", torch.float32, 3)
        _same_rows(points, normals, "normals")
        bgr = torch.empty_like(points)
        dirs = view_directions(points, view, normals, centres)
        for head in range(0, points.shape[0], int(max_batch)):
            p = points[head:head + max_batch]
            _, feat, _ = udf_network.value_feature_gradient(p)
            bgr[head:head + max_batch] = color_network(p, None, dirs[head:head + max_batch], feat)[1]
    else:
        raise ValueError('mode must be "image" or "network" (got %r)' % (mode,))
    return bgr.flip(1).contiguous()


@torch.no_grad()
def paint_mesh(verts64, faces, field, mats, centres, H, W, voxel, mode, *, images=None, udf_network=None,
               color_network=None, info=None, **trace):
    """(RGB fp32 [V,3] per vertex, view int32 [V]) of a mesh (fp64 verts [V,3], int64 faces [F,3], on the device): the
    normal lines are extract_mesh.vertex_normals (angle-weighted), the views surface_views' at the vertices' fp32
    rounding (`trace`: its keyword arguments), the colours point_colors'.  The mesh itself is not changed."""
    from neuraludf_b200.extract_mesh import vertex_normals
    p = verts64.float().contiguous()
    n = vertex_normals(verts64, faces.to(torch.int64)).contiguous()
    view, n = surface_views(field, p, n, mats, centres, H, W, voxel, info=info, **trace)
    return point_colors(p, view, n, mode, images=images, mats=mats, centres=centres, udf_network=udf_network,
                        color_network=color_network), view


def add_cli_args(ap, normals=True):
    """the painting flags of the cloud and mesh CLIs"""
    ap.add_argument("--scan_dir", default=None,
                    help="DTU-layout scan (image/*.png and the cameras file) whose cameras orient and colour the output")
    ap.add_argument("--scan_cameras", default="cameras.npz", help="the scan's cameras file (default cameras.npz)")
    if normals:
        ap.add_argument("--normals", action="store_true",
                        help="write float nx / ny / nz: the unit gradient, turned towards a camera of --scan_dir that sees "
                             "the point (kept as the gradient gives it where none does)")
    ap.add_argument("--colors", default=None, choices=("network", "image"),
                    help="write uchar red / green / blue: the colour network's colour seen from that camera, or that "
                         "camera's image at the point (black where no camera sees it); needs --scan_dir")


def cli_paint(a, ck, net, points, N, faces=None):
    """(oriented normals or None, RGB colours or None) for the CLIs' flags: points fp32 [M,3] in the network's frame (a
    mesh's fp64 vertices when faces are given), N the lattice resolution (voxel 2 / (N - 1)); prints the seen / unseen
    counts"""
    from neuraludf_b200.render import color_network_from_state, load_scan
    scan = load_scan(a.scan_dir, a.scan_cameras, points.device)
    mats, centres, H, W = scan_cameras(scan)
    col = None
    if a.colors == "network":
        if "color_network_fine" not in ck:
            raise SystemExit("--colors network needs the checkpoint's color_network_fine")
        col = color_network_from_state(ck["color_network_fine"]).to(points.device)
    info = {}
    kw = dict(images=scan.images, udf_network=net, color_network=col)
    voxel = 2.0 / (N - 1)
    if faces is not None:
        colors, view = paint_mesh(points, faces, net, mats, centres, H, W, voxel, a.colors, info=info, **kw)
        normals = None
    else:
        normals = point_normals(net, points)
        view, normals = surface_views(net, points, normals, mats, centres, H, W, voxel, info=info)
        colors = None if a.colors is None else point_colors(points, view, normals, a.colors, mats=mats, centres=centres, **kw)
    print("%d of %d points seen by a camera of %s, %d unseen (%d with no candidate camera)" % (
        info["seen"], view.shape[0], a.scan_dir, view.shape[0] - info["seen"], info["no_candidate"]))
    return normals, colors

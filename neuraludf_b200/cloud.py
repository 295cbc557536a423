"""Dense point clouds on the zero level set of a UDF, on the device, and `python -m neuraludf_b200.cloud`, a
checkpoint-to-PLY CLI.

`udf_point_cloud` is the gradient projection of NDF (Chibane et al., 2020): seeds are the lattice points of the block-sparse
narrow band (grid.udf_band_sparse) with udf < 2 voxels; each is moved K times by p <- p - u g / |g|; the points whose udf
ends below ratio * voxel are kept; jittered copies of kept points go through the same steps until `n_points` are kept
(DESIGN.md section 1 states the algorithm).  The steps, the filter and the jitter are the kernels of csrc/udf_cloud.cu;
tests/proto/udf_cloud.py restates them in NumPy.  The cloud needs no mesh: it keeps open and non-manifold surfaces whole,
and `evaluate.eval_dtu` / `eval_deepfashion` (or `python -m neuraludf_b200.evaluate ... --mode pcd`) score it as it is.
"""
import warnings

import torch

from neuraludf_b200 import _lib, grid
from neuraludf_b200._lib import check, ptr

MAX_ROUNDS = 4          # densify rounds at most


def _launch_step(p, u, g, counts, offsets=None, out=None):
    """the count pass (offsets None) or the emit pass of nudf_uc_step_* on one batch"""
    L, st = _lib.lib(), _lib.stream_ptr()
    if offsets is None:
        check(L.nudf_uc_step_count(ptr(p), ptr(u), ptr(g), p.shape[0], ptr(counts), st), "nudf_uc_step_count")
    else:
        check(L.nudf_uc_step_emit(ptr(p), ptr(u), ptr(g), p.shape[0], ptr(offsets), ptr(out), st), "nudf_uc_step_emit")


def _launch_filter(p, u, thr, counts, offsets=None, out=None):
    """the count pass (offsets None) or the emit pass of nudf_uc_filter_* on one batch"""
    L, st = _lib.lib(), _lib.stream_ptr()
    if offsets is None:
        check(L.nudf_uc_filter_count(ptr(p), ptr(u), p.shape[0], thr, ptr(counts), st), "nudf_uc_filter_count")
    else:
        check(L.nudf_uc_filter_emit(ptr(p), ptr(u), p.shape[0], thr, ptr(offsets), ptr(out), st), "nudf_uc_filter_emit")


def _compact(pts, max_batch, evaluate, launch):
    """the survivors of pts [n,3] in order, in batches of max_batch (_lib.compact_batches): evaluate(batch) gives the extra
    arguments of launch(batch, *args, counts, offsets, out)"""
    out = torch.empty_like(pts)

    def batch(lo, hi):
        p = pts[lo:hi]
        args = evaluate(p)
        return lambda counts, offsets=None: launch(p, *args, counts, offsets, out)

    return out[:_lib.compact_batches(pts.shape[0], max_batch, pts.device, batch)]


def _points(t, what):
    if not (t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.shape[1] == 3 and t.is_contiguous()):
        raise ValueError("%s must be a contiguous float32 CUDA tensor [P,3]" % what)
    return t


def _column(t, P, what):
    t = t.reshape(-1).float().contiguous()
    if t.numel() != P:
        raise ValueError("%s must hold one value per point (%d, got %d)" % (what, P, t.numel()))
    return t


def project_step(pts, u, g):
    """One projection step (nudf_uc_step_*) on pts [P,3] fp32 with the udf u [P] and its gradient g [P,3] there: the points
    q = p - (u / |g|) g, in order, of the rows whose u and g are finite, |g| != 0 and q in [-1,1]^3."""
    _points(pts, "pts")
    u = _column(u, pts.shape[0], "u")
    g = _points(g.reshape(-1, 3).float().contiguous(), "g")
    if g.shape[0] != pts.shape[0]:
        raise ValueError("g must hold one row per point")
    return _compact(pts, max(pts.shape[0], 1), lambda p: (u, g), _launch_step)


def filter_points(pts, u, thr):
    """the points of pts [P,3] fp32 with u < thr (thr rounded to fp32; nudf_uc_filter_*), in order"""
    _points(pts, "pts")
    u = _column(u, pts.shape[0], "u")
    return _compact(pts, max(pts.shape[0], 1), lambda p: (u, float(thr)), _launch_filter)


def resample(pool, m, seed, round_, voxel):
    """m jittered copies of points of pool [M,3] (nudf_uc_resample): copy i is pool[hash(seed, round_, i, 0) mod M] offset by
    ((b_a 2^-24 - 1/2) fp32(voxel))_a, b_a the top 24 bits of hash(seed, round_, i, 1 + a); the seed is taken mod 2^32"""
    _points(pool, "pool")
    out = torch.empty(int(m), 3, dtype=torch.float32, device=pool.device)
    check(_lib.lib().nudf_uc_resample(ptr(pool), pool.shape[0], int(m), int(seed) & 0xFFFFFFFF, int(round_), float(voxel),
                                      ptr(out), _lib.stream_ptr()), "nudf_uc_resample")
    return out


def _value_gradient(field, p):
    u, g = field.value_gradient(p)
    return u.reshape(-1).float().contiguous(), g.reshape(-1, 3).float().contiguous()


def _project(field, pts, steps, max_batch):
    """`steps` projection steps on pts: (survivors, survivor count after each step)"""
    counts = []
    for _ in range(steps):
        pts = _compact(pts, max_batch, lambda p: _value_gradient(field, p), _launch_step)
        counts.append(int(pts.shape[0]))
    return pts, counts


def _filter(field, pts, thr, max_batch):
    return _compact(pts, max_batch, lambda p: (field.udf_values(p).reshape(-1).float().contiguous(), thr), _launch_filter)


@torch.no_grad()
def udf_point_cloud(field, N, n_points, steps=5, dist_threshold_ratio=1.0, lipschitz=2.0, seed=0, max_batch=1 << 20,
                    info=None):
    """Points on the zero level set of a UDF: fp32 [M,3] on the device, M <= n_points.

    `field`: any object with udf_values(pts [P,3]) -> [P] and value_gradient(pts) -> (udf [P], grad [P,3]), both without
    autograd (a UDFNetwork, or closures).  N: lattice points per axis on [-1,1]^3, voxel h = 2 / (N - 1).
    1. Seeds: the points of grid.udf_band_sparse(field, N, lipschitz) with udf < 2 h (grid.near_surface_indices_sparse), in
       ascending flat-index order at their lattice coordinates: every lattice point with udf < 2 h when the field is
       `lipschitz`-Lipschitz, with no N^3 array.
    2. `steps` projection steps over batches of max_batch (project_step).
    3. The points with udf_values < fp32(dist_threshold_ratio h) are kept, in order.
    4. While fewer than n_points are kept, at most MAX_ROUNDS rounds: round r draws n_points - kept jittered copies of the
       points kept in 3 (resample(kept, ..., seed, r, h)), which go through 2 and 3 and are appended.
    5. The first n_points kept points.  When more than n_points survive 3, the cut follows the lattice order (x slowest)
       and a RuntimeWarning says so: a cloud meant to cover the whole surface wants n_points at least info["filtered"].
    A learned UDF need not reach 0: with a floor c, the points settle within about c of the surface, on either side, and
    the filter keeps them when c < dist_threshold_ratio h.  A field with no zero crossing in the box gives [0,3].

    info (a dict, filled when given): seeds, steps (survivors after each step), filtered (kept after 3), rounds (per densify
    round: drawn, steps, kept), rounds_used, points, truncated (kept points beyond n_points), band (udf_band_sparse's
    info) and ms, CUDA-event milliseconds per stage: band, seeds, projection, filter, densify."""
    N, n_points, steps, max_batch = int(N), int(n_points), int(steps), int(max_batch)
    if N < 2:
        raise ValueError("N must be at least 2 (got %d)" % N)
    if n_points < 0 or steps < 0 or max_batch < 1:
        raise ValueError("n_points and steps must be >= 0 and max_batch >= 1")
    voxel = 2.0 / (N - 1)
    thr = float(dist_threshold_ratio) * voxel
    events = []

    def mark():
        events.append(torch.cuda.Event(enable_timing=True))
        events[-1].record()

    mark()
    band, band_info = grid.udf_band_sparse(field, N, lipschitz, max_batch=max_batch)
    mark()
    idx = grid.near_surface_indices_sparse(band)
    del band
    pts = grid._index_points(idx, N)
    n_seeds = idx.numel()
    del idx
    mark()
    pts, step_counts = _project(field, pts, steps, max_batch)
    mark()
    pool = _filter(field, pts, thr, max_batch)
    del pts
    mark()
    kept, n_kept, rounds = [pool], pool.shape[0], []
    while n_kept < n_points and pool.shape[0] and len(rounds) < MAX_ROUNDS:
        m = n_points - n_kept
        new, s = _project(field, resample(pool, m, seed, len(rounds), voxel), steps, max_batch)
        new = _filter(field, new, thr, max_batch)
        rounds.append(dict(drawn=m, steps=s, kept=int(new.shape[0])))
        kept.append(new)
        n_kept += new.shape[0]
    out = torch.cat(kept)[:n_points] if len(kept) > 1 else pool[:n_points].contiguous()
    mark()
    if n_kept > n_points:
        warnings.warn("udf_point_cloud: %d points survive the filter, more than n_points=%d: the cloud is the first n_points "
                      "in lattice order (x slowest) and misses the rest of the surface; lower N or raise n_points"
                      % (n_kept, n_points), RuntimeWarning, stacklevel=3)
    torch.cuda.synchronize()
    if info is not None:
        ms = [a.elapsed_time(b) for a, b in zip(events, events[1:])]
        info.update(seeds=n_seeds, steps=step_counts, filtered=int(pool.shape[0]), rounds=rounds, rounds_used=len(rounds),
                    points=int(out.shape[0]), truncated=max(int(n_kept) - n_points, 0), band=band_info,
                    ms=dict(zip(["band", "seeds", "projection", "filter", "densify"], ms)))
    return out


def main(argv=None):
    """python -m neuraludf_b200.cloud: a runner checkpoint's UDF network -> PLY point cloud (see INTEGRATION.md)"""
    import argparse
    import numpy as np
    from neuraludf_b200.evaluate import write_ply_points
    from neuraludf_b200.mesh import udf_network_from_state
    from neuraludf_b200 import paint
    ap = argparse.ArgumentParser(prog="python -m neuraludf_b200.cloud",
                                 description="A dense point cloud on the zero level set of the UDF network of a runner "
                                             "checkpoint: narrow-band seeds projected along the gradient (udf_point_cloud).")
    ap.add_argument("--ckpt", required=True, help="checkpoint written by the runner (its udf_network_fine state dict is used)")
    ap.add_argument("--resolution", type=int, required=True, help="seed lattice points per axis (up to 2048)")
    ap.add_argument("--points", type=int, required=True, help="points wanted in the cloud")
    ap.add_argument("--steps", type=int, default=5, help="projection steps per point (default 5)")
    ap.add_argument("--dist_threshold_ratio", type=float, default=1.0,
                    help="keep the points whose final udf is below this many voxels (default 1)")
    ap.add_argument("--seed", type=int, default=0, help="seed of the densify rounds' jitter")
    ap.add_argument("--scale", type=float, default=1.0, help="the conf's udf_network.scale")
    ap.add_argument("--cameras", default=None, help="cameras_sphere.npz: map the cloud to world space with its scale_mat_0")
    paint.add_cli_args(ap)
    ap.add_argument("--out", required=True, help="output PLY")
    a = ap.parse_args(argv)
    if (a.normals or a.colors) and a.scan_dir is None:
        ap.error("--normals and --colors need --scan_dir")
    if not torch.cuda.is_available():
        raise SystemExit("point clouds are computed on a CUDA device")
    ck = torch.load(a.ckpt, map_location="cpu", weights_only=True)
    net = udf_network_from_state(ck["udf_network_fine"] if "udf_network_fine" in ck else ck, a.scale).cuda()
    info = {}
    pts = udf_point_cloud(net, a.resolution, a.points, a.steps, a.dist_threshold_ratio, seed=a.seed, info=info)
    normals, colors = paint.cli_paint(a, ck, net, pts, a.resolution) if a.scan_dir is not None else (None, None)
    v = pts.double().cpu().numpy()
    if a.cameras is not None:                     # as the mesh CLI: the dataset's fp32 scale_mat_0
        sm = np.load(a.cameras)["scale_mat_0"].astype(np.float32)
        v = v * sm[0, 0] + sm[:3, 3][None]        # a uniform scale and a shift: the normals are unchanged
    write_ply_points(a.out, v, colors=colors, normals=normals if a.normals else None)
    print("%s: %d points (%d seeds, %d after filtering, %d densify rounds)" % (a.out, v.shape[0], info["seeds"],
                                                                              info["filtered"], info["rounds_used"]))
    return v


if __name__ == "__main__":
    main()

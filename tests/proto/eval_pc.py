"""NumPy / sklearn restatement of the point-cloud evaluation protocols (neuraludf_b200/evaluate.py, csrc/eval_pc.cu): the
exact oracle of the CUDA stages at sizes beyond the golden fixtures.  Every stage is the reference scripts' own expression
(evaluation/eval_dtu_python.py, eval_deepfashion_python.py); the greedy downsampling is their sequential loop."""
import numpy as np
import sklearn.neighbors as skln


def sample_mesh(verts, faces, density):
    """vertices, then the samples of every triangle with area2 > 0 in triangle order (eval_dtu_python.py:21-30, 56-75)"""
    verts = np.asarray(verts, np.float64)
    tri_vert = verts[np.asarray(faces, np.int64)]
    v1 = tri_vert[:, 1] - tri_vert[:, 0]
    v2 = tri_vert[:, 2] - tri_vert[:, 0]
    l1 = np.linalg.norm(v1, axis=-1, keepdims=True)
    l2 = np.linalg.norm(v2, axis=-1, keepdims=True)
    area2 = np.linalg.norm(np.cross(v1, v2), axis=-1, keepdims=True)
    nz = (area2 > 0)[:, 0]
    l1, l2, area2, v1, v2, tri_vert = [a[nz] for a in [l1, l2, area2, v1, v2, tri_vert]]
    thr = density * np.sqrt(l1 * l2 / area2)
    n1 = np.floor(l1 / thr)
    n2 = np.floor(l2 / thr)
    pts = [verts]
    for i in range(len(n1)):
        c = np.mgrid[:n1[i, 0] + 1, :n2[i, 0] + 1]
        c += 0.5
        c[0] /= max(n1[i, 0], 1e-7)
        c[1] /= max(n2[i, 0], 1e-7)
        c = np.transpose(c, (1, 2, 0))
        k = c[c.sum(axis=-1) < 1]
        pts.append(v1[i:i + 1] * k[:, :1] + v2[i:i + 1] * k[:, 1:] + tri_vert[i:i + 1, 0])
    return np.concatenate(pts, axis=0)


def seeded_permutation(n, seed):
    return np.random.default_rng(seed).permutation(n)


def downsample(points, radius, perm):
    """(kept points, kept positions in the shuffled order): the scripts' loop over sklearn's radius neighbourhoods"""
    sp = np.asarray(points, np.float64)[np.asarray(perm)]
    nn = skln.NearestNeighbors(n_neighbors=1, radius=radius, algorithm="kd_tree", n_jobs=-1).fit(sp)
    idxs = nn.radius_neighbors(sp, radius=radius, return_distance=False)
    mask = np.ones(len(sp), dtype=np.bool_)
    for curr, ix in enumerate(idxs):
        if mask[curr]:
            mask[ix] = 0
            mask[curr] = 1
    kept = np.nonzero(mask)[0]
    return sp[kept], kept


def nearest(queries, targets):
    """sklearn KD-tree nearest distance (unbounded)"""
    queries = np.asarray(queries, np.float64).reshape(-1, 3)
    if len(queries) == 0:
        return np.zeros(0)
    nn = skln.NearestNeighbors(n_neighbors=1, algorithm="kd_tree", n_jobs=-1).fit(np.asarray(targets, np.float64))
    return nn.kneighbors(queries, n_neighbors=1, return_distance=True)[0][:, 0]


def dtu_masks(down, bb, res, obs_mask, patch):
    """(inbound [K] bool, grid_inbound [n_in] bool, in_obs [n_grid_in] bool) of eval_dtu_python.py:102-114"""
    BB = np.asarray(bb).astype(np.float32)
    inbound = ((down >= BB[:1] - patch) & (down < BB[1:] + patch * 2)).sum(axis=-1) == 3
    data_in = down[inbound]
    data_grid = np.around((data_in - BB[:1]) / res).astype(np.int32)
    grid_inbound = ((data_grid >= 0) & (data_grid < np.expand_dims(obs_mask.shape, 0))).sum(axis=-1) == 3
    g = data_grid[grid_inbound]
    in_obs = obs_mask[g[:, 0], g[:, 1], g[:, 2]].astype(np.bool_)
    return inbound, grid_inbound, in_obs


def plane_above(stl, plane):
    stl_hom = np.concatenate([stl, np.ones_like(stl[:, :1])], -1)
    return (np.asarray(plane).reshape((1, 4)) * stl_hom).sum(-1) > 0


def metrics(d2s, s2d, max_dist, thresholds):
    mean_d2s = d2s[d2s < max_dist].mean()
    mean_s2d = s2d[s2d < max_dist].mean()
    out = {"mean_d2gt": mean_d2s, "mean_gt2d": mean_s2d, "over_all": (mean_d2s + mean_s2d) / 2}
    for k, t in enumerate(thresholds, 1):
        p = len(d2s[d2s < t]) / len(d2s)
        r = len(s2d[s2d < t]) / len(s2d)
        out["precision_%d" % k], out["recall_%d" % k] = p, r
        out["fscore_%d" % k] = 2 * p * r / (p + r + 1e-6)
    return out


def error_colors(d, vis, max_dist):
    R, W, G = np.array([[1., 0, 0]]), np.array([[1., 1, 1]]), np.array([[0., 1, 0]])
    alpha = d[:, None].clip(max=vis) / vis
    c = R * alpha + W * (1 - alpha)
    c[d >= max_dist] = G
    return c


def eval_dtu(data, faces, gt, obs_mask, bb, res, plane, perm, density=0.2, patch=60.0, max_dist=20.0, vis=10.0,
             thresholds=(1.0, 2.0)):
    pcd = sample_mesh(data, faces, density) if faces is not None else np.asarray(data, np.float64)
    down, kept = downsample(pcd, density, perm)
    inbound, grid_inbound, in_obs = dtu_masks(down, bb, res, obs_mask, patch)
    data_in = down[inbound]
    data_in_obs = data_in[grid_inbound][in_obs]
    d2s = nearest(data_in_obs, gt)
    above = plane_above(gt, plane)
    s2d = nearest(gt[above], data_in)
    out = metrics(d2s, s2d, max_dist, thresholds)
    dc = np.tile(np.array([[0., 0, 1]]), (len(down), 1))
    dc[np.where(inbound)[0][grid_inbound][in_obs]] = error_colors(d2s, vis, max_dist)
    gc = np.tile(np.array([[0., 0, 1]]), (len(gt), 1))
    gc[np.where(above)[0]] = error_colors(s2d, vis, max_dist)
    out.update(data_pcd=pcd, kept_index=kept, data_down=down, inbound=inbound, grid_inbound=grid_inbound, in_obs=in_obs,
               above=above, dist_d2s=d2s, dist_s2d=s2d, data_color=dc, gt_color=gc)
    return out


def eval_deepfashion(data, faces, gt, perm, density=0.002, max_dist=0.1, vis=0.01, thresholds=(0.001, 0.002)):
    pcd = sample_mesh(data, faces, density) if faces is not None else np.asarray(data, np.float64)
    down, kept = downsample(pcd, density, perm)
    d2s = nearest(down, gt)
    s2d = nearest(gt, down)
    out = metrics(d2s, s2d, max_dist, thresholds)
    out.update(data_pcd=pcd, kept_index=kept, data_down=down, dist_d2s=d2s, dist_s2d=s2d,
               data_color=error_colors(d2s, vis, max_dist), gt_color=error_colors(s2d, vis, max_dist))
    return out

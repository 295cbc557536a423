"""CPU checks of the view renderer's host side (neuraludf_b200/render.py): the DTU-layout loader's cameras and source
views, the interpolated pose of rays_between, and the image files the CLI writes."""
import os

import numpy as np
import pytest

from neuraludf_b200 import render as R
from tests.runner_env import _look_at, write_synthetic_dtu


@pytest.fixture(scope="module")
def scan_dir(tmp_path_factory):
    return write_synthetic_dtu(str(tmp_path_factory.mktemp("scan")), n_images=10, width=64, height=48)


def test_load_scan_cameras(scan_dir):
    """intrinsics / pose of world_mat @ scale_mat decomposed as load_K_Rt_from_P: K of the writer, c2w = inv([R | t])"""
    s = R.load_scan(scan_dir, device="cpu")
    assert s.n_images == 10 and (s.H, s.W) == (48, 64)
    cams = np.load(os.path.join(scan_dir, "cameras.npz"))
    focal = 1.1 * 64
    K = np.array([[focal, 0, 31.5], [0, focal, 23.5], [0, 0, 1.0]])
    for i in range(s.n_images):
        P = cams["world_mat_%d" % i].astype(np.float32) @ cams["scale_mat_%d" % i].astype(np.float32)
        intr, pose = R.decompose_projection(P)
        assert intr.dtype == np.float64 and pose.dtype == np.float32
        np.testing.assert_allclose(intr[:3, :3], K, rtol=1e-5, atol=1e-4)
        Rw = np.linalg.inv(K) @ P[:3, :3]                  # the writer's world -> camera rotation
        np.testing.assert_allclose(pose[:3, :3], Rw.T, atol=2e-5)
        np.testing.assert_allclose(pose[:3, :3] @ pose[:3, :3].T, np.eye(3), atol=2e-5)
        np.testing.assert_allclose(s.pose_all[i].numpy(), pose)
        np.testing.assert_allclose(s.intrinsics_all[i].numpy(), intr.astype(np.float32))
        # the camera centre lies on the writer's ring of radius 2.5
        assert abs(np.linalg.norm(pose[:3, 3]) - 2.5) < 1e-4
    img = s.images[3].numpy()
    import cv2
    np.testing.assert_array_equal(img, (cv2.imread(s.images_lis[3]) / 256.0).astype(np.float32))


def test_source_views_nearest_centres_stable_ties():
    c = np.array([[0, 0, 0], [1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, 0, 3.0]])
    src = R.source_views(c, num=3)
    np.testing.assert_array_equal(src[0], [1, 2, 3])               # three equidistant neighbours in index order
    d = np.linalg.norm(c[:, None] - c[None], axis=-1)
    for i in range(len(c)):
        assert i not in src[i]
        assert np.all(np.diff(d[i, src[i]]) >= 0)


def test_pose_between_end_points():
    R0, t0 = _look_at(np.array([2.5, 0.0, 0.5]))
    R1, t1 = _look_at(np.array([0.0, 2.5, 0.3]))
    poses = []
    for Rw, t in ((R0, t0), (R1, t1)):
        w2c = np.eye(4)
        w2c[:3, :3], w2c[:3, 3] = Rw, t
        poses.append(np.linalg.inv(w2c).astype(np.float32))
    np.testing.assert_allclose(R.pose_between(poses[0], poses[1], 0.0), poses[0], atol=1e-5)
    np.testing.assert_allclose(R.pose_between(poses[0], poses[1], 1.0), poses[1], atol=1e-5)
    mid = R.pose_between(poses[0], poses[1], 0.5)
    np.testing.assert_allclose(mid[:3, :3] @ mid[:3, :3].T, np.eye(3), atol=1e-5)


def test_image_files_match_the_runner_expressions(tmp_path):
    """the bytes cv2 writes from the CLI's arrays equal those of validate()'s own expressions (:696-720)"""
    import cv2
    rng = np.random.RandomState(0)
    H, W = 12, 16
    color = rng.uniform(-0.1, 1.1, (H * W, 3)).astype(np.float32)
    pixel = rng.uniform(-0.1, 1.1, (H * W, 3)).astype(np.float32)
    normal = rng.uniform(-1.2, 1.2, (H * W, 3)).astype(np.float32)
    gt = rng.randint(0, 256, (H, W, 3)).astype(np.uint8)
    runner_fine = (np.concatenate([color], axis=0).reshape([H, W, 3]) * 256).clip(0, 255)
    runner_pixel = (np.concatenate([pixel], axis=0).reshape([H, W, 3]) * 256).clip(0, 255)
    runner_normal = (normal.reshape([H, W, 3]) * 128 + 128).clip(0, 255)[:, :, ::-1]
    pairs = [(np.concatenate([runner_fine, runner_pixel, gt]),
              np.concatenate([R.color_image(color.reshape(H, W, 3)), R.color_image(pixel.reshape(H, W, 3)), gt])),
             (runner_normal, R.normal_image(normal.reshape(H, W, 3)))]
    for k, (a, b) in enumerate(pairs):
        pa, pb = str(tmp_path / ("a%d.png" % k)), str(tmp_path / ("b%d.png" % k))
        assert cv2.imwrite(pa, a) and cv2.imwrite(pb, b)
        assert open(pa, "rb").read() == open(pb, "rb").read()


# ---- against the reference's own Dataset code (tests/golden/render_view.*.npz, oracle/make_golden_render.py) ----
@pytest.fixture(scope="module")
def fx():
    from tests.golden_util import Fixtures
    return Fixtures("render_view")


@pytest.fixture(scope="module")
def golden_scan(tmp_path_factory):
    from oracle.make_golden_render import HEIGHT, N_IMAGES, WIDTH
    return write_synthetic_dtu(str(tmp_path_factory.mktemp("gscan")), n_images=N_IMAGES, width=WIDTH, height=HEIGHT)


def test_load_scan_matches_reference_dataset(fx, golden_scan):
    """intrinsics and poses of load_K_Rt_from_P, the source-view pairs of prepare_ref_src_pairs"""
    s = R.load_scan(golden_scan, device="cpu")
    np.testing.assert_array_equal(s.intrinsics_all.numpy(), fx["intrinsics"])
    np.testing.assert_array_equal(s.pose_all.numpy(), fx["pose"])
    np.testing.assert_array_equal(s.src, fx["src_pairs"])


def test_pose_between_matches_gen_rays_between(fx, golden_scan):
    """the rays of pose_between's pose on gen_rays_between's pixel grid (intrinsics of image 0) at two interior ratios"""
    import torch
    from oracle.make_golden_render import LEVEL
    s = R.load_scan(golden_scan, device="cpu")
    for k in range(2):
        r = float(fx["between%d_ratio" % k])
        pose = torch.from_numpy(R.pose_between(s.pose_all[0].numpy(), s.pose_all[1].numpy(), r)).float()
        tx = torch.linspace(0, s.W - 1, s.W // LEVEL)
        ty = torch.linspace(0, s.H - 1, s.H // LEVEL)
        py, px = torch.meshgrid(ty, tx, indexing="ij")
        p = torch.stack([px, py, torch.ones_like(py)], dim=-1)
        p = (s.intrinsics_all_inv[0, :3, :3] @ p[..., None])[..., 0]
        v = p / torch.linalg.norm(p, ord=2, dim=-1, keepdim=True)
        v = (pose[:3, :3] @ v[..., None])[..., 0]
        np.testing.assert_allclose(v.numpy(), fx["between%d_rays_d" % k], atol=2e-6)
        np.testing.assert_allclose(np.broadcast_to(pose[:3, 3].numpy(), v.shape), fx["between%d_rays_o" % k], atol=2e-6)

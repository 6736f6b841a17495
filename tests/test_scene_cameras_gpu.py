"""Camera plumbing end to end: ground-truth images of a C1-like scene are rendered by the repository's own 3DGUT renderer from cameras the
test builds itself and written as lossless PNGs -- a NeRF-synthetic folder with RGBA images, and a COLMAP folder (at downsample factor 2)
with an OPENCV distorted pinhole and an OPENCV_FISHEYE camera.  Each view tuple the dataset yields is then rendered through 3DGUT and
3DGRT and compared with the same renderer's image from the test's own camera.

Where the dataset's rays come from the same `scenes` functions the test uses (the undistorted pinhole, the fisheye), the images must be
the same bytes: that checks the sensor the dataset hands to the 3DGUT projection (focal length, principal point, distortion slots,
max_angle, shutter) and the pose, not only the rays.  For the distorted pinhole the test computes its rays independently (a fixed-point
undistortion, not the dataset's Newton iteration), so the bar is a PSNR."""
from __future__ import annotations

import json
import math
import os

import numpy as np
import pytest
import torch

import scenes
import scene_data
from scene_fixtures import rotmat_to_qvec, run_conf, write_colmap, write_nerf, write_png

pytestmark = pytest.mark.gpu

ANGLE_X = 0.6911112070083618
OPENCV_FULL = [120.0, 118.0, 64.4, 47.6, -0.08, 0.015, 0.0012, -0.0009]   # fx fy cx cy k1 k2 p1 p2 at 128x96
FISHEYE_FULL = [60.0, 61.0, 63.2, 48.8, 0.04, -0.012, 0.003, -0.0006]    # fx fy cx cy k1 k2 k3 k4 at 128x96
# PSNR of the distorted camera's render from the dataset's rays against the test's independently undistorted rays, through each renderer.
# Measured on an H100 80GB HBM3 (700 W): infinite on every frame through both renderers (the uint8 images are the same bytes; the two ray
# computations agree far below what moves a pixel value).  The bar leaves room for a last-bit difference in a ray.
MIN_DISTORTED_PSNR = 50.0


def _u8(x):
    return (x.clamp(0, 1) * 255).round().byte().cpu().numpy()


def _psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return float("inf") if mse == 0 else 10 * math.log10(255.0 ** 2 / mse)


@pytest.fixture(scope="module")
def truth():
    """(3DGUT step, 3DGRT step) holding the ground-truth Gaussians."""
    from train_step import GaussianTrainStep, raw_params
    from train_step_grt import GaussianTrainStepGRT

    sc = scenes.scene_c1(n=1000)
    params = raw_params(torch.from_numpy(sc.particles).cuda(), torch.from_numpy(sc.sph).cuda())
    lrs = {k: 0.0 for k in params}
    grt_conf = {"render": run_conf("", "", method="3dgrt")["render"]}
    return sc, GaussianTrainStep(params, lrs, sph_degree=3), GaussianTrainStepGRT({k: v.clone() for k, v in params.items()}, lrs, conf=grt_conf,
                                                                                sph_degree=3)


def _gut(step, ro, rd, sensor, pose):
    return step.render(ro, rd, sensor, pose)[0][..., :3]


def _grt(step, ro, rd, T):
    return step.render(ro, rd, T)[0][0]


def _tracer():
    import threedgut_tracer.tracer as tr

    return tr


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ---- NeRF-synthetic, RGBA -------------------------------------------------------------------------------------------------------------

def test_nerf_views_render_the_stored_images(truth, tmp_path):
    sc, gut, grt = truth
    tr = _tracer()
    w = h = 64
    fx = float(0.5 * w / np.tan(0.5 * ANGLE_X))  # dataset_nerf.py:128
    ro, rd = (_cuda(a) for a in scenes.pinhole_rays(h, w, fx, fx, w / 2, h / 2))
    sensor = tr.fromOpenCVPinholeCameraModelParameters([w, h], tr.ShutterType.GLOBAL, [w / 2, h / 2], [fx, fx], np.zeros(6), np.zeros(2),
                                                        np.zeros(4))
    rows, want = [], []
    for i in range(4):
        c2w = scenes.orbit_c2w(i, 4, sc.camera_radius)
        c2w32 = c2w.astype(np.float32)
        pose = tr.Tracer._pose_from_c2w(c2w32)
        rgba = gut.render(ro, rd, sensor, pose)[0]
        img = np.concatenate([_u8(rgba[..., :3]), _u8(rgba[..., 3:])], -1)
        nerf = c2w.copy()
        nerf[:, 1:3] *= -1  # the file stores right-up-back
        rows.append((nerf, img, None))
        want.append((img, _u8(_grt(grt, ro, rd, torch.from_numpy(c2w32[None].copy())))))
    write_nerf(str(tmp_path), {"train": rows, "val": rows[:1], "test": rows[:1]}, camera_angle_x=ANGLE_X)
    conf = {"path": str(tmp_path), "dataset": {"type": "nerf"}, "model": {"background": {"color": "black"}}}
    data = scene_data.SceneData(conf)
    for i, (img, grt_img) in enumerate(want):
        a = img[..., 3:].astype(np.float32) / 255.0  # the RGBA composite onto black the dataset stores (dataset_nerf.py:416-445)
        np.testing.assert_array_equal(data.train.images[i].cpu().numpy(), ((img[..., :3].astype(np.float32) / 255.0 * a) * 255.0).astype(np.uint8))
        np.testing.assert_array_equal(_u8(_gut(gut, *data.train.view(i, "3dgut"))), img[..., :3])
        np.testing.assert_array_equal(_u8(_grt(grt, *data.train.view(i, "3dgrt"))), grt_img)


# ---- COLMAP: OPENCV (distorted) and OPENCV_FISHEYE at factor 2 -----------------------------------------------------------------------

def _qvec_to_R(q):
    """COLMAP's qvec (w, x, y, z) -> rotation, written out as the reference writes it (datasets/utils.py:413-432)."""
    w, x, y, z = q
    return np.array([[1 - 2 * y ** 2 - 2 * z ** 2, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
                     [2 * x * y + 2 * w * z, 1 - 2 * x ** 2 - 2 * z ** 2, 2 * y * z - 2 * w * x],
                     [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x ** 2 - 2 * y ** 2]])


def _undistort_fixed_point(h, w, fx, fy, cx, cy, k1, k2, p1, p2, iterations=200):
    """Rays of an OpenCV pinhole (k1, k2, p1, p2) by the classic fixed-point undistortion (as cv::undistortPoints iterates), float64."""
    v, u = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    xd, yd = (u + 0.5 - cx) / fx, (v + 0.5 - cy) / fy
    x, y = xd.copy(), yd.copy()
    for _ in range(iterations):
        r2 = x * x + y * y
        icd = 1 + k1 * r2 + k2 * r2 * r2
        x = (xd - (2 * p1 * x * y + p2 * (r2 + 2 * x * x))) / icd
        y = (yd - (p1 * (r2 + 2 * y * y) + 2 * p2 * x * y)) / icd
    d = np.stack([x, y, np.ones_like(x)], -1)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    return np.zeros((1, h, w, 3), np.float32), d[None].astype(np.float32)


def test_colmap_distorted_and_fisheye_views(truth, tmp_path):
    sc, gut, grt = truth
    tr = _tracer()
    factor, w, h = 2, 64, 48
    # the test's own cameras at factor 2, from COLMAP's parameter layout (the reference divides float32 parameters by the factor)
    q = np.float32(OPENCV_FULL)
    fx, fy, cx, cy = (float(v) for v in q[:4] / factor)
    k1, k2, p1, p2 = (float(v) for v in q[4:])
    opencv = dict(sensor=tr.fromOpenCVPinholeCameraModelParameters([w, h], tr.ShutterType.GLOBAL, [cx, cy], [fx, fy], [k1, k2, 0, 0, 0, 0],
                                                                   [p1, p2], np.zeros(4)),
                  rays=_undistort_fixed_point(h, w, fx, fy, cx, cy, k1, k2, p1, p2))
    fe = np.asarray(FISHEYE_FULL, np.float64)
    ffx, ffy, fcx, fcy = (float(v) for v in (fe[:4] / factor).astype(np.float32))
    radius = float(np.linalg.norm(np.array([fcx if fcx > w / 2 else w - fcx, fcy if fcy > h / 2 else h - fcy])))  # compute_max_radius
    max_angle = max(2 * radius / np.float32(ffx), 2 * radius / np.float32(ffy)) / 2  # create_fisheye_camera
    fisheye = dict(sensor=tr.fromOpenCVFisheyeCameraModelParameters([w, h], tr.ShutterType.GLOBAL, [fcx, fcy], [ffx, ffy], fe[4:8], max_angle),
                   rays=scenes.fisheye_rays(h, w, ffx, ffy, fcx, fcy, np.float32(fe[4:8])))
    cams = {1: ("OPENCV", 128, 96, OPENCV_FULL), 2: ("OPENCV_FISHEYE", 128, 96, FISHEYE_FULL)}
    images, want = [], []
    for i in range(6):
        cid = 1 + i % 2
        cam = opencv if cid == 1 else fisheye
        w2c = np.linalg.inv(scenes.orbit_c2w(i, 6, sc.camera_radius))
        qvec, tvec = rotmat_to_qvec(w2c[:3, :3]), w2c[:3, 3]
        W2C = np.eye(4, dtype=np.float32)
        W2C[:3, :3], W2C[:3, 3] = _qvec_to_R(qvec), tvec
        c2w32 = np.linalg.inv(W2C)
        ro, rd = (_cuda(a) for a in cam["rays"])
        img = _u8(_gut(gut, ro, rd, cam["sensor"], tr.Tracer._pose_from_c2w(c2w32)))
        name = f"img_{i:03d}.png"
        write_png(os.path.join(str(tmp_path), "images_2", name), img)
        images.append(dict(id=i + 1, qvec=qvec, tvec=tvec, camera_id=cid, name=name, xys=np.zeros((0, 2)), point3D_ids=np.zeros(0, np.int64)))
        want.append((cid, img, _u8(_grt(grt, ro, rd, torch.from_numpy(c2w32[None].copy())))))
    write_colmap(str(tmp_path), cams, images, binary=True)
    conf = {"path": str(tmp_path), "dataset": {"type": "colmap", "downsample_factor": factor, "test_split_interval": 0}}
    data = scene_data.SceneData(conf)
    report = {}
    for i, (cid, img, grt_img) in enumerate(want):
        np.testing.assert_array_equal(data.train.images[i].cpu().numpy(), img)
        got_gut = _u8(_gut(gut, *data.train.view(i, "3dgut")))
        got_grt = _u8(_grt(grt, *data.train.view(i, "3dgrt")))
        if cid == 2:  # fisheye: the same rays, so the same bytes
            np.testing.assert_array_equal(got_gut, img)
            np.testing.assert_array_equal(got_grt, grt_img)
        else:
            report[f"frame {i}"] = (_psnr(got_gut, img), _psnr(got_grt, grt_img))
    print("distorted camera PSNR (3DGUT, 3DGRT):", json.dumps(report))
    for p_gut, p_grt in report.values():
        assert p_gut >= MIN_DISTORTED_PSNR and p_grt >= MIN_DISTORTED_PSNR, report

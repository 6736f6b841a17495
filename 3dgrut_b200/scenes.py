"""Synthetic Gaussian scenes and cameras of the BASELINE.json configs (SURVEY.md section 8d).

numpy only; shared by tests and bench.py.  Conventions follow the reference:
  * particle record [N,12] = pos3, density, quat(w,x,y,z), scale3, pad   (threedgut_tracer/tracer.py:176-178)
  * camera space is [right, down, front]; rays pass through pixel centres
    ((u - cx + 0.5)/fx, (v - cy + 0.5)/fy, 1) normalised  (threedgrut/datasets/dataset_nerf.py:366-368)
  * sensor pose 7-vector = t.xyz, q.xyzw of the world->sensor transform
    (threedgut_tracer/tracer.py:360-380,414-423)
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np


def so3_matrix_to_quat_xyzw(R: np.ndarray) -> np.ndarray:
    """Rotation matrix -> unit quaternion (x,y,z,w); same branch structure as the reference helper
    (threedgut_tracer/tracer.py:88-136)."""
    R = np.asarray(R, dtype=np.float64)
    d = np.array([R[0, 0], R[1, 1], R[2, 2], R[0, 0] + R[1, 1] + R[2, 2]])
    c = int(np.argmax(d))
    q = np.zeros(4)
    if c != 3:
        i, j, k = c, (c + 1) % 3, (c + 2) % 3
        q[i] = 1 - d[3] + 2 * R[i, i]
        q[j] = R[j, i] + R[i, j]
        q[k] = R[k, i] + R[i, k]
        q[3] = R[k, j] - R[j, k]
    else:
        q[0] = R[2, 1] - R[1, 2]
        q[1] = R[0, 2] - R[2, 0]
        q[2] = R[1, 0] - R[0, 1]
        q[3] = 1 + d[3]
    return (q / np.linalg.norm(q)).astype(np.float32)


def pose7_from_c2w(c2w: np.ndarray) -> np.ndarray:
    """[t.xyz, q.xyzw] of world->sensor from a camera-to-world 4x4/3x4 (tracer.py:404-423)."""
    C2W = np.eye(4)
    C2W[:3, :4] = np.asarray(c2w, dtype=np.float64)[:3, :4]
    W2C = np.linalg.inv(C2W)
    return np.concatenate([W2C[:3, 3].astype(np.float32), so3_matrix_to_quat_xyzw(W2C[:3, :3])]).astype(np.float32)


def look_at_c2w(eye, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)) -> np.ndarray:
    eye, target, up = (np.asarray(v, dtype=np.float64) for v in (eye, target, up))
    f = target - eye
    f /= np.linalg.norm(f)
    r = np.cross(f, up)
    r /= np.linalg.norm(r)
    d = np.cross(f, r)
    c2w = np.eye(4)
    c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = r, d, f, eye
    return c2w


def orbit_c2w(i: int, n: int, radius: float, elevation_deg: float = 25.0) -> np.ndarray:
    az = 2.0 * math.pi * (i + 0.37) / max(n, 1)
    el = math.radians(elevation_deg + 10.0 * math.sin(3.1 * i))
    eye = radius * np.array([math.cos(az) * math.cos(el), math.sin(az) * math.cos(el), math.sin(el)])
    return look_at_c2w(eye)


def pinhole_rays(height: int, width: int, fx: float, fy: float, cx: float, cy: float):
    """rays_o [1,H,W,3] (zeros, camera space), rays_d [1,H,W,3] normalised."""
    u, v = np.meshgrid(np.arange(width, dtype=np.float32), np.arange(height, dtype=np.float32))
    d = np.stack([(u - cx + 0.5) / fx, (v - cy + 0.5) / fy, np.ones_like(u)], -1).astype(np.float32)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    return np.zeros((1, height, width, 3), np.float32), d[None].astype(np.float32)


def fisheye_rays(height: int, width: int, fx: float, fy: float, cx: float, cy: float, fisheye):
    """Sensor-space unit rays of an OpenCV fisheye camera (inverse of cameraProjections.cuh:120-146): the pixel centre at normalised
    distance r_d = |((u+.5-cx)/fx, (v+.5-cy)/fy)| comes from the angle theta with theta (1 + k1 th^2 + k2 th^4 + k3 th^6 + k4 th^8) = r_d
    (Newton iterations in float64).  Returns ([1,H,W,3] origins = 0, [1,H,W,3] directions) float32."""
    k1, k2, k3, k4 = (float(v) for v in fisheye[:4])
    v, u = np.meshgrid(np.arange(height, dtype=np.float64), np.arange(width, dtype=np.float64), indexing="ij")
    x = (u + 0.5 - cx) / fx
    y = (v + 0.5 - cy) / fy
    rd = np.sqrt(x * x + y * y)
    th = rd.copy()
    for _ in range(20):
        t2 = th * th
        f = th * (1 + t2 * (k1 + t2 * (k2 + t2 * (k3 + t2 * k4)))) - rd
        df = 1 + t2 * (3 * k1 + t2 * (5 * k2 + t2 * (7 * k3 + t2 * 9 * k4)))
        th = th - f / df
    s = np.where(rd > 0, np.sin(th) / np.maximum(rd, 1e-30), 0.0)
    d = np.stack([x * s, y * s, np.cos(th)], -1)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    return np.zeros((1, height, width, 3), np.float32), d[None].astype(np.float32)


def ftheta_rays(height: int, width: int, ft: dict):
    """Sensor-space unit rays of an f-theta camera (inverse of cameraProjections.cuh:148-198): pixel centre (u+.5, v+.5) lies at the
    offset (u - px, v - py) from the principal point (the model's origin is the centre of the first pixel); the offset is mapped
    through the inverse of the linear term [c d; e 1] and its length r through the BACKWARD polynomial theta = bw(r)."""
    c, d, e = (float(v) for v in ft["cde"])
    px, py = (float(v) for v in ft["principal"])
    v, u = np.meshgrid(np.arange(height, dtype=np.float64), np.arange(width, dtype=np.float64), indexing="ij")
    ox, oy = u - px, v - py
    det = c - d * e
    x = (ox - d * oy) / det
    y = (-e * ox + c * oy) / det
    r = np.sqrt(x * x + y * y)
    th = np.zeros_like(r)
    for k in reversed(range(6)):
        th = th * r + float(ft["bw"][k])
    s = np.where(r > 0, np.sin(th) / np.maximum(r, 1e-30), 0.0)
    dirs = np.stack([x * s, y * s, np.cos(th)], -1)
    dirs /= np.linalg.norm(dirs, axis=-1, keepdims=True)
    return np.zeros((1, height, width, 3), np.float32), dirs[None].astype(np.float32)


@dataclass
class Scene:
    name: str
    width: int
    height: int
    fx: float
    fy: float
    particles: np.ndarray  # [N,12] post-activation
    sph: np.ndarray  # [N,48]
    sph_degree: int
    camera_radius: float
    fisheye: tuple | None = None  # (k1, k2, k3, k4, max_angle): OpenCV fisheye camera instead of the pinhole (fx, fy = pixels per radian)
    ftheta: dict | None = None    # f-theta camera: dict(reference_poly=0|1, bw=[6], fw=[6], cde=[3], max_angle=..., principal=(px, py))

    @property
    def cx(self):
        return self.width / 2.0

    @property
    def cy(self):
        return self.height / 2.0

    @property
    def n(self):
        return self.particles.shape[0]

    def camera(self, i: int, n: int = 100):
        return orbit_c2w(i, n, self.camera_radius)

    def rays(self):
        if self.ftheta is not None:
            return ftheta_rays(self.height, self.width, self.ftheta)
        if self.fisheye is not None:
            return fisheye_rays(self.height, self.width, self.fx, self.fy, self.cx, self.cy, self.fisheye)
        return pinhole_rays(self.height, self.width, self.fx, self.fy, self.cx, self.cy)


def _pack(pos, dns, quat, scl):
    n = pos.shape[0]
    quat = quat / np.linalg.norm(quat, axis=1, keepdims=True)
    return np.concatenate([pos, dns.reshape(n, 1), quat, scl, np.zeros((n, 1))], 1).astype(np.float32)


def _sph(rng, n, dc_lo, dc_hi, band_sigma):
    sph = np.zeros((n, 16, 3), np.float32)
    sph[:, 0, :] = rng.uniform(dc_lo, dc_hi, (n, 3))
    if band_sigma > 0:
        sph[:, 1:, :] = rng.normal(0.0, band_sigma, (n, 15, 3))
    return sph.reshape(n, 48).astype(np.float32)


def scene_c1(n: int = 1000, seed: int = 42, bands: bool = True, width: int = 128, height: int = 128) -> Scene:
    """C1: 1k random Gaussians, 128x128 pinhole (init_from_random_point_cloud-like,
    threedgrut/model/model.py:553-612)."""
    rng = np.random.default_rng(seed)
    pos = rng.uniform(-1.5, 1.5, (n, 3))
    # no fallback: the stored reference outputs under tests/golden/ are of this exact scene
    from scipy.spatial import cKDTree

    dist = cKDTree(pos).query(pos, k=4)[0][:, 1:].mean(1)
    scl = 0.4 * np.repeat(np.clip(dist, 1e-3, None)[:, None], 3, 1) * rng.uniform(0.6, 1.4, (n, 3))
    quat = rng.uniform(0, 1, (n, 4))
    quat[:, 0] = 1.0
    dns = rng.uniform(0.05, 0.9, n)
    fx = 0.5 * width / math.tan(0.5 * 0.6911112070083618)
    return Scene("c1_random_1k", width, height, fx, fx, _pack(pos, dns, quat, scl),
                 _sph(rng, n, 0.3, 2.5, 0.1 if bands else 0.0), 3, 4.0)


def scene_c2(n: int = 300_000, seed: int = 7, width: int = 800, height: int = 800) -> Scene:
    """C2: lego-like 800x800, trained-like distribution: shell-concentrated positions in [-1.3,1.3]^3,
    log-normal scales (median 0.01, sigma 0.7), opacity Beta(2,2), full SH."""
    rng = np.random.default_rng(seed)
    dirs = rng.normal(size=(n, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    rad = np.clip(rng.normal(0.8, 0.25, n), 0.02, 1.3)
    pos = np.clip(dirs * rad[:, None] * np.array([1.0, 1.0, 0.7]), -1.3, 1.3)
    scl = np.exp(rng.normal(math.log(0.01), 0.7, (n, 3)))
    quat = rng.normal(size=(n, 4))
    dns = rng.beta(2.0, 2.0, n)
    fx = 0.5 * width / math.tan(0.5 * 0.6911112070083618)
    return Scene("c2_lego_like_300k", width, height, fx, fx, _pack(pos, dns, quat, scl), _sph(rng, n, -1.0, 2.0, 0.15), 3, 4.0)


def scene_c3(n: int = 6_000_000, seed: int = 11, width: int = 1237, height: int = 822) -> Scene:
    """C3: bicycle-like unbounded scene: 70 % within radius 3, 30 % background out to radius 50, scale ~ distance."""
    rng = np.random.default_rng(seed)
    n_in = int(0.7 * n)
    dirs = rng.normal(size=(n, 3)).astype(np.float32)
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    rad = np.concatenate([3.0 * rng.uniform(0, 1, n_in) ** (1 / 2.0), rng.uniform(3.0, 50.0, n - n_in)]).astype(np.float32)
    pos = dirs * rad[:, None]
    pos[:, 2] *= 0.35
    scl = (np.exp(rng.normal(math.log(0.006), 0.7, (n, 3))) * np.maximum(rad, 0.5)[:, None]).astype(np.float32)
    quat = rng.normal(size=(n, 4)).astype(np.float32)
    dns = rng.beta(2.0, 2.0, n).astype(np.float32)
    return Scene("c3_bicycle_like_6m", width, height, 1040.0, 1040.0, _pack(pos, dns, quat, scl), _sph(rng, n, -1.0, 2.0, 0.15), 3, 4.5)


# C5's mirror: the floor plane z = -1.2 with render_hybrid's reflectivity (hybrid.py); on C5's orbit (elevation 15-35 deg, vertical half-angle
# 21.6 deg) most pixels look down onto it, only the top rows of the lowest views look above the horizon
C5_MIRROR = dict(plane_point=(0.0, 0.0, -1.2), plane_normal=(0.0, 0.0, 1.0), reflectivity=0.3)


def scene_c5(n: int = 5_000_000, seed: int = 23, width: int = 1237, height: int = 822) -> Scene:
    """C5: garden-like unbounded scene for the 3DGRUT hybrid (primary rays through 3DGUT, C5_MIRROR reflections through 3DGRT): C3's
    generator at 5M Gaussians with a seed of its own."""
    sc = scene_c3(n=n, seed=seed, width=width, height=height)
    sc.name = "c5_garden_like_5m"
    return sc

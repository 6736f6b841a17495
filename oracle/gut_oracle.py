"""ctypes/numpy front-end of the CPU oracle (oracle/gut_oracle.c).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module; the product package never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_LIB64 = None


class Camera(C.Structure):
    _fields_ = [
        ("width", C.c_int32), ("height", C.c_int32),
        ("principal", C.c_float * 2), ("focal", C.c_float * 2),
        ("radial", C.c_float * 6), ("tangential", C.c_float * 2), ("thin_prism", C.c_float * 4),
        ("pose_start", C.c_float * 7), ("pose_end", C.c_float * 7),
        ("model", C.c_int32), ("max_angle", C.c_float),
        ("ftheta_reference_poly", C.c_int32), ("ftheta_bw", C.c_float * 6), ("ftheta_fw", C.c_float * 6), ("ftheta_cde", C.c_float * 3),
        ("rolling_shutter", C.c_int32),
    ]


class Config(C.Structure):
    _fields_ = [
        ("kernel_degree", C.c_int32), ("min_kernel_density", C.c_float), ("min_alpha", C.c_float),
        ("max_alpha", C.c_float), ("min_transmittance", C.c_float),
        ("ut_alpha", C.c_float), ("ut_beta", C.c_float), ("ut_kappa", C.c_float), ("ut_delta", C.c_float),
        ("ut_margin", C.c_float),
        ("rect_bounding", C.c_int32), ("tight_opacity_bounding", C.c_int32), ("tile_culling", C.c_int32),
        ("global_z_order", C.c_int32), ("n_rolling_shutter_iterations", C.c_int32),
    ]


def build(force: bool = False, name: str = "libgut_oracle.so") -> str:
    so = os.path.join(_HERE, name)
    src = os.path.join(_HERE, "gut_oracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, name], stdout=subprocess.DEVNULL)
    return so


def _setup(l):
    l.gut_oracle_bin.restype = C.c_int64
    l.gut_oracle_higher_msb.restype = C.c_uint32
    l.gut_oracle_hit_forward.restype = C.c_int
    return l


def lib(f64: bool = False):
    """The oracle proper (fp32), or with f64=True the variant whose per-ray compositing maths runs in double
    on the same fp32 inputs and sorted lists (used only to size tolerances)."""
    global _LIB, _LIB64
    if f64:
        if _LIB64 is None:
            _LIB64 = _setup(C.CDLL(build(name="libgut_oracle_f64.so")))
        return _LIB64
    if _LIB is None:
        _LIB = _setup(C.CDLL(build()))
    return _LIB


def default_config() -> Config:
    cfg = Config()
    lib().gut_oracle_default_config(C.byref(cfg))
    return cfg


def make_camera(width, height, fx, fy, cx, cy, pose_start, pose_end=None, fisheye=None, ftheta=None, rolling_shutter=0) -> Camera:
    """fisheye: None (OpenCV pinhole) or (k1, k2, k3, k4, max_angle) for the OpenCV fisheye model.
    ftheta: None or dict(reference_poly=0|1, bw=[6], fw=[6], cde=[3], max_angle=..., principal=(px, py)) for the f-theta model."""
    cam = Camera()
    cam.width, cam.height = int(width), int(height)
    cam.principal[:] = [cx, cy]
    cam.focal[:] = [fx, fy]
    cam.pose_start[:] = [float(v) for v in pose_start]
    cam.pose_end[:] = [float(v) for v in (pose_end if pose_end is not None else pose_start)]
    if fisheye is not None:
        cam.model = 1
        cam.radial[0:4] = [float(v) for v in fisheye[0:4]]
        cam.max_angle = float(fisheye[4])
    if ftheta is not None:
        cam.model = 2
        cam.principal[:] = [float(v) for v in ftheta["principal"]]
        cam.ftheta_reference_poly = int(ftheta["reference_poly"])
        cam.ftheta_bw[:] = [float(v) for v in ftheta["bw"]]
        cam.ftheta_fw[:] = [float(v) for v in ftheta["fw"]]
        cam.ftheta_cde[:] = [float(v) for v in ftheta["cde"]]
        cam.max_angle = float(ftheta["max_angle"])
    cam.rolling_shutter = int(rolling_shutter)  # 0 global, 1..4 = rolling top-to-bottom / left-to-right / bottom-to-top / right-to-left
    return cam


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


@dataclass
class Projection:
    tiles_count: np.ndarray
    proj_pos: np.ndarray
    conic_opacity: np.ndarray
    extent: np.ndarray
    depth: np.ndarray
    rgb: np.ndarray
    visibility: np.ndarray


@dataclass
class Binning:
    unsorted_keys: np.ndarray
    unsorted_values: np.ndarray
    sorted_keys: np.ndarray
    sorted_values: np.ndarray
    ranges: np.ndarray


def sensor_matrices(cam: Camera):
    view = np.zeros(12, np.float32)
    inv = np.zeros(12, np.float32)
    pos = np.zeros(3, np.float32)
    lib().gut_oracle_sensor_matrices(C.byref(cam), _p(view, C.c_float), _p(inv, C.c_float), _p(pos, C.c_float))
    return view.reshape(4, 3), inv.reshape(4, 3), pos


def project(cfg, cam, particles, sph, sph_degree) -> Projection:
    particles, sph = _f32(particles), _f32(sph)
    n = particles.shape[0]
    out = Projection(np.zeros(n, np.uint32), np.zeros((n, 2), np.float32), np.zeros((n, 4), np.float32),
                     np.zeros((n, 2), np.float32), np.zeros(n, np.float32), np.zeros((n, 3), np.float32),
                     np.zeros(n, np.int32))
    lib().gut_oracle_project(C.byref(cfg), C.byref(cam), C.c_int64(n), _p(particles, C.c_float), _p(sph, C.c_float),
                             C.c_int32(sph_degree), _p(out.tiles_count, C.c_uint32), _p(out.proj_pos, C.c_float),
                             _p(out.conic_opacity, C.c_float), _p(out.extent, C.c_float), _p(out.depth, C.c_float),
                             _p(out.rgb, C.c_float), _p(out.visibility, C.c_int32))
    return out


def bin_tiles(cfg, cam, pr: Projection) -> Binning:
    n = pr.tiles_count.shape[0]
    total = int(pr.tiles_count.astype(np.int64).sum())
    gx, gy = (cam.width + 15) // 16, (cam.height + 15) // 16
    m = max(total, 1)
    b = Binning(np.zeros(m, np.uint64), np.zeros(m, np.uint32), np.zeros(m, np.uint64), np.zeros(m, np.uint32),
                np.zeros((gx * gy, 2), np.uint32))
    got = lib().gut_oracle_bin(C.byref(cfg), C.byref(cam), C.c_int64(n), _p(pr.tiles_count, C.c_uint32),
                               _p(pr.proj_pos, C.c_float), _p(pr.conic_opacity, C.c_float), _p(pr.extent, C.c_float),
                               _p(pr.depth, C.c_float), _p(b.unsorted_keys, C.c_uint64), _p(b.unsorted_values, C.c_uint32),
                               _p(b.sorted_keys, C.c_uint64), _p(b.sorted_values, C.c_uint32), _p(b.ranges, C.c_uint32))
    assert got == total
    for k in ("unsorted_keys", "unsorted_values", "sorted_keys", "sorted_values"):
        setattr(b, k, getattr(b, k)[:total])
    return b


def render_forward(cfg, cam, rays_o, rays_d, particles, pr: Projection, bn: Binning, f64: bool = False):
    rays_o, rays_d, particles = _f32(rays_o).reshape(-1, 3), _f32(rays_d).reshape(-1, 3), _f32(particles)
    h, w = cam.height, cam.width
    rgba = np.zeros((h, w, 4), np.float32)
    dist = np.zeros((h, w, 1), np.float32)
    hits = np.zeros((h, w, 1), np.float32)
    sv = bn.sorted_values if bn.sorted_values.size else np.zeros(1, np.uint32)
    lib(f64).gut_oracle_render_forward(C.byref(cfg), C.byref(cam), _p(rays_o, C.c_float), _p(rays_d, C.c_float),
                                    _p(particles, C.c_float), _p(pr.rgb, C.c_float), _p(sv, C.c_uint32),
                                    _p(bn.ranges, C.c_uint32), _p(rgba, C.c_float), _p(dist, C.c_float),
                                    _p(hits, C.c_float))
    return rgba, dist, hits


def render_forward_kbuffer(cfg, cam, k: int, rays_o, rays_d, particles, pr: Projection, bn: Binning, f64: bool = False):
    """Sorted 3DGUT forward (GAUSSIAN_K_BUFFER_SIZE = k > 0, gutKBufferRenderer.cuh:62-112,274-352); CUDA twin: gut_render_kbuffer.cu."""
    rays_o, rays_d, particles = _f32(rays_o).reshape(-1, 3), _f32(rays_d).reshape(-1, 3), _f32(particles)
    h, w = cam.height, cam.width
    rgba = np.zeros((h, w, 4), np.float32)
    dist = np.zeros((h, w, 1), np.float32)
    hits = np.zeros((h, w, 1), np.float32)
    sv = bn.sorted_values if bn.sorted_values.size else np.zeros(1, np.uint32)
    lib(f64).gut_oracle_render_forward_kbuffer(C.byref(cfg), C.byref(cam), C.c_int32(int(k)), _p(rays_o, C.c_float), _p(rays_d, C.c_float),
                                               _p(particles, C.c_float), _p(pr.rgb, C.c_float), _p(sv, C.c_uint32),
                                               _p(bn.ranges, C.c_uint32), _p(rgba, C.c_float), _p(dist, C.c_float), _p(hits, C.c_float))
    return rgba, dist, hits


def render_backward(cfg, cam, rays_o, rays_d, particles, sph, sph_degree, pr, bn, rgba, dist, d_rgba, d_dist, f64: bool = False):
    rays_o, rays_d = _f32(rays_o).reshape(-1, 3), _f32(rays_d).reshape(-1, 3)
    particles, sph = _f32(particles), _f32(sph)
    rgba, dist, d_rgba, d_dist = _f32(rgba), _f32(dist), _f32(d_rgba), _f32(d_dist)
    n = particles.shape[0]
    dp = np.zeros((n, 12), np.float32)
    ds = np.zeros((n, 48), np.float32)
    sv = bn.sorted_values if bn.sorted_values.size else np.zeros(1, np.uint32)
    lib(f64).gut_oracle_render_backward(C.byref(cfg), C.byref(cam), C.c_int64(n), _p(rays_o, C.c_float), _p(rays_d, C.c_float),
                                     _p(particles, C.c_float), _p(sph, C.c_float), C.c_int32(sph_degree),
                                     _p(pr.rgb, C.c_float), _p(pr.tiles_count, C.c_uint32), _p(sv, C.c_uint32),
                                     _p(bn.ranges, C.c_uint32), _p(rgba, C.c_float), _p(dist, C.c_float),
                                     _p(d_rgba, C.c_float), _p(d_dist, C.c_float), _p(dp, C.c_float), _p(ds, C.c_float))
    return dp, ds


def render_backward_kbuffer(cfg, cam, k: int, rays_o, rays_d, particles, sph, sph_degree, pr, bn, rgba, dist, d_rgba, d_dist, f64: bool = False):
    """Adjoint of render_forward_kbuffer (the per-hit adjoint applied in the buffer's processing order) + the SH adjoint."""
    rays_o, rays_d = _f32(rays_o).reshape(-1, 3), _f32(rays_d).reshape(-1, 3)
    particles, sph = _f32(particles), _f32(sph)
    rgba, dist, d_rgba, d_dist = _f32(rgba), _f32(dist), _f32(d_rgba), _f32(d_dist)
    n = particles.shape[0]
    dp = np.zeros((n, 12), np.float32)
    ds = np.zeros((n, 48), np.float32)
    sv = bn.sorted_values if bn.sorted_values.size else np.zeros(1, np.uint32)
    lib(f64).gut_oracle_render_backward_kbuffer(C.byref(cfg), C.byref(cam), C.c_int32(int(k)), C.c_int64(n), _p(rays_o, C.c_float),
                                                _p(rays_d, C.c_float), _p(particles, C.c_float), _p(sph, C.c_float), C.c_int32(sph_degree),
                                                _p(pr.rgb, C.c_float), _p(pr.tiles_count, C.c_uint32), _p(sv, C.c_uint32),
                                                _p(bn.ranges, C.c_uint32), _p(rgba, C.c_float), _p(dist, C.c_float),
                                                _p(d_rgba, C.c_float), _p(d_dist, C.c_float), _p(dp, C.c_float), _p(ds, C.c_float))
    return dp, ds


def forward_all(cfg, cam, rays_o, rays_d, particles, sph, sph_degree):
    pr = project(cfg, cam, particles, sph, sph_degree)
    bn = bin_tiles(cfg, cam, pr)
    rgba, dist, hits = render_forward(cfg, cam, rays_o, rays_d, particles, pr, bn)
    return pr, bn, rgba, dist, hits


def hit_forward(cfg, ro, rd, particle):
    a, t = C.c_float(0), C.c_float(0)
    acc = lib().gut_oracle_hit_forward(C.byref(cfg), _p(_f32(ro), C.c_float), _p(_f32(rd), C.c_float), _p(_f32(particle), C.c_float),
                                       C.byref(a), C.byref(t))
    return acc, a.value, t.value


def hit_backward(cfg, ro, rd, particle, prgb, Tint, T, Tgrad, Cint, Cacc, Cgrad, Dint, D, Dgrad):
    T_, D_ = C.c_float(T), C.c_float(D)
    Cc = _f32(Cacc).copy()
    grad, rg = np.zeros(11, np.float32), np.zeros(3, np.float32)
    acc = lib().gut_oracle_hit_backward(C.byref(cfg), _p(_f32(ro), C.c_float), _p(_f32(rd), C.c_float), _p(_f32(particle), C.c_float),
                                        _p(_f32(prgb), C.c_float), C.c_float(Tint), C.byref(T_), C.c_float(Tgrad), _p(_f32(Cint), C.c_float),
                                        _p(Cc, C.c_float), _p(_f32(Cgrad), C.c_float), C.c_float(Dint), C.byref(D_), C.c_float(Dgrad),
                                        _p(grad, C.c_float), _p(rg, C.c_float))
    return acc, grad, rg, T_.value, Cc, D_.value


def sph_eval(degree, coeffs, direction):
    out = np.zeros(3, np.float32)
    lib().gut_oracle_sph_eval(C.c_int32(degree), _p(_f32(coeffs), C.c_float), _p(_f32(direction), C.c_float), _p(out, C.c_float))
    return out


def set_tile_stride(k: int):
    lib().gut_oracle_set_tile_stride(C.c_int(int(k)))


# ---------------------------------------------------------------------------------------------------------------
# 3DGRT brute-force oracle (grt_oracle_* in gut_oracle.c)

def grt_config() -> Config:
    """configs/render/3dgrt.yaml: degree-4 kernel, min transmittance 1e-3."""
    cfg = default_config()
    cfg.kernel_degree = 4
    cfg.min_transmittance = 0.001
    return cfg


def grt_proxies(cfg, particles, clamping=True):
    particles = _f32(particles)
    n = particles.shape[0]
    kscl, bb = np.zeros((n, 3), np.float32), np.zeros(6, np.float32)
    lib().grt_oracle_proxies(C.byref(cfg), C.c_int32(int(clamping)), C.c_int64(n), _p(particles, C.c_float), _p(kscl, C.c_float), _p(bb, C.c_float))
    return kscl, bb


def grt_trace(cfg, particles, sph, sph_degree, rays_o, rays_d, ray_to_world, clamping=True, f64=False):
    particles, sph = _f32(particles), _f32(sph)
    shape = np.asarray(rays_o).shape[:-1]
    ro, rd = _f32(rays_o).reshape(-1, 3), _f32(rays_d).reshape(-1, 3)
    r2w = _f32(np.asarray(ray_to_world)[:3, :4])
    n, r = particles.shape[0], ro.shape[0]
    rgb, alpha, dist, hits, vis = (np.zeros((r, 3), np.float32), np.zeros(r, np.float32), np.zeros((r, 2), np.float32),
                                   np.zeros(r, np.float32), np.zeros(max(n, 1), np.float32))
    lib(f64).grt_oracle_trace(C.byref(cfg), C.c_int32(int(clamping)), C.c_int64(n), _p(particles, C.c_float), _p(sph, C.c_float),
                              C.c_int32(sph_degree), C.c_int64(r), _p(ro, C.c_float), _p(rd, C.c_float), _p(r2w, C.c_float),
                              _p(rgb, C.c_float), _p(alpha, C.c_float), _p(dist, C.c_float), _p(hits, C.c_float), _p(vis, C.c_float))
    return (rgb.reshape(*shape, 3), alpha.reshape(*shape, 1), dist.reshape(*shape, 2), hits.reshape(*shape, 1), vis[:n].reshape(n, 1))


def grt_trace_bwd(cfg, particles, sph, sph_degree, rays_o, rays_d, ray_to_world, rgb, alpha, dist, d_rgb, d_alpha, d_dist,
                  clamping=True, f64=False):
    particles, sph = _f32(particles), _f32(sph)
    ro, rd = _f32(rays_o).reshape(-1, 3), _f32(rays_d).reshape(-1, 3)
    r2w = _f32(np.asarray(ray_to_world)[:3, :4])
    n, r = particles.shape[0], ro.shape[0]
    rgb, alpha, dist = _f32(rgb).reshape(r, 3), _f32(alpha).reshape(r), _f32(dist).reshape(r, 2)
    d_rgb, d_alpha, d_dist = _f32(d_rgb).reshape(r, 3), _f32(d_alpha).reshape(r), _f32(d_dist).reshape(r)
    dp, ds = np.zeros((max(n, 1), 12), np.float32), np.zeros((max(n, 1), 48), np.float32)
    lib(f64).grt_oracle_trace_bwd(C.byref(cfg), C.c_int32(int(clamping)), C.c_int64(n), _p(particles, C.c_float), _p(sph, C.c_float),
                                  C.c_int32(sph_degree), C.c_int64(r), _p(ro, C.c_float), _p(rd, C.c_float), _p(r2w, C.c_float),
                                  _p(rgb, C.c_float), _p(alpha, C.c_float), _p(dist, C.c_float), _p(d_rgb, C.c_float),
                                  _p(d_alpha, C.c_float), _p(d_dist, C.c_float), _p(dp, C.c_float), _p(ds, C.c_float))
    return dp[:n], ds[:n]

"""ctypes front-end of the 3DGRT oracle with the reference's icosahedron proxies (tests/host_emul/grt_icosahedron_oracle.c).
TEST INFRASTRUCTURE ONLY.

grt_proxies / grt_trace / grt_trace_bwd take the arguments of their namesakes in oracle/gut_oracle.py plus
primitive="instances" | "icosahedron"; "instances" calls the oracle proper.  The library is compiled on first use into a
per-user temporary directory (the tree may be read-only), fp32 and -DORACLE_F64 like oracle/Makefile.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import gut_oracle as go

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "host_emul", "grt_icosahedron_oracle.c")
DEPS = [SRC, os.path.join(ROOT, "oracle", "gut_oracle.c"), os.path.join(ROOT, "oracle", "gut_oracle.h")]
_LIBS = {}


def _build(f64: bool) -> str:
    h = hashlib.sha256()
    for p in DEPS:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(b"f64" if f64 else b"f32")
    out_dir = os.path.join(tempfile.gettempdir(), f"grt_ico_oracle_{os.getuid()}")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, f"libgrt_ico_oracle_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        cc = os.environ.get("CC", "gcc")
        flags = ["-O2", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-w"]  # oracle/Makefile
        if os.path.isdir("/usr/lib/gcc/x86_64-linux-gnu/13"):
            flags.insert(0, "-B/usr/lib/gcc/x86_64-linux-gnu/13")
        if f64:
            flags.append("-DORACLE_F64")
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.check_call([cc, *flags, "-shared", "-o", tmp, SRC, "-lm"])
        os.replace(tmp, so)
    return so


def lib(f64: bool = False):
    if f64 not in _LIBS:
        _LIBS[f64] = C.CDLL(_build(f64))
    return _LIBS[f64]


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _check(primitive):
    if primitive not in ("instances", "icosahedron"):
        raise ValueError(f"unknown primitive {primitive!r}")
    return primitive == "icosahedron"


def table():
    """The reference's icosahedron: unscaled vertices [12,3] and faces [20,3] (particlePrimitives.cu:468-486)."""
    v, t = np.zeros((12, 3), np.float32), np.zeros((20, 3), np.int32)
    lib().grt_ico_oracle_table(_p(v, C.c_float), _p(t, C.c_int32))
    return v, t


ICO_VRT_SCALE = float(np.float32(0.5 * float(np.float32(1.323169076499215))))  # icosaVrtScale


def grt_proxies(cfg, particles, clamping=True, primitive="instances"):
    """instances: (kscl [N,3], scene box [6]); icosahedron: (world-space vertices [N,12,3], scene box [6])."""
    if not _check(primitive):
        return go.grt_proxies(cfg, particles, clamping)
    particles = _f32(particles)
    n = particles.shape[0]
    vrt, bb = np.zeros((max(n, 1), 12, 3), np.float32), np.zeros(6, np.float32)
    lib().grt_ico_oracle_proxies(C.byref(cfg), C.c_int32(int(clamping)), C.c_int64(n), _p(particles, C.c_float), _p(vrt, C.c_float),
                                 _p(bb, C.c_float))
    return vrt[:n], bb


def entry_t(cfg, particles, rays_o, rays_d, tmin=0.0, clamping=True, f64=False):
    """Icosahedron candidate keys of world-space rays x particles: smallest front-face t beyond tmin, +inf where there is none
    (f64: triangles intersected in double)."""
    particles = _f32(particles)
    ro, rd = _f32(rays_o).reshape(-1, 3), _f32(rays_d).reshape(-1, 3)
    n, r = particles.shape[0], ro.shape[0]
    t = np.zeros((r, max(n, 1)), np.float32)
    lib(f64).grt_ico_oracle_entry(C.byref(cfg), C.c_int32(int(clamping)), C.c_int64(n), _p(particles, C.c_float), C.c_int64(r),
                               _p(ro, C.c_float), _p(rd, C.c_float), C.c_float(tmin), _p(t, C.c_float))
    return t[:, :n]


def grt_trace(cfg, particles, sph, sph_degree, rays_o, rays_d, ray_to_world, clamping=True, f64=False, primitive="instances"):
    if not _check(primitive):
        return go.grt_trace(cfg, particles, sph, sph_degree, rays_o, rays_d, ray_to_world, clamping=clamping, f64=f64)
    particles, sph = _f32(particles), _f32(sph)
    shape = np.asarray(rays_o).shape[:-1]
    ro, rd = _f32(rays_o).reshape(-1, 3), _f32(rays_d).reshape(-1, 3)
    r2w = _f32(np.asarray(ray_to_world)[:3, :4])
    n, r = particles.shape[0], ro.shape[0]
    rgb, alpha, dist, hits, vis = (np.zeros((r, 3), np.float32), np.zeros(r, np.float32), np.zeros((r, 2), np.float32),
                                   np.zeros(r, np.float32), np.zeros(max(n, 1), np.float32))
    lib(f64).grt_ico_oracle_trace(C.byref(cfg), C.c_int32(int(clamping)), C.c_int64(n), _p(particles, C.c_float), _p(sph, C.c_float),
                                  C.c_int32(sph_degree), C.c_int64(r), _p(ro, C.c_float), _p(rd, C.c_float), _p(r2w, C.c_float),
                                  _p(rgb, C.c_float), _p(alpha, C.c_float), _p(dist, C.c_float), _p(hits, C.c_float), _p(vis, C.c_float))
    return (rgb.reshape(*shape, 3), alpha.reshape(*shape, 1), dist.reshape(*shape, 2), hits.reshape(*shape, 1), vis[:n].reshape(n, 1))


def grt_trace_bwd(cfg, particles, sph, sph_degree, rays_o, rays_d, ray_to_world, rgb, alpha, dist, d_rgb, d_alpha, d_dist,
                  clamping=True, f64=False, primitive="instances"):
    if not _check(primitive):
        return go.grt_trace_bwd(cfg, particles, sph, sph_degree, rays_o, rays_d, ray_to_world, rgb, alpha, dist, d_rgb, d_alpha, d_dist,
                                clamping=clamping, f64=f64)
    particles, sph = _f32(particles), _f32(sph)
    ro, rd = _f32(rays_o).reshape(-1, 3), _f32(rays_d).reshape(-1, 3)
    r2w = _f32(np.asarray(ray_to_world)[:3, :4])
    n, r = particles.shape[0], ro.shape[0]
    rgb, alpha, dist = _f32(rgb).reshape(r, 3), _f32(alpha).reshape(r), _f32(dist).reshape(r, 2)
    d_rgb, d_alpha, d_dist = _f32(d_rgb).reshape(r, 3), _f32(d_alpha).reshape(r), _f32(d_dist).reshape(r)
    dp, ds = np.zeros((max(n, 1), 12), np.float32), np.zeros((max(n, 1), 48), np.float32)
    lib(f64).grt_ico_oracle_trace_bwd(C.byref(cfg), C.c_int32(int(clamping)), C.c_int64(n), _p(particles, C.c_float), _p(sph, C.c_float),
                                      C.c_int32(sph_degree), C.c_int64(r), _p(ro, C.c_float), _p(rd, C.c_float), _p(r2w, C.c_float),
                                      _p(rgb, C.c_float), _p(alpha, C.c_float), _p(dist, C.c_float), _p(d_rgb, C.c_float),
                                      _p(d_alpha, C.c_float), _p(d_dist, C.c_float), _p(dp, C.c_float), _p(ds, C.c_float))
    return dp[:n], ds[:n]


def paper_config(degree: int):
    """oracle config of configs/paper/3dgrt/base_ours_reference.yaml (degree 2) / base_ours.yaml (degree 4); clamping is passed
    separately (False there)."""
    cfg = go.grt_config()
    cfg.kernel_degree = int(degree)
    return cfg

"""Shared helpers of the tests."""
import os
import re

import numpy as np

import scenes
from oracle import gut_oracle as go

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def prototypes(header):
    """{name: (return type, [parameter types])} of the functions include/<header> declares, comments stripped; a parameter type keeps
    its `const` and `*` ("const float*", "float* const*"), `(void)` is no parameters."""
    text = open(os.path.join(ROOT, "include", header)).read()
    text = re.sub(r"/\*.*?\*/|//[^\n]*", "", text, flags=re.S)
    out = {}
    for ret, name, params in re.findall(r"^[ \t]*([A-Za-z_][\w \t*]*?)\s*\b([a-z]+b200_\w+)\s*\(([^;]*?)\)\s*;", text, re.M):
        types = [re.sub(r"\s*\b\w+\s*$", "", p.strip()) for p in params.split(",") if p.strip() not in ("", "void")]
        out[name] = (ret.strip(), types)
    return out


def declared(header):
    """Names of the functions include/<header> declares."""
    return set(prototypes(header))


def oracle_camera(sc, c2w, pose=None):
    pose = scenes.pose7_from_c2w(c2w) if pose is None else pose
    return go.make_camera(sc.width, sc.height, sc.fx, sc.fy, sc.cx, sc.cy, pose, fisheye=getattr(sc, "fisheye", None),
                          ftheta=getattr(sc, "ftheta", None)), pose


def tracer_pose(c2w):
    """The [t, q.xyzw] pose the reference-facing Tracer derives from a float32 T_to_world (tracer.py:404-423)."""
    from threedgut_tracer.tracer import Tracer

    return Tracer._pose_from_c2w(np.asarray(c2w, np.float32))


def oracle_frame(sc, c2w, seed=0, pose=None, with_f64=False):
    """Full oracle forward + backward for one camera; returns a dict of numpy arrays.  with_f64 adds the
    double-precision evaluation of the compositing on the same lists (keys *_64): the tolerance yardstick."""
    cfg = go.default_config()
    cam, pose = oracle_camera(sc, c2w, pose)
    ro, rd = sc.rays()
    pr, bn, rgba, dist, hits = go.forward_all(cfg, cam, ro, rd, sc.particles, sc.sph, sc.sph_degree)
    rng = np.random.default_rng(seed)
    d_rgba = rng.normal(size=rgba.shape).astype(np.float32)
    d_dist = (0.1 * rng.normal(size=dist.shape)).astype(np.float32)
    dp, ds = go.render_backward(cfg, cam, ro, rd, sc.particles, sc.sph, sc.sph_degree, pr, bn, rgba, dist, d_rgba, d_dist)
    out = dict(cfg=cfg, cam=cam, pose=pose, ro=ro, rd=rd, pr=pr, bn=bn, rgba=rgba, dist=dist, hits=hits, d_rgba=d_rgba,
               d_dist=d_dist, dp=dp, ds=ds)
    if with_f64:
        r64, d64, h64 = go.render_forward(cfg, cam, ro, rd, sc.particles, pr, bn, f64=True)
        dp64, ds64 = go.render_backward(cfg, cam, ro, rd, sc.particles, sc.sph, sc.sph_degree, pr, bn, r64, d64, d_rgba, d_dist, f64=True)
        out.update(rgba_64=r64, dist_64=d64, hits_64=h64, dp_64=dp64, ds_64=ds64)
    return out


def kbuffer_premises(label, cfg, cam, k, ro, rd, particles, pr, bn, hits):
    """What a k-buffer case exercises, from the oracle on the same lists: the longest tile list, the share of pixels whose ray accepts more
    than k hits (the full buffer flushes its closest hit before the list ends), and the pixels whose ray stops below min_transmittance
    before its last accepted hit -- at a flush (the walk stops inside the list) or while the buffer drains after the list.  `hits` are the
    case's composited hit counts.  The accepted hits of every ray come from the float64 oracle with min_transmittance = 0 (nothing stops,
    nothing underflows)."""
    lens = bn.ranges[:, 1].astype(np.int64) - bn.ranges[:, 0]
    open_cfg = type(cfg).from_buffer_copy(cfg)
    open_cfg.min_transmittance = 0.0
    accepted = go.render_forward_kbuffer(open_cfg, cam, k, ro, rd, particles, pr, bn, f64=True)[2].reshape(-1)
    hits = np.asarray(hits, np.float32).reshape(-1)
    stopped = hits < accepted
    out = dict(longest=int(lens.max()) if lens.size else 0, over_k=float(np.mean(accepted > k)),
               at_flush=float(np.mean(stopped & (hits <= accepted - k))), in_drain=float(np.mean(stopped & (hits > accepted - k))))
    print(f"[kbuffer] {label} K={k}: longest tile list {out['longest']}, pixels with > K accepted hits {out['over_k'] * 100:.2f} %, "
          f"stopped below min_transmittance at a flush {out['at_flush'] * 100:.2f} % / while draining {out['in_drain'] * 100:.2f} %")
    return out


def image_error_report(name, got, ref, atol=1e-4):
    """(mean abs err, max abs err, number of pixels with any channel off by more than atol)"""
    e = np.abs(np.asarray(got, np.float64) - np.asarray(ref, np.float64)).reshape(ref.shape[0] * ref.shape[1], -1).max(1)
    rep = (float(e.mean()), float(e.max()), int((e > atol).sum()))
    print(f"[parity] {name}: mean|err|={rep[0]:.3e} max|err|={rep[1]:.3e} pixels>{atol:g}: {rep[2]}/{e.size}")
    return rep


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


def ray_sample(height, width, k, seed):
    """Sorted flat pixel indices of a seeded uniform sample of k pixels of a height x width frame, plus its last row and last column
    (the partly filled 8x4 ray blocks of a ragged frame)."""
    idx = np.random.default_rng(seed).choice(height * width, size=k, replace=False)
    edge = np.concatenate([(height - 1) * width + np.arange(width), np.arange(height) * width + width - 1])
    return np.unique(np.concatenate([idx, edge]))


def frac_within(a, b, atol):
    return float(np.mean(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)) <= atol))

"""Shared helpers of the tests."""
import dataclasses
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


D_DIST_MODES = ("random", "zero", "mixed")


def warp_blocks(height, width):
    """[H, W] index of the 8x4 pixel block each pixel belongs to: the pixels of one warp of the render kernels (tile_pixel,
    render_tile.cuh).  Tiles are 16x16 and start on multiples of 16, so the blocks tile the frame from its origin."""
    y, x = np.mgrid[0:height, 0:width]
    return (y // 4) * ((width + 7) // 8) + x // 8


def dist_grad_mask(height, width, mode, seed=0):
    """[H, W] bool: the pixels whose distance gradient is non-zero.  "random": all; "zero": none (every training step: no loss term
    reads the distance, so each warp of the backward skips its depth branch); "mixed": every third 8x4 warp block plus a seeded 1 % of
    the other pixels, so warps with and without the depth branch add into the same gradient rows, and some warps run it with most lanes
    at zero."""
    if mode == "random":
        return np.ones((height, width), bool)
    if mode == "zero":
        return np.zeros((height, width), bool)
    if mode == "mixed":
        rng = np.random.default_rng(1000 + seed)
        return (warp_blocks(height, width) % 3 == 0) | (rng.random((height, width)) < 0.01)
    raise ValueError(mode)


def dist_grad_blocks(d_dist):
    """(warp blocks with a non-zero distance gradient on some pixel, warp blocks without) of an [H, W(, 1)] gradient."""
    h, w = d_dist.shape[:2]
    blocks = warp_blocks(h, w).reshape(-1)
    has = np.zeros(blocks.max() + 1, bool)
    np.logical_or.at(has, blocks, np.asarray(d_dist).reshape(h * w, -1).any(1))
    return int(has.sum()), int((~has).sum())


def output_grads(shape_rgba, seed=0, d_dist="random", d_alpha="random"):
    """The seeded output gradients (d_rgba [H,W,C], d_dist [H,W,1]) of a backward; d_dist in D_DIST_MODES (dist_grad_mask), d_alpha
    "zero" clears the last channel (an L1 / L2 image loss on a black background never reads the opacity).  "random" in both draws
    what this helper always drew."""
    h, w = shape_rgba[:2]
    rng = np.random.default_rng(seed)
    d_rgba = rng.normal(size=shape_rgba).astype(np.float32)
    dd = (0.1 * rng.normal(size=(h, w, 1))).astype(np.float32)
    dd *= dist_grad_mask(h, w, d_dist, seed)[..., None]
    if d_alpha == "zero":
        d_rgba[..., -1] = 0.0
    elif d_alpha != "random":
        raise ValueError(d_alpha)
    return d_rgba, dd


def oracle_frame(sc, c2w, seed=0, pose=None, with_f64=False, d_dist="random", d_alpha="random"):
    """Full oracle forward + backward for one camera; returns a dict of numpy arrays.  with_f64 adds the
    double-precision evaluation of the compositing on the same lists (keys *_64): the tolerance yardstick.  d_dist / d_alpha: which
    output gradients the backward gets (output_grads); the float64 backward gets the same ones."""
    cfg = go.default_config()
    cam, pose = oracle_camera(sc, c2w, pose)
    ro, rd = sc.rays()
    pr, bn, rgba, dist, hits = go.forward_all(cfg, cam, ro, rd, sc.particles, sc.sph, sc.sph_degree)
    d_rgba, d_dist = output_grads(rgba.shape, seed, d_dist, d_alpha)
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


def tile_sample(ranges, height, width, heaviest=16, k=48, seed=0):
    """Sorted indices of a sample of the 16x16 tiles of a height x width frame: the `heaviest` longest lists of `ranges` ([T, 2] begin /
    end of each tile's list), every tile of the last row and last column (partly filled on a ragged frame), and a seeded `k` others."""
    gx, gy = (width + 15) // 16, (height + 15) // 16
    lens = ranges[:, 1].astype(np.int64) - ranges[:, 0]
    heavy = np.argsort(-lens, kind="stable")[:heaviest]
    edge = np.concatenate([(gy - 1) * gx + np.arange(gx), np.arange(gy) * gx + gx - 1])
    rest = np.setdiff1d(np.arange(gx * gy), np.concatenate([heavy, edge]))
    pick = np.random.default_rng(seed).choice(rest, size=min(k, rest.size), replace=False)
    return np.unique(np.concatenate([heavy, edge, pick]))


def restrict_to_tiles(particles, sph, pr, bn, tiles):
    """The oracle's frame cut down to the tiles `tiles`: a copy of the binning `bn` in which every other tile has an empty list, over
    the particles those lists name alone.  Returns (rows, particles, sph, pr, bn): `rows` are the sorted indices of the kept particles in
    the full scene, and the kept lists name them by their position in `rows`.  A pixel reads only its tile's list, so on the sampled
    pixels the oracle's forward over the cut frame is the full frame's; with the output gradients zero on every other pixel, so is its
    backward at `rows`, and every other particle's gradient is zero (tests/test_oracle_tile_sample.py pins both).  Dropping the other
    particles keeps the backward's per-thread float64 accumulators at the size of the sample instead of the scene."""
    ranges = np.zeros_like(bn.ranges)
    ranges[tiles] = bn.ranges[tiles]
    keep = np.zeros(len(bn.sorted_values), bool)
    for b, e in bn.ranges[tiles]:
        keep[b:e] = True
    keep &= bn.sorted_values != 0xFFFFFFFF  # a list ends at its first invalid entry; that one stays as it is
    rows = np.unique(bn.sorted_values[keep])
    values = bn.sorted_values.copy()
    values[keep] = np.searchsorted(rows, bn.sorted_values[keep]).astype(np.uint32)
    sub_pr = dataclasses.replace(pr, **{f.name: getattr(pr, f.name)[rows] for f in dataclasses.fields(pr)})
    sub_bn = dataclasses.replace(bn, sorted_values=values, ranges=ranges)
    return rows, particles[rows], sph[rows], sub_pr, sub_bn


def tile_pixels(tiles, height, width):
    """[H, W] bool: the pixels of the 16x16 tiles `tiles` (row-major tile index, (width + 15) // 16 tiles per row)."""
    gx = (width + 15) // 16
    y, x = np.mgrid[0:height, 0:width]
    mask = np.zeros(((height + 15) // 16) * gx, bool)
    mask[tiles] = True
    return mask[(y // 16) * gx + x // 16]


def frac_within(a, b, atol):
    return float(np.mean(np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)) <= atol))

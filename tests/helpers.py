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
    pr = go.project(cfg, cam, sc.particles, sc.sph, sc.sph_degree)
    bn = go.bin_tiles(cfg, cam, pr)
    d_rgba, d_dist = output_grads((cam.height, cam.width, 4), seed, d_dist, d_alpha)
    out = oracle_on_lists(cfg, cam, ro, rd, sc.particles, sc.sph, sc.sph_degree, pr, bn, d_rgba, d_dist, with_f64=with_f64)
    out.update(cfg=cfg, cam=cam, pose=pose, ro=ro, rd=rd, pr=pr, bn=bn, d_rgba=d_rgba, d_dist=d_dist)
    return out


def oracle_on_lists(cfg, cam, ro, rd, particles, sph, sph_degree, pr, bn, d_rgba, d_dist, k=0, with_f64=True, spreads=False):
    """The oracle's forward (rgba, dist, hits) and backward (dp, ds) over the lists of the binning `bn`, with the radiance and tile counts
    of the projection `pr`; with_f64 adds the float64 evaluation of the compositing on the same lists (keys *_64), the yardstick of the
    gradient bar; spreads adds "spreads": the (dp, ds) of that and of the float32 oracle with nudged_configs, for check_gradients.  k > 0:
    the sorted variant with a buffer of k hits."""
    out = {}
    if spreads:
        out["spreads"] = [oracle_on_lists(c, cam, ro, rd, particles, sph, sph_degree, pr, bn, d_rgba, d_dist, k, with_f64=False)
                          for c in nudged_configs(cfg)]
        out["spreads"] = [(o["dp"], o["ds"]) for o in out["spreads"]]
    for f64 in (False, True) if with_f64 else (False,):
        if k:
            rgba, dist, hits = go.render_forward_kbuffer(cfg, cam, k, ro, rd, particles, pr, bn, f64=f64)
            dp, ds = go.render_backward_kbuffer(cfg, cam, k, ro, rd, particles, sph, sph_degree, pr, bn, rgba, dist, d_rgba, d_dist, f64=f64)
        else:
            rgba, dist, hits = go.render_forward(cfg, cam, ro, rd, particles, pr, bn, f64=f64)
            dp, ds = go.render_backward(cfg, cam, ro, rd, particles, sph, sph_degree, pr, bn, rgba, dist, d_rgba, d_dist, f64=f64)
        sfx = "_64" if f64 else ""
        out.update({"rgba" + sfx: rgba, "dist" + sfx: dist, "hits" + sfx: hits, "dp" + sfx: dp, "ds" + sfx: ds})
    if spreads:
        out["spreads"].append((out["dp_64"], out["ds_64"]))
    return out


def nudged_configs(cfg, rel=5e-5):
    """Two copies of the oracle config `cfg` with the accept thresholds (min_kernel_density, min_alpha) and the early stop
    (min_transmittance) moved by -rel and +rel of their values.  The oracle run with them changes the gradient of exactly the particles
    with a (pixel, particle) pair on the edge of a decision, which the render kernels' approximate exp may take the other way even where
    the oracle's float32 and float64 evaluations agree."""
    out = []
    for s in (-rel, rel):
        c = type(cfg).from_buffer_copy(cfg)
        for f in ("min_kernel_density", "min_alpha", "min_transmittance"):
            setattr(c, f, getattr(c, f) * (1.0 + s))
        out.append(c)
    return out


GRAD_COLS = dict(pos=slice(0, 3), dns=slice(3, 4), quat=slice(4, 8), scl=slice(8, 11))


def check_gradients(label, dp, ds, ref, spreads):
    """The gradient bar of test_gut_headline_parity_gpu.py against the oracle's (ref_dp, ref_ds) = `ref`, with the oracle's own spread
    taken over several evaluations on the same lists, `spreads` = [(dp, ds), ...] (float32 against float64, nudged_configs).  Per tensor
    (pos, density, quat, scale, sph): err <= max(1e-3, 1.5 x the largest spread), and err <= 1e-3 once the ten particles whose gradient
    moves most across those evaluations are left out -- picked from the oracle, never from the output under test."""
    rdp, rds = np.asarray(ref[0], np.float64), np.asarray(ref[1], np.float64)
    pairs = {k: (dp[:, v], rdp[:, v]) for k, v in GRAD_COLS.items()}
    pairs["sph"] = (ds, rds)
    errs = {k: rel_l2(a, b) for k, (a, b) in pairs.items()}
    yard = {k: max(rel_l2(b if k == "sph" else a[:, GRAD_COLS[k]], pairs[k][1]) for a, b in spreads) for k in pairs}
    e2 = np.zeros(len(dp))
    for a, b in spreads:
        e2 = np.maximum(e2, ((np.asarray(a, np.float64)[:, 0:11] - rdp[:, 0:11]) ** 2).sum(1) / max(float((rdp[:, 0:11] ** 2).sum()), 1e-300)
                        + ((np.asarray(b, np.float64) - rds) ** 2).sum(1) / max(float((rds ** 2).sum()), 1e-300))
    keep = np.ones(len(dp), bool)
    keep[np.argsort(-e2)[:10]] = False
    robust = {k: rel_l2(a[keep], b[keep]) for k, (a, b) in pairs.items()}
    fmt = lambda d: {k: f"{v:.2e}" for k, v in d.items()}  # noqa: E731
    print(f"[gradients] {label} rel-L2 vs oracle: {fmt(errs)}; oracle spread (bar max(1e-3, 1.5 x)): {fmt(yard)}; without the oracle's "
          f"10 most unsettled particles (bar 1e-3): {fmt(robust)}")
    for k in errs:
        assert errs[k] <= max(1e-3, 1.5 * yard[k]), (k, errs[k], yard[k])
        assert robust[k] <= 1e-3, (k, robust[k])


def binning_from_lists(sorted_keys, sorted_values, ranges):
    """An oracle Binning over sorted tile lists made elsewhere (the GPU's: gpu_binning).  The oracle's renders read only `sorted_values`
    and `ranges` of a Binning (gut_oracle.c: gut_oracle_render_forward*, render_backward_impl).  The key fields hold the lists' own
    (tile << 32 | depth bits) keys, sorted and unsorted alike: the order the lists were binned in is not known, and no render reads it."""
    keys, values = np.asarray(sorted_keys, np.uint64), np.asarray(sorted_values, np.uint32)
    return go.Binning(unsorted_keys=keys.copy(), unsorted_values=values.copy(), sorted_keys=keys, sorted_values=values,
                      ranges=np.ascontiguousarray(ranges, np.uint32))


def gpu_binning(ctx):
    """The sorted tile lists the last forward of the native context `ctx` walked, as an oracle Binning.  DBG_SORTED_KEYS are the
    reference's 64-bit keys, rebuilt on the device from the tile ranges, the sorted values and the depths."""
    import b200_native as nat

    return binning_from_lists(ctx.debug_copy(nat.DBG_SORTED_KEYS), ctx.debug_copy(nat.DBG_SORTED_VALUES), ctx.debug_copy(nat.DBG_TILE_RANGES))


def sh_radiance(cam, particles, sph, sph_degree, rows):
    """[len(rows), 3] radiance of the particles `rows` as gut_oracle_project evaluates it: the SH along the float32 unit direction from the
    camera position (gut_oracle_sensor_matrices) to the particle, whatever the sensor model."""
    campos = go.sensor_matrices(cam)[2]
    out = np.zeros((len(rows), 3), np.float32)
    for j, i in enumerate(rows):
        s = np.asarray(particles[i, 0:3], np.float32) - campos
        dist = np.sqrt(s[0] * s[0] + s[1] * s[1] + s[2] * s[2])
        out[j] = go.sph_eval(sph_degree, sph[i], s / dist)
    return out


def projection_for_lists(pr, tiles_count, cam, particles, sph, sph_degree):
    """The oracle's projection `pr` with the tile counts `tiles_count` of other lists (the GPU's).  The renders read two fields of a
    Projection: the radiance `rgb`, and in the backward whether a particle's count is non-zero (only counted particles get the SH adjoint).
    The oracle leaves the radiance zero where its own count is zero, so the particles only the other lists count get theirs from
    sh_radiance.  The conic, extent and depth stay the oracle's: the renders evaluate each particle in 3D and never read them."""
    tiles_count = np.asarray(tiles_count, np.uint32)
    rgb = pr.rgb.copy()
    extra = np.flatnonzero((tiles_count > 0) & (pr.tiles_count == 0))
    if extra.size:
        rgb[extra] = sh_radiance(cam, particles, sph, sph_degree, extra)
    return dataclasses.replace(pr, tiles_count=tiles_count, rgb=rgb)


FISHEYE_K = (0.04, -0.012, 0.003, -0.0006)    # the k1..k4 of test_scene_cameras_gpu.FISHEYE_FULL
OPENCV_K = (-0.08, 0.015, 0.0012, -0.0009)    # the k1, k2, p1, p2 of test_scene_cameras_gpu.OPENCV_FULL


def ftheta_sensor(width, height, reference_poly):
    """An f-theta sensor whose polynomials use all six coefficients, so that every order of both shows in the projection.  The forward
    polynomial is only roughly the backward one's inverse; its last coefficient moves a particle by a pixel at the edge of the frame."""
    f = 0.9 * width
    return dict(reference_poly=reference_poly, bw=[0.0, 1.0 / f, 0.0, 0.04 / f ** 3, 0.0, 0.01 / f ** 5],
                fw=[0.0, f, 0.0, -0.04 * f, 0.0, 0.02 * f], cde=[1.0, 0.001, -0.002], max_angle=1.0,
                principal=(width / 2.0 - 0.5, height / 2.0 - 0.5))


def colmap_sensor(name, width, height, fx):
    """(COLMAP camera model, its parameters) of the "opencv" (distorted pinhole of focal length fx) or "fisheye" sensor of a
    width x height frame, principal points off centre."""
    if name == "opencv":
        return "OPENCV", [fx, fx, width / 2 + 0.4, height / 2 - 0.4, *OPENCV_K]
    return "OPENCV_FISHEYE", [0.47 * width, 0.48 * width, width / 2 - 0.8, height / 2 + 0.8, *FISHEYE_K]


SENSORS = ("opencv", "fisheye", "ftheta_bw", "ftheta_fw", "rs1", "rs2", "rs3", "rs4", "rs1_fisheye")


def sensor_frame(name, width=128, height=128):
    """(scene, oracle camera, rays_o, rays_d) of the C1 scene seen through the sensor `name` of SENSORS:
      opencv       OpenCV pinhole with k1, k2, p1, p2 (COLMAP's OPENCV model), rays from the dataset's Newton inversion;
      fisheye      OpenCV fisheye (OPENCV_FISHEYE) of about 1.5 rad half-angle, from an orbit close enough to the scene that particles
                   reach beyond 1 rad off axis, where the high-order terms move them by a fraction of a pixel;
      ftheta_bw/fw f-theta with the backward / forward polynomial as the reference (ftheta_sensor);
      rs1..rs4     pinhole with a rolling shutter read out top to bottom, left to right, bottom to top, right to left, the sensor moving
                   between two orbit cameras during the exposure;
      rs1_fisheye  the fisheye above with the top-to-bottom rolling shutter."""
    import scene_data

    sc = scenes.scene_c1(width=width, height=height)
    fisheye = name in ("fisheye", "rs1_fisheye")
    if fisheye:
        sc = dataclasses.replace(sc, camera_radius=2.5)
    rolling = int(name[2]) if name.startswith("rs") else 0
    if rolling:
        p0, p1 = scenes.pose7_from_c2w(sc.camera(1, 40)), scenes.pose7_from_c2w(sc.camera(2, 40))
    else:
        p0 = p1 = scenes.pose7_from_c2w(sc.camera(5 if name == "opencv" else 1, 10))
    if name.startswith("ftheta"):
        ft = ftheta_sensor(width, height, 0 if name == "ftheta_bw" else 1)
        cam = go.make_camera(width, height, 1.0, 1.0, 0.0, 0.0, p0, p1, ftheta=ft)
        ro, rd = scenes.ftheta_rays(height, width, ft)
        return dataclasses.replace(sc, fx=1.0, fy=1.0, ftheta=ft), cam, ro, rd
    if fisheye or name == "opencv":
        sensor = scene_data.colmap_camera(*colmap_sensor("fisheye" if fisheye else "opencv", width, height, sc.fx), width, height, 1)
    else:
        sensor = scene_data.colmap_camera("PINHOLE", [sc.fx, sc.fy, sc.cx, sc.cy], width, height, 1)
    p = sensor.params
    cam = go.make_camera(width, height, p["fx"], p["fy"], p["cx"], p["cy"], p0, p1, rolling_shutter=rolling,
                         fisheye=(*p["radial"][:4], p["max_angle"]) if fisheye else None)
    if name == "opencv":
        cam.radial[:] = [float(v) for v in p["radial"]]
        cam.tangential[:] = [float(v) for v in p["tangential"]]
    ro, rd = sensor.host_rays()
    return sc, cam, ro, rd


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


def shuffled_pixels(height, width, seed=0):
    """A fixed seeded permutation of the pixels of a height x width frame.  3DGRT traces each 8x4 block of consecutive rays as one warp
    and walks the tree as a packet only when the warp's rays are coherent: rays put in this order come from all over the frame, so every
    warp fails that vote and takes the per-lane walk, where the camera's own order takes the packet walk."""
    return np.random.default_rng(seed).permutation(height * width)


def permute_pixels(a, perm):
    """`a` ([H, W, ...], [1, H, W, ...] or [H * W, ...]) with its pixels in the order `perm`: pixel j of the result is pixel perm[j]."""
    a = np.asarray(a)
    return np.ascontiguousarray(a.reshape(len(perm), -1)[perm].reshape(a.shape))


def unpermute_pixels(a, perm):
    """The inverse of permute_pixels: the outputs of rays traced in the order `perm`, back in the camera's order."""
    a = np.asarray(a)
    out = np.empty_like(a).reshape(len(perm), -1)
    out[perm] = a.reshape(len(perm), -1)
    return out.reshape(a.shape)


def packet_share(particles, sph, c2w, ro, rd, **config):
    """Share of the rays (ro, rd: [1, H, W, 3]) that one 3DGRT forward walks as a packet, from grtb200_debug_trace_counters; `config`
    sets fields of grtb200_config."""
    import b200_native as nat
    import torch

    cfg = nat.grt_default_config()
    for k, v in config.items():
        setattr(cfg, k, v)
    ctx = nat.GrtContext(cfg, 0)
    s = torch.cuda.current_stream().cuda_stream
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()  # noqa: E731
    p, f, tro, trd = t(particles), t(sph), t(ro), t(rd)
    n = int(p.shape[0])
    ctx.build_bvh_packed(s, n, p.data_ptr())
    vis = torch.zeros(n, device="cuda")
    r2w = np.ascontiguousarray(np.asarray(c2w, np.float32)[:3, :4])
    b, h, w = ro.shape[:3]
    c = ctx.trace_counters(s, n, p.data_ptr(), f.data_ptr(), 3, 1e-3, b, h, w, tro.data_ptr(), trd.data_ptr(), r2w.ctypes.data, vis.data_ptr())
    ctx.close()
    print(f"[walk] trace counters {c}: packet-walked rays {100 * c['packet_rays'] / c['rays']:.1f} %")
    return c["packet_rays"] / c["rays"]

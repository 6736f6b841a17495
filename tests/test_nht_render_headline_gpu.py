"""The 3DGUT NHT renderer (gutb200_forward_nht / gutb200_backward_nht) on whole headline-scale frames against the float64 NHT oracle
(tests/nht_render_oracle.py) on sampled tiles: the 16 heaviest tiles, the last tile row and column where the frame is ragged, and 32
seeded tiles with at least one list entry (frames of at most 256 tiles are compared whole).  The output gradients are exactly zero on every other pixel, so the kernel's backward is the
backward of the sampled pixels alone (pinned on the CPU by test_tile_subset_backward_is_the_masked_full_frame_backward).

Frames: C2 (300k, 800x800) at the colmap_3dgut_mcmc_nht render settings (ut_alpha 0.1, fp16 features, max_alpha 0.99, degree 2) with
every 7th density at 3.0 so that many pairs reach the clamp, two backwards on one forward (d_dist = 0 as training passes it, and a random
d_dist); the C3-like frame (400k, 1237x822: ragged tiles, particles behind the camera) with fp32 features at degree 4; on the 60k dense
256x256 scene, a fisheye camera, a distorted pinhole with a rolling shutter, and per-pixel jittered ray origins (the GENERAL path of both
kernels).

Bars: tile counts, sorted keys / values and tile ranges bit-exact with the C oracle where the projection calls no atan2f / acosf (else
>= 99.9 % of the tile counts equal, and a sampled tile whose list differs is left out); the DESIGN.md section 5 image bar on the
compared pixels; hit counts equal on >= 99.9 % of them; gradients per tensor err <= max(1e-3, 1.5 x yardstick) with the yardstick the
oracle in float32 against float64 on the same lists, and <= 1e-3 flat without the ten particles of the largest yardstick error."""
import dataclasses
import math
import time

import numpy as np
import pytest

import scenes
from helpers import dist_grad_blocks, dist_grad_mask, image_error_report, rel_l2, tracer_pose
from oracle import gut_oracle as go

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import nht_render_oracle as nro  # noqa: E402

SHIPPED = {"particle_kernel_max_alpha": 0.99, "splat": {"ut_alpha": 0.1}}  # configs/apps/colmap_3dgut_mcmc_nht.yaml's render settings
COLS = dict(pos=slice(0, 3), dns=slice(3, 4), quat=slice(4, 8), scl=slice(8, 11))


def _configs(render, degree):
    """(native config as threedgut_tracer builds it from `render`, the oracle's config with the same fields)"""
    from threedgut_tracer.tracer import _native_config

    nat_cfg = _native_config({"render": dict(render, particle_kernel_degree=degree)})
    cfg = go.default_config()
    for name, _ in go.Config._fields_:
        setattr(cfg, name, getattr(nat_cfg, name))
    return nat_cfg, cfg


def _dense(model=None):
    base = scenes.scene_c2(n=60_000, width=256, height=256)
    if model == "fisheye":
        f = 0.9 * base.width
        return dataclasses.replace(base, fx=f, fy=f, fisheye=(0.05, -0.01, 0.002, -0.0003, 0.6))
    return base


def _sample_tiles(ranges, width, height, seed):
    lens = ranges[:, 1].astype(np.int64) - ranges[:, 0]
    gx, gy = (width + 15) // 16, (height + 15) // 16
    chosen = set(np.argsort(-lens, kind="stable")[:16].tolist())
    if width % 16:
        chosen |= {ty * gx + gx - 1 for ty in range(gy)}
    if height % 16:
        chosen |= {(gy - 1) * gx + tx for tx in range(gx)}
    rest = np.setdiff1d(np.nonzero(lens > 0)[0], np.fromiter(chosen, np.int64))
    chosen |= set(np.random.default_rng(seed).choice(rest, min(32, len(rest)), replace=False).tolist())
    return np.array(sorted(chosen))


def _run_case(label, sc, cam, render, degree, half, d_dist_modes, ro=None, rd=None, exact=True, seed=0, min_clamped=0):
    import b200_native as nat

    t0 = time.time()
    nat_cfg, cfg = _configs(render, degree)
    if ro is None:
        ro, rd = sc.rays()
    ro, rd = np.ascontiguousarray(ro, np.float32).reshape(-1, 3), np.ascontiguousarray(rd, np.float32).reshape(-1, 3)
    n, H, W = sc.n, sc.height, sc.width
    feats = np.random.default_rng(seed).uniform(-math.pi / 2, math.pi / 2, (n, 48)).astype(np.float32)
    if half:
        feats = feats.astype(np.float16).astype(np.float32)  # what the kernel reads
    pr = go.project(cfg, cam, sc.particles, np.zeros((n, 48), np.float32), 0)
    bn = go.bin_tiles(cfg, cam, pr)

    # the kernels, whole frame
    ctx = nat.Context(nat_cfg, 0)
    ncam = nat.Camera.from_buffer_copy(bytes(cam))
    stream = torch.cuda.current_stream().cuda_stream
    dev = torch.device("cuda", 0)
    p_d, ro_d, rd_d = (torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (sc.particles, ro, rd))
    f_d = torch.from_numpy(feats).to(dev).to(torch.float16 if half else torch.float32).contiguous()
    out, dist, hits = torch.zeros((H, W, 25), device=dev), torch.zeros((H, W, 1), device=dev), torch.zeros((H, W, 1), device=dev)
    vis = torch.zeros((n, 1), device=dev)
    ctx.forward_nht(stream, ncam, n, p_d.data_ptr(), f_d.data_ptr(), 48, int(half), ro_d.data_ptr(), rd_d.data_ptr(), out.data_ptr(),
                    dist.data_ptr(), hits.data_ptr(), vis.data_ptr())
    torch.cuda.synchronize()
    count = ctx.debug_copy(nat.DBG_TILES_COUNT)
    same = count == pr.tiles_count
    print(f"[nht-headline] {label}: N={n} I={len(bn.sorted_values)}, tile counts equal on {same.mean() * 100:.4f} % of the particles")
    # a frame of at most 256 tiles (the dense 256x256 scene) is compared whole: the image bar then counts the same pixels as the SH tests'
    tiles = _sample_tiles(bn.ranges, W, H, seed) if len(bn.ranges) > 256 else np.arange(len(bn.ranges))
    if exact:
        assert same.all()
        assert np.array_equal(ctx.debug_copy(nat.DBG_SORTED_KEYS), bn.sorted_keys)
        assert np.array_equal(ctx.debug_copy(nat.DBG_SORTED_VALUES), bn.sorted_values)
        assert np.array_equal(ctx.debug_copy(nat.DBG_TILE_RANGES), bn.ranges)
    else:
        assert same.mean() >= 0.999
        g_ranges, g_vals = ctx.debug_copy(nat.DBG_TILE_RANGES), ctx.debug_copy(nat.DBG_SORTED_VALUES)
        keep = [t for t in tiles if np.array_equal(g_vals[g_ranges[t, 0]:g_ranges[t, 1]], bn.sorted_values[bn.ranges[t, 0]:bn.ranges[t, 1]])]
        print(f"[nht-headline] {label}: {len(tiles) - len(keep)} of {len(tiles)} sampled tiles left out (their list differs)")
        assert len(keep) >= len(tiles) - 4
        tiles = np.array(keep)
    mask = np.zeros(H * W, bool)
    for t in tiles:
        mask[nro.tile_pixels(int(t), W, H)] = True
    mask = mask.reshape(H, W)
    lens = bn.ranges[:, 1].astype(np.int64) - bn.ranges[:, 0]
    longest = int(lens[tiles].max())
    print(f"[nht-headline] {label}: {len(tiles)} tiles, {int(mask.sum())} compared pixels, longest sampled list {longest} "
          f"({int(np.ceil(longest / 128))} batches of 128 entries; longest of the frame {int(lens.max())})")

    # outputs on the compared pixels
    rng = np.random.default_rng(seed + 1)
    d_out = (rng.normal(size=(H, W, 25)) * mask[..., None]).astype(np.float32)
    d_dist_rand = (0.1 * rng.normal(size=(H, W, 1)) * mask[..., None]).astype(np.float32)
    kw = dict(pr=pr, bn=bn, device="cuda", tiles=tiles)
    got = dict(out=out.cpu().numpy(), dist=dist.cpu().numpy(), hits=hits.cpu().numpy())
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base_mem, t1 = torch.cuda.memory_allocated(), time.time()
    ref = nro.frame(cfg, cam, sc.particles, feats, ro, rd, go, **kw)
    print(f"[nht-headline] {label}: oracle forward on the sampled tiles {time.time() - t1:.1f} s")
    print(f"[nht-headline] {label}: oracle composites up to {ref['longest']} pairs per pixel, {ref['clamped']} clamped at max_alpha "
          f"{cfg.max_alpha:g}")
    assert ref["clamped"] >= min_clamped
    P = int(mask.sum())
    mean, mx, bad = image_error_report(f"{label} features+alpha", got["out"][mask][:, None], ref["out"][mask][:, None])
    assert mean <= 1e-5 and mx <= 2e-2 and bad <= max(3, int(2e-4 * P)), (mean, mx, bad)
    dscale = max(1.0, float(np.abs(ref["dist"][mask]).max()))
    mean, mx, bad = image_error_report(f"{label} dist", got["dist"][mask][:, None], ref["dist"][mask][:, None], atol=1e-4 * dscale)
    assert mean <= 1e-5 * dscale and bad <= max(3, int(2e-4 * P)), (mean, mx, bad)
    same_hits = float(np.mean(got["hits"][mask] == ref["hits"][mask]))
    print(f"[nht-headline] {label}: hit counts equal on {same_hits * 100:.4f} % of the compared pixels")
    assert same_hits >= 0.999

    # backwards on the one forward
    for mode in d_dist_modes:
        d_dist = d_dist_rand * dist_grad_mask(H, W, mode, seed)[..., None]
        with_d, without_d = dist_grad_blocks(np.where(mask[..., None], d_dist, 0.0))
        t1 = time.time()
        r64 = nro.frame(cfg, cam, sc.particles, feats, ro, rd, go, d_out=d_out, d_dist=d_dist, **kw)
        t2 = time.time()
        r32 = nro.frame(cfg, cam, sc.particles, feats, ro, rd, go, d_out=d_out, d_dist=d_dist, dtype=torch.float32, **kw)
        print(f"[nht-headline] {label} d_dist={mode}: oracle forward + backward f64 {t2 - t1:.1f} s, f32 {time.time() - t2:.1f} s, peak "
              f"device memory of the oracle {(torch.cuda.max_memory_allocated() - base_mem) / 2 ** 30:.2f} GiB")
        dd_o, dd_d = torch.from_numpy(d_out).to(dev), torch.from_numpy(d_dist).to(dev)
        dp, df = torch.zeros((n, 12), device=dev), torch.zeros((n, 48), device=dev)
        ctx.backward_nht(stream, ncam, n, p_d.data_ptr(), f_d.data_ptr(), 48, int(half), ro_d.data_ptr(), rd_d.data_ptr(), out.data_ptr(),
                         dd_o.data_ptr(), dist.data_ptr(), dd_d.data_ptr(), dp.data_ptr(), df.data_ptr())
        torch.cuda.synchronize()
        dp, df = dp.cpu().numpy(), df.cpu().numpy()
        errs = {k: rel_l2(dp[:, v], r64["dp"][:, v]) for k, v in COLS.items()}
        errs["features"] = rel_l2(df, r64["df"])
        yard = {k: rel_l2(r32["dp"][:, v], r64["dp"][:, v]) for k, v in COLS.items()}
        yard["features"] = rel_l2(r32["df"], r64["df"])
        e2 = ((r32["dp"] - r64["dp"]) ** 2).sum(1) / max(float((r64["dp"] ** 2).sum()), 1e-300) \
            + ((r32["df"] - r64["df"]) ** 2).sum(1) / max(float((r64["df"] ** 2).sum()), 1e-300)
        keep = np.ones(n, bool)
        keep[np.argsort(-e2)[:10]] = False
        robust = {k: rel_l2(dp[keep][:, v], r64["dp"][keep][:, v]) for k, v in COLS.items()}
        robust["features"] = rel_l2(df[keep], r64["df"][keep])
        fmt = lambda d: {k: f"{v:.2e}" for k, v in d.items()}  # noqa: E731
        tag = f"{label} d_dist={mode} (warp blocks with / without a distance gradient: {with_d} / {without_d})"
        print(f"[nht-headline] {tag} gradient rel-L2 vs oracle f64:", fmt(errs))
        print(f"[nht-headline] {tag} yardstick (oracle f32 vs f64, same lists):", fmt(yard))
        print(f"[nht-headline] {tag} without the oracle's 10 flip particles:", fmt(robust))
        assert np.abs(r64["df"]).max() > 0
        for k in errs:
            assert errs[k] <= max(1e-3, 1.5 * yard[k]), (mode, k, errs[k], yard[k])
            assert robust[k] <= 1e-3, (mode, k, robust[k])
        assert np.all(dp[:, 11] == 0)
    ctx.close()
    print(f"[nht-headline] {label}: {time.time() - t0:.1f} s")


def test_c2_at_the_shipped_nht_settings():
    """C2 camera 3 of 100 at colmap_3dgut_mcmc_nht's render settings, every 7th density at 3.0: clamped pairs and tile lists of thousands
    of entries; the backward as training runs it (d_dist = 0) and with a random distance gradient, on the same forward."""
    sc = scenes.scene_c2()
    particles = sc.particles.copy()
    particles[::7, 3] = 3.0
    sc = dataclasses.replace(sc, particles=particles)
    c2w = sc.camera(3, 100)
    cam, _ = _oracle_camera(sc, tracer_pose(c2w))
    _run_case("c2 cam3 shipped", sc, cam, SHIPPED, 2, True, ("zero", "random"), seed=3, min_clamped=1)


def test_c3_like_fp32_degree4():
    sc = scenes.scene_c3(n=400_000)
    c2w = sc.camera(1, 10)
    cam, _ = _oracle_camera(sc, tracer_pose(c2w))
    _run_case("c3_small cam1 fp32 deg4", sc, cam, {}, 4, False, ("zero", "mixed"), seed=11)


def test_fisheye_on_the_dense_scene():
    sc = _dense("fisheye")
    cam, _ = _oracle_camera(sc, tracer_pose(sc.camera(2, 10)))
    _run_case("dense fisheye", sc, cam, SHIPPED, 2, True, ("mixed",), exact=False, seed=2)


def test_distorted_pinhole_with_rolling_shutter_on_the_dense_scene():
    sc = _dense()
    p0, p1 = scenes.pose7_from_c2w(sc.camera(1, 40)), scenes.pose7_from_c2w(sc.camera(2, 40))
    cam = go.make_camera(sc.width, sc.height, sc.fx, sc.fy, sc.cx, sc.cy, p0, p1, rolling_shutter=1)
    cam.radial[:] = [0.05, -0.01, 0.002, 0.01, 0.0, 0.0]
    cam.tangential[:] = [0.001, -0.0005]
    cam.thin_prism[:] = [0.0003, 0.0, -0.0002, 0.0]
    _run_case("dense distorted pinhole + rolling shutter", sc, cam, {}, 4, False, ("zero",), exact=False, seed=5)


def test_jittered_origins_on_the_dense_scene():
    """Per-pixel ray origins: the GENERAL (non-uniform origin) path of both NHT kernels at lists of thousands of entries."""
    sc = _dense()
    cam, _ = _oracle_camera(sc, scenes.pose7_from_c2w(sc.camera(3, 10)))
    ro, rd = sc.rays()
    ro = ro + 0.01 * np.random.default_rng(4).normal(size=ro.shape).astype(np.float32)
    _run_case("dense jittered origins", sc, cam, SHIPPED, 2, True, ("zero", "mixed"), ro=ro, rd=rd, seed=6)


def _oracle_camera(sc, pose):
    from helpers import oracle_camera

    return oracle_camera(sc, None, pose)

"""GPU parity of the CUDA 3DGUT path against the CPU oracle OFF the default path: active SH degrees 0-2 (the first 3000 steps of every
training run raise the degree from 0), each render setting of gutb200_config away from its default, the backward's half-warp and
whole-warp sub-blocks (subtile_culling bits 4-5), and cloned particles (equal depth keys, as densification produces them).

Every case sets the same field on the oracle's config and on the native one.  Bars (DESIGN.md section 5, as test_gut_parity_gpu.py):
  * tile counts, depth bits, sorted keys and values, tile ranges and visibility: BIT-EXACT;
  * RGBA / distance: mean |diff| <= 1e-5, at most max(3, 2e-4 P) pixels off by more than 1e-4, max |diff| <= 2e-2;
  * hit counts equal on >= 99.9 % of the pixels;
  * gradients: rel-L2 <= 1e-3 for each of pos, density, quat, scale and sph.  On the dense scenes (tile lists of thousands of entries)
    the gradient bar is the yardstick rule of test_gut_headline_parity_gpu.py: err <= max(1e-3, 1.5 x (oracle f32 vs oracle f64 on the
    same lists)), and err <= 1e-3 flat once the oracle's ten largest f32-vs-f64 flip particles are left out.  Both are printed."""
import dataclasses
import os
import subprocess
import sys

import numpy as np
import pytest

import scenes
from helpers import image_error_report, oracle_camera, rel_l2, tracer_pose
from oracle import gut_oracle as go

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

COLS = dict(pos=slice(0, 3), dns=slice(3, 4), quat=slice(4, 8), scl=slice(8, 11))


def _dense():
    """>= 50k Gaussians on a 256x256 image: several hundred entries per tile."""
    return scenes.scene_c2(n=60_000, width=256, height=256)


def _c1_frame(which):
    """(scene, camera index, number of orbit cameras) of the named frame."""
    if which == "c1_cam0":
        return scenes.scene_c1(), 0, 10
    if which == "c1_cam7":
        return scenes.scene_c1(), 7, 10
    if which == "c1_ragged":  # partial tiles and partially filled warps
        return scenes.scene_c1(width=75, height=53), 5, 10
    if which == "dense":
        return _dense(), 2, 10
    raise ValueError(which)


def _set(cfg, settings):
    for k, v in settings.items():
        setattr(cfg, k, v)
    return cfg


def _oracle(sc, pose, settings, deg, seed, ro=None, rd=None, with_f64=False):
    """Oracle forward + backward with `settings` applied to go.default_config(), SH degree `deg`; optional per-pixel rays."""
    cfg = _set(go.default_config(), settings)
    cam = go.make_camera(sc.width, sc.height, sc.fx, sc.fy, sc.cx, sc.cy, pose)
    if ro is None:
        ro, rd = sc.rays()
    pr, bn, rgba, dist, hits = go.forward_all(cfg, cam, ro, rd, sc.particles, sc.sph, deg)
    rng = np.random.default_rng(seed)
    d_rgba = rng.normal(size=rgba.shape).astype(np.float32)
    d_dist = (0.1 * rng.normal(size=dist.shape)).astype(np.float32)
    dp, ds = go.render_backward(cfg, cam, ro, rd, sc.particles, sc.sph, deg, pr, bn, rgba, dist, d_rgba, d_dist)
    out = dict(ro=ro, rd=rd, pr=pr, bn=bn, rgba=rgba, dist=dist, hits=hits, d_rgba=d_rgba, d_dist=d_dist, dp=dp, ds=ds)
    if with_f64:
        r64, d64, _ = go.render_forward(cfg, cam, ro, rd, sc.particles, pr, bn, f64=True)
        out["dp_64"], out["ds_64"] = go.render_backward(cfg, cam, ro, rd, sc.particles, sc.sph, deg, pr, bn, r64, d64, d_rgba, d_dist, f64=True)
    return out


def _native_camera(sc, pose):
    import b200_native as nat

    cam = nat.Camera()
    cam.width, cam.height = sc.width, sc.height
    cam.principal[:] = [sc.cx, sc.cy]
    cam.focal[:] = [sc.fx, sc.fy]
    cam.pose_start[:] = [float(v) for v in pose]
    cam.pose_end[:] = [float(v) for v in pose]
    return cam


def _native(sc, pose, settings, deg, ro, rd, d_rgba, d_dist):
    """Forward + backward through the C ABI's host entry points with `settings` applied to nat.default_config()."""
    import b200_native as nat

    ctx = nat.Context(_set(nat.default_config(), settings), 0)
    cam = _native_camera(sc, pose)
    n, hw = sc.n, sc.width * sc.height
    rgba, dist, hits, vis = (np.zeros((hw, 4), np.float32), np.zeros(hw, np.float32), np.zeros(hw, np.float32), np.zeros(n, np.float32))
    p = lambda a: a.ctypes.data  # noqa: E731
    ro, rd = np.ascontiguousarray(ro, np.float32), np.ascontiguousarray(rd, np.float32)
    d_rgba, d_dist = np.ascontiguousarray(d_rgba, np.float32), np.ascontiguousarray(d_dist, np.float32)
    ctx.forward_host(cam, n, p(sc.particles), p(sc.sph), deg, p(ro), p(rd), p(rgba), p(dist), p(hits), p(vis))
    out = {k: ctx.debug_copy(v) for k, v in dict(count=nat.DBG_TILES_COUNT, keys=nat.DBG_SORTED_KEYS, vals=nat.DBG_SORTED_VALUES,
                                                 ranges=nat.DBG_TILE_RANGES, depth=nat.DBG_DEPTH, rgb=nat.DBG_RGB).items()}
    dp, ds = np.zeros((n, 12), np.float32), np.zeros((n, 48), np.float32)
    ctx.backward_host(cam, n, p(sc.particles), p(sc.sph), deg, p(ro), p(rd), p(rgba), p(d_rgba), p(dist), p(d_dist), p(dp), p(ds))
    ctx.close()
    out.update(rgba=rgba.reshape(sc.height, sc.width, 4), dist=dist.reshape(sc.height, sc.width, 1), hits=hits.reshape(sc.height, sc.width, 1),
               vis=vis, dp=dp, ds=ds)
    return out


def _list_stats(label, bn):
    lens = bn.ranges[:, 1].astype(np.int64) - bn.ranges[:, 0]
    print(f"[off-default] {label}: I={len(bn.sorted_keys)} longest tile list {int(lens.max())}")
    return lens


def _check_integers(label, got, ref):
    assert np.array_equal(got["count"], ref["pr"].tiles_count), f"{label}: tile counts"
    assert np.array_equal(got["depth"].view(np.uint32), ref["pr"].depth.view(np.uint32)), f"{label}: depth bits"
    assert np.array_equal(got["keys"], ref["bn"].sorted_keys), f"{label}: sorted keys"
    assert np.array_equal(got["vals"], ref["bn"].sorted_values), f"{label}: sorted values"
    assert np.array_equal(got["ranges"], ref["bn"].ranges), f"{label}: tile ranges"
    assert np.array_equal(got["vis"].view(np.int32) != 0, ref["pr"].visibility != 0), f"{label}: visibility"


def _check_image(label, rgba, dist, hits, ref):
    P = rgba.shape[0] * rgba.shape[1]
    mean_e, max_e, bad = image_error_report(f"{label} rgba", rgba, ref["rgba"])
    print(f"[off-default] {label} rgba bar: mean <= 1e-5, max <= 2e-2, pixels > 1e-4 <= {max(3, int(2e-4 * P))}")
    assert mean_e <= 1e-5 and max_e <= 2e-2 and bad <= max(3, int(2e-4 * P))
    dscale = max(1.0, float(np.abs(ref["dist"]).max()))
    mean_e, max_e, bad = image_error_report(f"{label} dist", dist, ref["dist"], atol=1e-4 * dscale)
    assert mean_e <= 1e-5 * dscale and bad <= max(3, int(2e-4 * P))
    same = float(np.mean(hits == ref["hits"]))
    print(f"[off-default] {label}: hit counts equal on {same * 100:.4f} % of the pixels (bar 99.9 %)")
    assert same >= 0.999


def _check_gradients(label, dp, ds, ref):
    """Flat 1e-3 per tensor; with the f64 yardstick in `ref` (dense scenes), the rule of test_gut_headline_parity_gpu.py."""
    errs = {k: rel_l2(dp[:, v], ref["dp"][:, v]) for k, v in COLS.items()}
    errs["sph"] = rel_l2(ds, ref["ds"])
    fmt = lambda d: {k: f"{v:.2e}" for k, v in d.items()}  # noqa: E731
    print(f"[off-default] {label} gradient rel-L2 vs oracle:", fmt(errs))
    if "dp_64" not in ref:
        print(f"[off-default] {label} gradient bar: 1e-3")
        assert max(errs.values()) <= 1e-3, errs
        return
    rdp, rdp64, rds, rds64 = ref["dp"], ref["dp_64"], ref["ds"], ref["ds_64"]
    yard = {k: rel_l2(rdp[:, v], rdp64[:, v]) for k, v in COLS.items()}
    yard["sph"] = rel_l2(rds, rds64)
    e2 = ((rdp.astype(np.float64) - rdp64) ** 2).sum(1) / max(float((rdp64 ** 2).sum()), 1e-300) \
        + ((rds.astype(np.float64) - rds64) ** 2).sum(1) / max(float((rds64 ** 2).sum()), 1e-300)
    keep = np.ones(len(dp), bool)
    keep[np.argsort(-e2)[:10]] = False
    robust = {k: rel_l2(dp[keep][:, v], rdp[keep][:, v]) for k, v in COLS.items()}
    robust["sph"] = rel_l2(ds[keep], rds[keep])
    print(f"[off-default] {label} yardstick (oracle f32 vs f64, same lists); bar max(1e-3, 1.5 x yardstick):", fmt(yard))
    print(f"[off-default] {label} without the oracle's 10 flip particles (bar 1e-3):", fmt(robust))
    for k in errs:
        assert errs[k] <= max(1e-3, 1.5 * yard[k]), (k, errs[k], yard[k])
        assert robust[k] <= 1e-3, (k, robust[k])


def _check_sh_zeros(label, ds, deg, visible):
    """The SH gradient of a coefficient the active degree does not use, and of a particle no tile sees, is exactly zero."""
    ds = ds.reshape(len(ds), 16, 3)
    used = (deg + 1) ** 2
    assert np.all(ds[:, used:, :] == 0), f"{label}: non-zero d_sph beyond the {used} active coefficients"
    assert np.all(ds[~visible] == 0), f"{label}: non-zero d_sph on an invisible particle"
    assert np.abs(ds[visible, :used, :]).max() > 0


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. active SH degree 0, 1, 2


class _Gaussians:
    def __init__(self, sc, deg, device):
        p = torch.from_numpy(sc.particles).to(device)
        self.positions = p[:, 0:3].clone().requires_grad_(True)
        self._dns = p[:, 3:4].clone().requires_grad_(True)
        self._rot = p[:, 4:8].clone().requires_grad_(True)
        self._scl = p[:, 8:11].clone().requires_grad_(True)
        self._sph = torch.from_numpy(sc.sph).to(device).requires_grad_(True)
        self.n_active_features = deg
        self.ray_feature_dim = 3
        self.num_gaussians = sc.n

    def get_rotation(self):
        return self._rot

    def get_scale(self):
        return self._scl

    def get_density(self):
        return self._dns

    def get_features(self):
        return self._sph


def _tracer_render(sc, c2w, deg, ref):
    """Tracer.render + autograd with the oracle's output gradients; returns (rgba, dist, hits, dp [N,12], ds [N,48])."""
    import threedgut_tracer
    from test_gut_parity_gpu import _Batch

    dev = torch.device("cuda", 0)
    tr = threedgut_tracer.Tracer({"render": {}})
    g = _Gaussians(sc, deg, dev)
    out = tr.render(g, _Batch(sc, c2w, dev), train=True)
    loss = (out["pred_features"] * torch.from_numpy(ref["d_rgba"][None, ..., :3]).to(dev)).sum() \
        + (out["pred_opacity"] * torch.from_numpy(ref["d_rgba"][None, ..., 3:]).to(dev)).sum() \
        + (out["pred_dist"] * torch.from_numpy(ref["d_dist"][None]).to(dev)).sum()
    loss.backward()
    torch.cuda.synchronize()
    rgba = torch.cat([out["pred_features"], out["pred_opacity"]], -1)[0].detach().cpu().numpy()
    dp = np.zeros((sc.n, 12), np.float32)
    dp[:, 0:3], dp[:, 3:4] = g.positions.grad.cpu().numpy(), g._dns.grad.cpu().numpy()
    dp[:, 4:8], dp[:, 8:11] = g._rot.grad.cpu().numpy(), g._scl.grad.cpu().numpy()
    return rgba, out["pred_dist"][0].detach().cpu().numpy(), out["hits_count"][0].detach().cpu().numpy(), dp, g._sph.grad.cpu().numpy()


@pytest.mark.parametrize("frame", ["c1_cam0", "dense"])
@pytest.mark.parametrize("deg", [0, 1, 2])
def test_sh_degree_parity(deg, frame):
    """n_active_features = deg < 3 through the C ABI and through Tracer.render: the projection's radiance (DBG_RGB), the image, the five
    gradients, and exact zeros in d_sph beyond (deg + 1)^2 coefficients and on invisible particles.  At degree 0 the radiance does not
    depend on the view direction, so d_pos carries no direction term; it is checked on its own as well."""
    sc, cam_index, n_cams = _c1_frame(frame)
    sc = dataclasses.replace(sc, sph_degree=deg)
    c2w = sc.camera(cam_index, n_cams)
    pose = tracer_pose(c2w)
    dense = frame == "dense"
    ref = _oracle(sc, pose, {}, deg, seed=10 + deg, with_f64=dense)
    if dense:
        assert _list_stats(f"{frame} sh{deg}", ref["bn"]).max() > 256
    visible = ref["pr"].tiles_count > 0
    label = f"{frame} sh{deg} c-abi"
    got = _native(sc, pose, {}, deg, ref["ro"], ref["rd"], ref["d_rgba"], ref["d_dist"])
    _check_integers(label, got, ref)
    rgb_err = float(np.abs(got["rgb"][visible] - ref["pr"].rgb[visible]).max())
    print(f"[off-default] {label}: projected radiance max |diff| {rgb_err:.2e} (bar 2e-6 + 1e-6 rel)")
    assert np.allclose(got["rgb"][visible], ref["pr"].rgb[visible], atol=2e-6, rtol=1e-6)
    _check_image(label, got["rgba"], got["dist"], got["hits"], ref)
    _check_gradients(label, got["dp"], got["ds"], ref)
    _check_sh_zeros(label, got["ds"], deg, visible)
    if deg == 0:
        e = rel_l2(got["dp"][:, 0:3], ref["dp"][:, 0:3])
        print(f"[off-default] {label}: d_pos rel-L2 {e:.2e} (no direction term at degree 0)")
        assert e <= 1e-3 or dense  # dense: covered by the yardstick rule above
    label = f"{frame} sh{deg} Tracer.render"
    rgba, dist, hits, dp, ds = _tracer_render(sc, c2w, deg, ref)
    _check_image(label, rgba, dist, hits, ref)
    _check_gradients(label, dp, ds, ref)
    _check_sh_zeros(label, ds, deg, visible)


@pytest.mark.parametrize("deg", [0, 1, 2])
def test_compact_exchange_at_sh_degree(deg):
    """gutb200_backward_compact + gutb200_sph_grad_from_views at an active degree below 3: the SH gradient rebuilt from two views'
    [N,4] radiance gradients equals the sum of the two views' full d_sph rows, zeros beyond (deg + 1)^2 included."""
    import threedgut_tracer
    from threedgut_tracer.tracer import ShutterType, fromOpenCVPinholeCameraModelParameters

    dev = torch.device("cuda", 0)
    sc = scenes.scene_c1()
    raster = threedgut_tracer.Tracer({"render": {}}).tracer_wrapper
    particles, sph = torch.from_numpy(sc.particles).to(dev), torch.from_numpy(sc.sph).to(dev)
    ro, rd = sc.rays()
    rays_o, rays_d = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)
    W, H = sc.width, sc.height
    sensor = fromOpenCVPinholeCameraModelParameters(np.array([W, H]), ShutterType.GLOBAL, np.array([sc.cx, sc.cy], np.float32),
                                                    np.array([sc.fx, sc.fy], np.float32), np.zeros(6, np.float32), np.zeros(2, np.float32),
                                                    np.zeros(4, np.float32))
    gen = torch.Generator(device=dev).manual_seed(deg)
    full_ds, gs, pos = [], [], []
    for view in (2, 7):
        pose = scenes.pose7_from_c2w(sc.camera(view, 10))
        d_rgba = torch.randn((H, W, 4), device=dev, generator=gen)
        d_dist = 0.05 * torch.randn((H, W, 1), device=dev, generator=gen)
        rgba, dst, hits, vis = raster.trace(0, deg, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose)
        dp, ds = raster.trace_bwd(0, deg, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose, rgba, d_rgba, dst, d_dist)
        full_ds.append(ds.clone())
        rgba, dst, hits, vis = raster.trace(0, deg, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose)
        dp2, g = raster.trace_bwd_compact(0, deg, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose, rgba, d_rgba, dst, d_dist)
        assert rel_l2(dp2.cpu().numpy(), dp.cpu().numpy()) <= 2e-5
        gs.append(g.clone())
        pos.append(raster.sensor_position(sensor, pose, pose, W, H))
    ds_sum = (full_ds[0] + full_ds[1]).cpu().numpy()
    rebuilt = raster.sph_grad_from_views(deg, particles, np.stack(pos), torch.stack(gs)).cpu().numpy()
    err = rel_l2(rebuilt, ds_sum)
    print(f"[off-default] compact exchange sh{deg}: rebuilt d_sph rel-L2 {err:.2e} (bar 2e-6)")
    assert np.abs(ds_sum).max() > 0
    assert err <= 2e-6
    assert np.abs(rebuilt - ds_sum).max() <= 1e-5 * max(1.0, float(np.abs(ds_sum).max()))
    used = (deg + 1) ** 2
    assert np.all(rebuilt.reshape(-1, 16, 3)[:, used:] == 0) and np.all(ds_sum.reshape(-1, 16, 3)[:, used:] == 0)


def test_kbuffer_at_sh_degree_1():
    """The sorted (k-buffer, K = 16) variant at active SH degree 1 against the oracle's k-buffer forward and backward."""
    import b200_native as nat

    deg, k = 1, 16
    sc = scenes.scene_c1()
    sc.particles[:, 8:11] *= 2.0  # overlapping Gaussians: the per-ray hit order differs from the depth order of the lists
    c2w = sc.camera(3, 10)
    pose = tracer_pose(c2w)
    cfg = go.default_config()
    cam, _ = oracle_camera(sc, c2w, pose)
    ro, rd = sc.rays()
    pr = go.project(cfg, cam, sc.particles, sc.sph, deg)
    bn = go.bin_tiles(cfg, cam, pr)
    rgba_ref, dist_ref, hits_ref = go.render_forward_kbuffer(cfg, cam, k, ro, rd, sc.particles, pr, bn)
    rng = np.random.default_rng(1)
    d_rgba = rng.normal(size=rgba_ref.shape).astype(np.float32)
    d_dist = (0.1 * rng.normal(size=dist_ref.shape)).astype(np.float32)
    dp_ref, ds_ref = go.render_backward_kbuffer(cfg, cam, k, ro, rd, sc.particles, sc.sph, deg, pr, bn, rgba_ref, dist_ref, d_rgba, d_dist)
    got = _native(sc, pose, dict(k_buffer_size=k), deg, ro, rd, d_rgba, d_dist)
    ref = dict(rgba=rgba_ref, dist=dist_ref, hits=hits_ref, dp=dp_ref, ds=ds_ref)
    _check_image("kbuffer K=16 sh1", got["rgba"], got["dist"], got["hits"], ref)
    _check_gradients("kbuffer K=16 sh1", got["dp"], got["ds"], ref)
    _check_sh_zeros("kbuffer K=16 sh1", got["ds"], deg, pr.tiles_count > 0)


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. render settings off their defaults, one at a time

SETTINGS = {
    "rect_bounding=0": dict(rect_bounding=0),
    "tight_opacity_bounding=0": dict(tight_opacity_bounding=0),
    "tile_culling=0": dict(tile_culling=0),
    "global_z_order=0": dict(global_z_order=0),
    # the UT weights follow ut_alpha (gutb200_config, as the oracle); the sigma-point spread ut_delta stays at its default on both
    # sides, so the projected footprints grow: the long-list case of tile_sort (~23 k entries in one tile of the dense scene)
    "ut_alpha=0.1": dict(ut_alpha=0.1),
    "min_transmittance=0.03": dict(min_transmittance=0.03),  # the reference's 3DGRT inference configs; the tile-wide early exit
    "max_alpha=0.999": dict(max_alpha=0.999),                # the reference's MCMC configs; see _opaque
    "kernel_degree=4": dict(kernel_degree=4),
}


def _opaque(sc):
    """Every fifth particle at density 1: the scenes' densities stay below 0.99, where max_alpha would never clamp anything."""
    particles = sc.particles.copy()
    particles[::5, 3] = 1.0
    return dataclasses.replace(sc, particles=particles)


@pytest.mark.parametrize("frame", ["c1_cam0", "c1_cam7", "c1_ragged", "dense"])
@pytest.mark.parametrize("setting", list(SETTINGS))
def test_render_setting_parity(setting, frame):
    sc, cam_index, n_cams = _c1_frame(frame)
    if setting.startswith("max_alpha"):
        sc = _opaque(sc)
    pose = tracer_pose(sc.camera(cam_index, n_cams))
    settings = SETTINGS[setting]
    dense = frame == "dense"
    ref = _oracle(sc, pose, settings, 3, seed=cam_index, with_f64=dense)
    label = f"{setting} {frame}"
    lens = _list_stats(label, ref["bn"])
    if dense:
        assert lens.max() > 256
    # the setting changes what the oracle computes on this frame (else the case would test nothing new)
    base = _oracle(sc, pose, {}, 3, seed=cam_index)
    assert not (np.array_equal(base["bn"].sorted_values, ref["bn"].sorted_values) and np.array_equal(base["rgba"], ref["rgba"])
                and np.array_equal(base["dp"], ref["dp"])), f"{setting} does not change the oracle's output on {frame}"
    got = _native(sc, pose, settings, 3, ref["ro"], ref["rd"], ref["d_rgba"], ref["d_dist"])
    _check_integers(label, got, ref)
    _check_image(label, got["rgba"], got["dist"], got["hits"], ref)
    _check_gradients(label, got["dp"], got["ds"], ref)


# ---------------------------------------------------------------------------------------------------------------------------------
# 3. the backward's sub-block widths (subtile_culling bits 4-5: 16 = half-warps, 32 = whole warps)


def _banded_rays(sc):
    """The three bands of test_per_pixel_ray_origins_take_the_general_path: the frame's origin (backward FAST), another origin common to
    the tile (backward GENERAL with the origin-offset terms), per-pixel jitter."""
    ro, rd = sc.rays()
    rng = np.random.default_rng(3)
    ro = (ro + 0.02 * rng.normal(size=ro.shape)).astype(np.float32)
    ro[:, :32] = ro[0, 0, 0]
    ro[:, 32:64] = ro[0, 0, 0] + np.array([0.03, -0.02, 0.05], np.float32)
    return ro, rd


@pytest.mark.parametrize("frame", ["c1_cam0", "dense", "bands"])
@pytest.mark.parametrize("kernel_degree", [2, 4])
@pytest.mark.parametrize("mode", [23, 39])
def test_backward_sub_block_widths(mode, kernel_degree, frame):
    """subtile_culling 23 (half-warp sub-blocks) and 39 (whole-warp sub-blocks) against the oracle; the forward does not depend on the
    backward's sub-block and must be bit-identical to the default mode 7."""
    if frame == "bands":
        sc, cam_index, n_cams = scenes.scene_c1(), 4, 10
        ro, rd = _banded_rays(sc)
    else:
        sc, cam_index, n_cams = _c1_frame(frame)
        ro = rd = None
    pose = tracer_pose(sc.camera(cam_index, n_cams))
    dense = frame == "dense"
    ref = _oracle(sc, pose, dict(kernel_degree=kernel_degree), 3, seed=mode + kernel_degree, ro=ro, rd=rd, with_f64=dense)
    label = f"subtile_culling={mode} kernel_degree={kernel_degree} {frame}"
    _list_stats(label, ref["bn"])
    got = _native(sc, pose, dict(kernel_degree=kernel_degree, subtile_culling=mode), 3, ref["ro"], ref["rd"], ref["d_rgba"], ref["d_dist"])
    base = _native(sc, pose, dict(kernel_degree=kernel_degree, subtile_culling=7), 3, ref["ro"], ref["rd"], ref["d_rgba"], ref["d_dist"])
    for k in ("rgba", "dist", "hits"):
        assert np.array_equal(got[k].view(np.uint32), base[k].view(np.uint32)), f"{label}: forward {k} differs from mode 7"
    _check_integers(label, got, ref)
    _check_image(label, got["rgba"], got["dist"], got["hits"], ref)
    _check_gradients(label, got["dp"], got["ds"], ref)
    e = max(rel_l2(got["dp"], base["dp"]), rel_l2(got["ds"], base["ds"]))
    # the sub-block decides which list entries the backward walks (those some pixel of the sub-block accepted in the forward); the
    # backward re-tests every pair it walks, so only a borderline pair accepted by one arithmetic and not the other can differ, plus the
    # order of the atomic sums -- the bar of test_subtile_culling_is_bit_identical for hit words on / off
    print(f"[off-default] {label}: gradients vs mode 7 rel-L2 {e:.2e} (bar 3e-4)")
    assert e <= 3e-4


# ---------------------------------------------------------------------------------------------------------------------------------
# 4. cloned particles: equal depth keys


def clone_scene(base, singles, doubles, forties, seed=0):
    """`base` plus copies of some of its particles: `singles` particles copied once, `doubles` twice, `forties` 40 times, every copy
    shuffled to a scattered index (densification's clones share the position, hence the depth, of their source).  Returns the scene and
    for each particle the index of its source in `base` (its clone group)."""
    rng = np.random.default_rng(seed)
    src = rng.choice(base.n, singles + doubles + forties, replace=False)
    reps = np.concatenate([np.full(singles, 1), np.full(doubles, 2), np.full(forties, 40)])
    group = np.concatenate([np.arange(base.n), np.repeat(src, reps)])[rng.permutation(base.n + int(reps.sum()))]
    sc = dataclasses.replace(base, particles=np.ascontiguousarray(base.particles[group]), sph=np.ascontiguousarray(base.sph[group]))
    return sc, group


def _equal_depth_runs(keys):
    """(number of runs of >= 2 equal (tile, depth) keys, longest run, runs of >= 32)"""
    if len(keys) < 2:
        return 0, 1, 0
    edges = np.flatnonzero(np.diff(keys) != 0)
    lens = np.diff(np.concatenate([[-1], edges, [len(keys) - 1]]))
    return int((lens >= 2).sum()), int(lens.max()), int((lens >= 32).sum())


def check_cloned_particles_3dgut():
    """The clone comparison on its own (also run in a child process with GUTB200_SORT_MATCH=1)."""
    base = scenes.scene_c2(n=50_000, width=256, height=256)
    sc, _ = clone_scene(base, 6000, 300, 8)
    c2w = sc.camera(2, 10)
    pose = tracer_pose(c2w)
    ref = _oracle(sc, pose, {}, 3, seed=5, with_f64=True)
    runs, longest, long_runs = _equal_depth_runs(ref["bn"].sorted_keys)
    lens = _list_stats(f"clones N={sc.n}", ref["bn"])
    print(f"[off-default] clones: {runs} equal-depth runs in the sorted stream, longest {longest}, {long_runs} of >= 32 entries")
    assert runs > 1000 and longest >= 32 and lens.max() > 256
    got = _native(sc, pose, {}, 3, ref["ro"], ref["rd"], ref["d_rgba"], ref["d_dist"])
    _check_integers("clones", got, ref)
    _check_image("clones", got["rgba"], got["dist"], got["hits"], ref)
    _check_gradients("clones", got["dp"], got["ds"], ref)


def test_cloned_particles_3dgut():
    """Clones of the dense scene's 50k particles: 6000 singles, 300 doubles and 8 particles copied 40 times.  Their depth bits are equal,
    so tile_sort orders each run by particle index in its fix-up pass (the atomic slot claims arrive in any order): sorted keys, values
    and ranges bit-exact, and -- (depth, index) being a total order -- the image and the per-particle gradients within the bars."""
    check_cloned_particles_3dgut()


def test_cloned_particles_3dgut_match_any_sort():
    """The same comparison with the match.any variant of tile_sort (GUTB200_SORT_MATCH=1, read once per process): in a child process,
    which must run to completion and exit."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, GUTB200_SORT_MATCH="1")
    env["PYTHONPATH"] = os.pathsep.join([root, os.path.join(root, "3dgrut_b200"), os.path.join(root, "tests")]
                                        + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    flags = ["-s"] if sys.flags.no_user_site else []
    code = "import test_gut_off_default_gpu as t; t.check_cloned_particles_3dgut(); print('[off-default] match-any sort: done')"
    r = subprocess.run([sys.executable, *flags, "-c", code], env=env, cwd=root, capture_output=True, text=True, timeout=900)
    print(r.stdout)
    print(r.stderr[-4000:])
    assert r.returncode == 0
    assert "match-any sort: done" in r.stdout


# ---------------------------------------------------------------------------------------------------------------------------------
# 5. argument checks


def test_out_of_range_arguments_are_rejected():
    """sph_degree outside 0..3 (it used to be clamped silently) and subtile_culling sub-block code 3 (it used to fall back to
    quarter-warps) fail with a message on forward, backward and backward_compact."""
    import b200_native as nat

    sc = scenes.scene_c1(n=64, width=32, height=32)
    pose = tracer_pose(sc.camera(1, 10))
    cam = _native_camera(sc, pose)
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    ro, rd = sc.rays()
    particles, sph, tro, trd = t(sc.particles), t(sc.sph), t(ro), t(rd)
    hw, n = sc.width * sc.height, sc.n
    rgba, dist, hits, vis = (torch.zeros((hw, 4), device=dev), torch.zeros(hw, device=dev), torch.zeros(hw, device=dev),
                             torch.zeros(n, device=dev))
    dp, ds = torch.zeros((n, 12), device=dev), torch.zeros((n, 48), device=dev)
    s = torch.cuda.current_stream(dev).cuda_stream

    def fwd(ctx, deg):
        ctx.forward(s, cam, n, particles.data_ptr(), sph.data_ptr(), deg, tro.data_ptr(), trd.data_ptr(), rgba.data_ptr(), dist.data_ptr(),
                    hits.data_ptr(), vis.data_ptr())

    def bwd(ctx, deg, compact=False):
        f = ctx.backward_compact if compact else ctx.backward
        f(s, cam, n, particles.data_ptr(), sph.data_ptr(), deg, tro.data_ptr(), trd.data_ptr(), rgba.data_ptr(), rgba.data_ptr(),
          dist.data_ptr(), dist.data_ptr(), dp.data_ptr(), ds.data_ptr())

    ctx = nat.Context(nat.default_config(), 0)
    for deg in (-1, 4):
        with pytest.raises(RuntimeError, match=f"sph_degree {deg} out of range"):
            fwd(ctx, deg)
    fwd(ctx, 3)
    for deg in (-1, 4):
        with pytest.raises(RuntimeError, match=f"sph_degree {deg} out of range"):
            bwd(ctx, deg)
        with pytest.raises(RuntimeError, match=f"sph_degree {deg} out of range"):
            bwd(ctx, deg, compact=True)
    bwd(ctx, 3)
    ctx.close()
    cfg = nat.default_config()
    cfg.subtile_culling = 7 | (3 << 4)
    bad = nat.Context(cfg, 0)
    with pytest.raises(RuntimeError, match="sub-block code 3"):
        fwd(bad, 3)
    bad.close()
    torch.cuda.synchronize()

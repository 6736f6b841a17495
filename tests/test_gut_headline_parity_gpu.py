"""Oracle parity of the CUDA 3DGUT path AT THE HEADLINE SCALES (BASELINE configs[1] = C2: 800x800, 300k Gaussians; a C3-like unbounded scene
with 400k Gaussians at 1237x822; one >= 50k-Gaussian case per camera model), through the C ABI's host entry points
(gutb200_forward_host / gutb200_backward_host).  The C1-scale tests (test_gut_parity_gpu.py) have ~30 list entries per tile; here the tile
lists run to thousands of entries, so the multi-batch loop of the render kernels (256 entries per staged batch), the tile-wide early exit,
heaviest-tile-first ordering and sub-tile culling are all compared with the oracle, not with themselves.

Bars (same policy as test_gut_parity_gpu.py / DESIGN.md section 5): tile counts, depth bits, the sorted (key, value) stream and tile ranges
BIT-EXACT; RGBA / distance: mean |diff| <= 1e-5, |diff| <= 1e-4 on all but max(3, 2e-4 P) pixels, max <= 2e-2; hit counts equal on
>= 99.9 % of the pixels; the five gradient tensors rel-L2 <= 1e-3 each -- see below.  The full-frame oracle costs ~5 s per view on the box.

Gradient bar, as first run and as it stands: with a flat 1e-3 on every tensor, 1 of the 2 C2
cameras FAILED -- cam41, d_quat rel-L2 2.22e-3 (the other four tensors 1.3e-4 .. 6.5e-4; cam3: all <= 4.5e-4).  The same frame evaluated by the
oracle in fp32 and in fp64 ON THE SAME LISTS (no CUDA involved) differs by 2.24e-3 in d_quat, 93.6 % of the squared error in ONE anisotropic
particle (scale ratio 18), 99.2 % in ten: a borderline accept flip (response > 0.0113 / alpha > 1/255 are discontinuous) on an elongated
Gaussian, whose rotation gradient is large, dominates the norm.  A flat 1e-3 is below the fp32 noise floor of that frame for that tensor.
Both cameras stay in the test.  The check is therefore, per tensor:  (1) err <= max(1e-3, 1.5 x yardstick), yardstick = oracle f32 vs
oracle f64 of THIS frame, printed;  (2) with the ten particles that carry the largest yardstick error removed -- picked from the oracle
pair, never from our output -- err <= 1e-3 flat.  (2) cannot be met by a systematic error; (1) keeps 1e-3 wherever the frame allows it."""
import dataclasses

import numpy as np
import pytest

import scenes
from helpers import dist_grad_blocks, image_error_report, oracle_frame, rel_l2, tracer_pose

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _native_camera(sc, pose):
    import b200_native as nat

    cam = nat.Camera()
    cam.width, cam.height = sc.width, sc.height
    cam.principal[:] = [sc.cx, sc.cy]
    cam.focal[:] = [sc.fx, sc.fy]
    cam.pose_start[:] = [float(v) for v in pose]
    cam.pose_end[:] = [float(v) for v in pose]
    return cam


def _check_frame(label, sc, cam_index, n_cams, seed, d_dist="random", d_alpha="random"):
    """d_dist / d_alpha: the output gradients of the backward (helpers.output_grads); "zero" d_dist is what every training step passes."""
    import b200_native as nat

    c2w = sc.camera(cam_index, n_cams)
    pose = tracer_pose(c2w)
    ref = oracle_frame(sc, c2w, seed=seed, pose=pose, with_f64=True, d_dist=d_dist, d_alpha=d_alpha)
    lens = ref["bn"].ranges[:, 1].astype(np.int64) - ref["bn"].ranges[:, 0]
    if d_dist != "random" or d_alpha != "random":
        label = f"{label} d_dist={d_dist} d_alpha={d_alpha}"
    print(f"[headline] {label} cam{cam_index}: N={sc.n} I={len(ref['bn'].sorted_keys)} longest tile list {int(lens.max())} "
          f"(batches of 256: {int(np.ceil(lens.max() / 256))}), hits {int(ref['hits'].sum())}, warp blocks with / without a distance "
          f"gradient {dist_grad_blocks(ref['d_dist'])}")
    assert lens.max() > 512, "the case is meant to exercise several staged batches per tile"

    ctx = nat.Context(nat.default_config(), 0)
    cam = _native_camera(sc, pose)
    n, hw = sc.n, sc.width * sc.height
    rgba, dist, hits, vis = (np.zeros((hw, 4), np.float32), np.zeros(hw, np.float32), np.zeros(hw, np.float32), np.zeros(n, np.float32))
    p = lambda a: a.ctypes.data  # noqa: E731
    ro, rd = np.ascontiguousarray(ref["ro"]), np.ascontiguousarray(ref["rd"])
    ctx.forward_host(cam, n, p(sc.particles), p(sc.sph), sc.sph_degree, p(ro), p(rd), p(rgba), p(dist), p(hits), p(vis))
    # integer artefacts: bit-exact
    assert np.array_equal(ctx.debug_copy(nat.DBG_TILES_COUNT), ref["pr"].tiles_count)
    assert np.array_equal(ctx.debug_copy(nat.DBG_DEPTH).view(np.uint32), ref["pr"].depth.view(np.uint32))
    assert np.array_equal(ctx.debug_copy(nat.DBG_SORTED_KEYS), ref["bn"].sorted_keys)
    assert np.array_equal(ctx.debug_copy(nat.DBG_SORTED_VALUES), ref["bn"].sorted_values)
    assert np.array_equal(ctx.debug_copy(nat.DBG_TILE_RANGES), ref["bn"].ranges)
    assert np.array_equal(vis.view(np.int32) != 0, ref["pr"].visibility != 0)
    st = ctx.stats()
    assert st["I"] == len(ref["bn"].sorted_keys) and st["V"] == int((ref["pr"].tiles_count > 0).sum())
    # image
    P = hw
    mean_e, max_e, bad = image_error_report(f"{label} cam{cam_index} rgba", rgba.reshape(ref["rgba"].shape), ref["rgba"])
    assert mean_e <= 1e-5 and max_e <= 2e-2 and bad <= max(3, int(2e-4 * P))
    dscale = max(1.0, float(np.abs(ref["dist"]).max()))
    mean_e, max_e, bad = image_error_report(f"{label} cam{cam_index} dist", dist.reshape(ref["dist"].shape), ref["dist"], atol=1e-4 * dscale)
    assert mean_e <= 1e-5 * dscale and bad <= max(3, int(2e-4 * P))
    same_hits = float(np.mean(hits.reshape(ref["hits"].shape) == ref["hits"]))
    print(f"[headline] {label} cam{cam_index}: hit counts equal on {same_hits * 100:.4f} % of the pixels")
    assert same_hits >= 0.999
    # gradients (the oracle's backward starts from ITS forward outputs, ours from ours: the comparison includes that difference)
    dp, ds = np.zeros((n, 12), np.float32), np.zeros((n, 48), np.float32)
    ctx.backward_host(cam, n, p(sc.particles), p(sc.sph), sc.sph_degree, p(ro), p(rd), p(rgba), p(ref["d_rgba"]), p(dist), p(ref["d_dist"]),
                      p(dp), p(ds))
    rdp, rdp64 = ref["dp"], ref["dp_64"]
    cols = dict(pos=slice(0, 3), dns=slice(3, 4), quat=slice(4, 8), scl=slice(8, 11))
    errs = {k: rel_l2(dp[:, v], rdp[:, v]) for k, v in cols.items()}
    errs["sph"] = rel_l2(ds, ref["ds"])
    yard = {k: rel_l2(rdp[:, v], rdp64[:, v]) for k, v in cols.items()}
    yard["sph"] = rel_l2(ref["ds"], ref["ds_64"])
    # the ten particles with the largest f32-vs-f64 disagreement OF THE ORACLE (all gradient columns): borderline accept flips
    e2 = ((rdp.astype(np.float64) - rdp64) ** 2).sum(1) / max(float((rdp64 ** 2).sum()), 1e-300) \
        + ((ref["ds"].astype(np.float64) - ref["ds_64"]) ** 2).sum(1) / max(float((ref["ds_64"] ** 2).sum()), 1e-300)
    keep = np.ones(n, bool)
    keep[np.argsort(-e2)[:10]] = False
    robust = {k: rel_l2(dp[keep][:, v], rdp[keep][:, v]) for k, v in cols.items()}
    robust["sph"] = rel_l2(ds[keep], ref["ds"][keep])
    fmt = lambda d: {k: f"{v:.2e}" for k, v in d.items()}  # noqa: E731
    print(f"[headline] {label} cam{cam_index} gradient rel-L2 vs oracle:", fmt(errs))
    print(f"[headline] {label} cam{cam_index} yardstick (oracle f32 vs f64, same lists):", fmt(yard))
    print(f"[headline] {label} cam{cam_index} gradient rel-L2 without the oracle's 10 flip particles:", fmt(robust))
    over = {k: v for k, v in errs.items() if v > 1e-3}
    if over:
        print(f"[headline] {label} cam{cam_index}: ABOVE the flat 1e-3 bar: {fmt(over)} -- allowed only up to 1.5 x this frame's yardstick")
    for k in errs:
        assert errs[k] <= max(1e-3, 1.5 * yard[k]), (k, errs[k], yard[k])
        assert robust[k] <= 1e-3, (k, robust[k])
    assert np.all(dp[:, 11] == 0)
    ctx.close()


@pytest.mark.parametrize("cam_index,d_dist,d_alpha", [
    pytest.param(3, "random", "random", id="3"), pytest.param(41, "random", "random", id="41"),
    pytest.param(3, "zero", "random", id="3-zero_d_dist"), pytest.param(3, "zero", "zero", id="3-zero_d_dist-zero_d_alpha"),
    pytest.param(41, "mixed", "random", id="41-mixed_d_dist")])
def test_c2_full_scale_oracle_parity(cam_index, d_dist, d_alpha):
    """BASELINE configs[1]: the bench workload itself (scenes.scene_c2(): 300k Gaussians, 800x800), two of its 100 orbit cameras.
    zero d_dist: the backward as training runs it (each warp skips the depth branch: the closed-form normalize adjoint, 4 flushed
    gradient columns), with zero d_alpha as well for an image loss on a black background; mixed: warps with and without the depth branch
    in one frame (helpers.dist_grad_mask)."""
    _check_frame("c2", scenes.scene_c2(), cam_index, 100, seed=cam_index, d_dist=d_dist, d_alpha=d_alpha)


def test_c3_like_oracle_parity():
    """C3-like unbounded scene (70 % within radius 3, background to radius 50, particles partly behind the camera) at the C3 resolution
    1237x822 (ragged: 78 x 52 tiles, partial tiles on both edges) with 400k Gaussians: tile lists beyond 1000 entries."""
    _check_frame("c3_small", scenes.scene_c3(n=400_000), 1, 10, seed=11)


def test_c3_like_oracle_parity_without_distance_gradient():
    """The C3-like frame above with the backward as training runs it: d_dist = 0 on every pixel."""
    _check_frame("c3_small", scenes.scene_c3(n=400_000), 1, 10, seed=11, d_dist="zero")


def _dense(model):
    """>= 50k Gaussians on a 256x256 image: ~700 entries per tile."""
    base = scenes.scene_c2(n=60_000, width=256, height=256)
    if model == "pinhole_distorted":
        return base
    f = 0.9 * base.width
    if model == "fisheye":
        return dataclasses.replace(base, fx=f, fy=f, fisheye=(0.05, -0.01, 0.002, -0.0003, 0.6))
    a1, a3 = 1.0 / f, 0.04 / f ** 3
    ft = dict(reference_poly=0, bw=[0.0, a1, 0.0, a3, 0.0, 0.0], fw=[0.0, f, 0.0, -0.04 * f, 0.0, 0.0], cde=[1.0, 0.001, -0.002],
              max_angle=0.6, principal=(base.width / 2.0 - 0.5, base.height / 2.0 - 0.5))
    return dataclasses.replace(base, fx=1.0, fy=1.0, ftheta=ft)


@pytest.mark.parametrize("model", ["fisheye", "ftheta"])
def test_wide_angle_models_on_a_dense_scene(model):
    """One case per non-pinhole camera model with tile lists well beyond one staged batch.  atan2f is not correctly rounded on either side,
    so tile counts are compared per particle (>= 99.9 % equal) and the image bar is widened by the differing particles (as in
    test_fisheye_camera_parity)."""
    from test_gut_parity_gpu import _run

    sc = _dense(model)
    c2w = sc.camera(2, 10)
    ref = oracle_frame(sc, c2w, seed=2, pose=tracer_pose(c2w))
    lens = ref["bn"].ranges[:, 1].astype(np.int64) - ref["bn"].ranges[:, 0]
    print(f"[headline] {model}: I={len(ref['bn'].sorted_keys)} longest tile list {int(lens.max())}")
    assert lens.max() > 256
    tr, g, out, dbg = _run(sc, c2w, ref)
    same = dbg["count"] == ref["pr"].tiles_count
    print(f"[headline] {model}: tile counts equal on {same.mean() * 100:.4f} % of the particles")
    assert same.mean() >= 0.999
    ok = same & (dbg["count"] > 0)
    assert np.array_equal(dbg["depth"].view(np.uint32)[ok], ref["pr"].depth.view(np.uint32)[ok])
    if same.all():
        assert np.array_equal(dbg["keys"], ref["bn"].sorted_keys) and np.array_equal(dbg["vals"], ref["bn"].sorted_values)
    rgba = torch.cat([out["pred_features"], out["pred_opacity"]], -1)[0].detach().cpu().numpy()
    P = rgba.shape[0] * rgba.shape[1]
    mean_e, max_e, bad = image_error_report(f"{model} dense rgba", rgba, ref["rgba"])
    assert mean_e <= 1e-5 and bad <= max(3, int(2e-4 * P)) + 16 * int((~same).sum())
    if same.all():
        dp = ref["dp"]
        errs = dict(pos=rel_l2(g.positions.grad.cpu().numpy(), dp[:, 0:3]), dns=rel_l2(g._dns.grad.cpu().numpy(), dp[:, 3:4]),
                    quat=rel_l2(g._rot.grad.cpu().numpy(), dp[:, 4:8]), scl=rel_l2(g._scl.grad.cpu().numpy(), dp[:, 8:11]),
                    sph=rel_l2(g._sph.grad.cpu().numpy(), ref["ds"]))
        print(f"[headline] {model} dense gradient rel-L2:", {k: f"{v:.2e}" for k, v in errs.items()})
        assert max(errs.values()) <= 1e-3


def test_distorted_pinhole_and_rolling_shutter_on_a_dense_scene():
    """OpenCV pinhole with all distortion terms + a rolling shutter on the dense scene: integer artefacts per particle (the pose interpolation
    calls acosf / sinf), image within the standard bar."""
    import b200_native as nat
    from oracle import gut_oracle as go

    sc = _dense("pinhole_distorted")
    p0 = scenes.pose7_from_c2w(sc.camera(1, 40))
    p1 = scenes.pose7_from_c2w(sc.camera(2, 40))
    ocam = go.make_camera(sc.width, sc.height, sc.fx, sc.fy, sc.cx, sc.cy, p0, p1, rolling_shutter=1)
    cam = _native_camera(sc, p0)
    cam.pose_end[:] = [float(v) for v in p1]
    cam.rolling_shutter = 1
    for c in (ocam, cam):
        c.radial[:] = [0.05, -0.01, 0.002, 0.01, 0.0, 0.0]
        c.tangential[:] = [0.001, -0.0005]
        c.thin_prism[:] = [0.0003, 0.0, -0.0002, 0.0]
    ro, rd = sc.rays()
    cfg = go.default_config()
    pr, bn, rgba_ref, dist_ref, hits_ref = go.forward_all(cfg, ocam, ro, rd, sc.particles, sc.sph, 3)
    lens = bn.ranges[:, 1].astype(np.int64) - bn.ranges[:, 0]
    assert lens.max() > 256
    ctx = nat.Context(nat.default_config(), 0)
    n, hw = sc.n, sc.width * sc.height
    rgba, dist, hits, vis = (np.zeros((hw, 4), np.float32), np.zeros(hw, np.float32), np.zeros(hw, np.float32), np.zeros(n, np.float32))
    p = lambda a: a.ctypes.data  # noqa: E731
    ro_c, rd_c = np.ascontiguousarray(ro), np.ascontiguousarray(rd)
    ctx.forward_host(cam, n, p(sc.particles), p(sc.sph), 3, p(ro_c), p(rd_c), p(rgba), p(dist), p(hits), p(vis))
    count = ctx.debug_copy(nat.DBG_TILES_COUNT)
    same = count == pr.tiles_count
    print(f"[headline] distorted pinhole + rolling shutter: I={len(bn.sorted_keys)} longest list {int(lens.max())}, tile counts equal on "
          f"{same.mean() * 100:.4f} % of the particles")
    assert same.mean() >= 0.999
    if same.all():
        assert np.array_equal(ctx.debug_copy(nat.DBG_SORTED_KEYS), bn.sorted_keys)
        assert np.array_equal(ctx.debug_copy(nat.DBG_SORTED_VALUES), bn.sorted_values)
    mean_e, max_e, bad = image_error_report("distorted pinhole + rolling shutter rgba", rgba.reshape(rgba_ref.shape), rgba_ref)
    assert mean_e <= 1e-5 and bad <= max(3, int(2e-4 * hw)) + 16 * int((~same).sum())
    ctx.close()

"""GPU parity of the CUDA 3DGUT path against the CPU oracle (SURVEY.md section 8c).

Tolerance policy (DESIGN.md section 5):
  * tile counts, depth bits, sorted (key, value) stream, tile ranges: BIT-EXACT;
  * RGBA / distance: mean |diff| <= 1e-5, |diff| <= 1e-4 on all but max(3, 2e-4 * P) pixels, max |diff| <= 2e-2.
    The accept test `response > 0.0113 and alpha > 1/255` is discontinuous: two valid fp32 evaluation orders can flip a
    borderline (pixel, particle) pair, which moves that pixel by up to alpha ~ 1e-2.  The yardstick is the oracle itself
    evaluated in double on the same lists (oracle f32 vs f64 shows the same kind of isolated flips at C2-like scales);
  * hit counts equal on >= 99.9 % of pixels;
  * gradients: relative L2 error <= 1e-3 per tensor (fp32 atomics reorder the sums; flips add ~3e-4 at C2-like scales).
"""
import numpy as np
import pytest

import scenes
from helpers import frac_within, image_error_report, oracle_frame, rel_l2, tracer_pose

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def _tracer():
    import threedgut_tracer

    return threedgut_tracer.Tracer({"render": {"enable_kernel_timings": True}})


class _Gaussians:
    """Minimal stand-in for MixtureOfGaussians: the attributes Tracer.render reads (SURVEY 8b)."""

    def __init__(self, sc, device):
        p = torch.from_numpy(sc.particles).to(device)
        self.positions = p[:, 0:3].clone().requires_grad_(True)
        self._dns = p[:, 3:4].clone().requires_grad_(True)
        self._rot = p[:, 4:8].clone().requires_grad_(True)
        self._scl = p[:, 8:11].clone().requires_grad_(True)
        self._sph = torch.from_numpy(sc.sph).to(device).requires_grad_(True)
        self.n_active_features = sc.sph_degree
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


class _Batch:
    def __init__(self, sc, c2w, device):
        ro, rd = sc.rays()
        self.rays_ori = torch.from_numpy(ro).to(device)
        self.rays_dir = torch.from_numpy(rd).to(device)
        self.T_to_world = torch.from_numpy(np.asarray(c2w, np.float32))[None]
        self.T_to_world_end = None
        self.rays_in_world_space = False
        self.intrinsics = None
        self.intrinsics_OpenCVPinholeCameraModelParameters = dict(
            resolution=np.array([sc.width, sc.height]), shutter_type="GLOBAL", principal_point=np.array([sc.cx, sc.cy], np.float32),
            focal_length=np.array([sc.fx, sc.fy], np.float32), radial_coeffs=np.zeros(6, np.float32),
            tangential_coeffs=np.zeros(2, np.float32), thin_prism_coeffs=np.zeros(4, np.float32))
        if getattr(sc, "ftheta", None) is not None:
            ft = sc.ftheta
            self.intrinsics_OpenCVPinholeCameraModelParameters = None
            self.intrinsics_FThetaCameraModelParameters = dict(
                resolution=np.array([sc.width, sc.height]), shutter_type="GLOBAL", principal_point=np.asarray(ft["principal"], np.float32),
                reference_poly="PIXELDIST_TO_ANGLE" if ft["reference_poly"] == 0 else "ANGLE_TO_PIXELDIST",
                pixeldist_to_angle_poly=np.asarray(ft["bw"], np.float32), angle_to_pixeldist_poly=np.asarray(ft["fw"], np.float32),
                max_angle=float(ft["max_angle"]), linear_cde=np.asarray(ft["cde"], np.float32))
        elif getattr(sc, "fisheye", None) is not None:
            self.intrinsics_OpenCVPinholeCameraModelParameters = None
            self.intrinsics_OpenCVFisheyeCameraModelParameters = dict(
                resolution=np.array([sc.width, sc.height]), shutter_type="GLOBAL", principal_point=np.array([sc.cx, sc.cy], np.float32),
                focal_length=np.array([sc.fx, sc.fy], np.float32), radial_coeffs=np.asarray(sc.fisheye[:4], np.float32),
                max_angle=float(sc.fisheye[4]))


def _run(sc, c2w, ref):
    dev = torch.device("cuda", 0)
    tr = _tracer()
    g = _Gaussians(sc, dev)
    out = tr.render(g, _Batch(sc, c2w, dev), train=True)
    ctx = tr.tracer_wrapper.native_context(dev)
    import b200_native as nat

    dbg = {k: ctx.debug_copy(v) for k, v in dict(count=nat.DBG_TILES_COUNT, keys=nat.DBG_SORTED_KEYS, vals=nat.DBG_SORTED_VALUES,
                                                 ranges=nat.DBG_TILE_RANGES, depth=nat.DBG_DEPTH, rgb=nat.DBG_RGB).items()}
    loss = (out["pred_features"] * torch.from_numpy(ref["d_rgba"][None, ..., :3]).to(dev)).sum() \
        + (out["pred_opacity"] * torch.from_numpy(ref["d_rgba"][None, ..., 3:]).to(dev)).sum() \
        + (out["pred_dist"] * torch.from_numpy(ref["d_dist"][None]).to(dev)).sum()
    loss.backward()
    torch.cuda.synchronize()
    return tr, g, out, dbg


@pytest.mark.parametrize("cam_index,size", [(0, (128, 128)), (3, (128, 128)), (7, (128, 128)), (5, (75, 53))])
@pytest.mark.parametrize("bands", [False, True])
def test_c1_integer_artifacts_bit_exact(cam_index, bands, size):
    sc = scenes.scene_c1(bands=bands, width=size[0], height=size[1])
    c2w = sc.camera(cam_index, 10)
    ref = oracle_frame(sc, c2w, pose=tracer_pose(c2w))
    _, _, _, dbg = _run(sc, c2w, ref)
    assert np.array_equal(dbg["count"], ref["pr"].tiles_count)
    assert np.array_equal(dbg["depth"].view(np.uint32), ref["pr"].depth.view(np.uint32))
    assert np.array_equal(dbg["keys"], ref["bn"].sorted_keys)
    assert np.array_equal(dbg["vals"], ref["bn"].sorted_values)
    assert np.array_equal(dbg["ranges"], ref["bn"].ranges)
    vis = ref["pr"].tiles_count > 0
    assert np.allclose(dbg["rgb"][vis], ref["pr"].rgb[vis], atol=2e-6, rtol=1e-6)


@pytest.mark.parametrize("cam_index,size", [(0, (128, 128)), (3, (128, 128)), (7, (128, 128)), (5, (75, 53))])
def test_c1_forward_and_gradients(cam_index, size):
    """size (75, 53): ragged image -- partial tiles and partially filled warps in the render kernels and their culling."""
    sc = scenes.scene_c1(width=size[0], height=size[1])
    c2w = sc.camera(cam_index, 10)
    ref = oracle_frame(sc, c2w, seed=cam_index, pose=tracer_pose(c2w))
    tr, g, out, _ = _run(sc, c2w, ref)
    rgba = torch.cat([out["pred_features"], out["pred_opacity"]], -1)[0].detach().cpu().numpy()
    dist = out["pred_dist"][0].detach().cpu().numpy()
    hits = out["hits_count"][0].detach().cpu().numpy()
    mean_e, max_e, bad = image_error_report(f"c1 cam{cam_index} rgba", rgba, ref["rgba"])
    assert mean_e <= 1e-5 and max_e <= 2e-2 and bad <= max(3, int(2e-4 * rgba.shape[0] * rgba.shape[1]))
    mean_e, max_e, bad = image_error_report(f"c1 cam{cam_index} dist", dist, ref["dist"], atol=1e-4 * max(1.0, float(np.abs(ref["dist"]).max())))
    assert mean_e <= 1e-4 and bad <= max(3, int(2e-4 * rgba.shape[0] * rgba.shape[1]))
    assert float(np.mean(hits == ref["hits"])) >= 0.999
    vis = out["mog_visibility"].detach().cpu().numpy().view(np.int32).reshape(-1)
    assert np.array_equal(vis != 0, ref["pr"].visibility != 0)
    dp = ref["dp"]
    errs = dict(pos=rel_l2(g.positions.grad.cpu().numpy(), dp[:, 0:3]), dns=rel_l2(g._dns.grad.cpu().numpy(), dp[:, 3:4]),
                quat=rel_l2(g._rot.grad.cpu().numpy(), dp[:, 4:8]), scl=rel_l2(g._scl.grad.cpu().numpy(), dp[:, 8:11]),
                sph=rel_l2(g._sph.grad.cpu().numpy(), ref["ds"]))
    print("[parity] c1 cam%d gradient rel-L2:" % cam_index, {k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) <= 1e-3
    t = tr.timings
    assert "forward_render" in t or "backward_render" in t


def test_c_abi_host_entry_points_match_device_path():
    """gutb200_forward_host / backward_host (the e2e path) give the same numbers as the device-pointer path."""
    import b200_native as nat

    sc = scenes.scene_c1()
    c2w = sc.camera(2, 10)
    ref = oracle_frame(sc, c2w)
    cfg = nat.default_config()
    ctx = nat.Context(cfg, 0)
    cam = nat.Camera()
    cam.width, cam.height = sc.width, sc.height
    cam.principal[:] = [sc.cx, sc.cy]
    cam.focal[:] = [sc.fx, sc.fy]
    cam.pose_start[:] = [float(v) for v in ref["pose"]]
    cam.pose_end[:] = [float(v) for v in ref["pose"]]
    n, hw = sc.n, sc.width * sc.height
    rgba, dist, hits, vis = (np.zeros((hw, 4), np.float32), np.zeros(hw, np.float32), np.zeros(hw, np.float32), np.zeros(n, np.float32))
    p = lambda a: a.ctypes.data  # noqa: E731
    ro, rd = np.ascontiguousarray(ref["ro"]), np.ascontiguousarray(ref["rd"])
    ctx.forward_host(cam, n, p(sc.particles), p(sc.sph), 3, p(ro), p(rd), p(rgba), p(dist), p(hits), p(vis))
    mean_e, max_e, bad = image_error_report("c-abi host rgba", rgba.reshape(ref["rgba"].shape), ref["rgba"])
    assert mean_e <= 1e-5 and max_e <= 2e-2 and bad <= 3
    dp, ds = np.zeros((n, 12), np.float32), np.zeros((n, 48), np.float32)
    ctx.backward_host(cam, n, p(sc.particles), p(sc.sph), 3, p(ro), p(rd), p(rgba), p(ref["d_rgba"]), p(dist), p(ref["d_dist"]), p(dp), p(ds))
    assert rel_l2(dp, ref["dp"]) <= 1e-3
    assert rel_l2(ds, ref["ds"]) <= 1e-3
    assert ctx.launch_count() >= 6
    ctx.close()


def _host_frame(ctx, sc, pose, d_rgba, d_dist):
    import b200_native as nat

    cam = nat.Camera()
    cam.width, cam.height = sc.width, sc.height
    cam.principal[:] = [sc.cx, sc.cy]
    cam.focal[:] = [sc.fx, sc.fy]
    cam.pose_start[:] = [float(v) for v in pose]
    cam.pose_end[:] = [float(v) for v in pose]
    n, hw = sc.n, sc.width * sc.height
    rgba, dist, hits, vis = (np.zeros((hw, 4), np.float32), np.zeros(hw, np.float32), np.zeros(hw, np.float32), np.zeros(n, np.float32))
    p = lambda a: a.ctypes.data  # noqa: E731
    ro, rd = sc.rays()
    ro, rd = np.ascontiguousarray(ro), np.ascontiguousarray(rd)
    ctx.forward_host(cam, n, p(sc.particles), p(sc.sph), sc.sph_degree, p(ro), p(rd), p(rgba), p(dist), p(hits), p(vis))
    dp, ds = np.zeros((n, 12), np.float32), np.zeros((n, 48), np.float32)
    ctx.backward_host(cam, n, p(sc.particles), p(sc.sph), sc.sph_degree, p(ro), p(rd), p(rgba), p(d_rgba), p(dist), p(d_dist), p(dp), p(ds))
    return rgba, dist, hits, dp, ds


@pytest.mark.parametrize("scene_name,degree", [("c1", 2), ("c1", 4), ("c2", 2), ("c2", 4), ("c3_small", 2)])
def test_subtile_culling_is_bit_identical(scene_name, degree):
    """The conic pre-test of the render kernels (gut_render.cu, ours) only drops (pixel, particle) pairs the exact test
    would reject: forward outputs must be BIT-identical with the switch on and off, gradients equal up to the order of
    the atomics.  Covers tiny particles (c1), a dense object (c2, both kernel degrees) and an unbounded scene with
    large / partly-behind-the-camera particles (c3)."""
    import b200_native as nat

    if scene_name == "c1":
        sc = scenes.scene_c1()
    elif scene_name == "c2":
        sc = scenes.scene_c2()
    else:
        sc = scenes.scene_c3(n=400_000, width=640, height=400)
    rng = np.random.default_rng(5)
    hw = sc.width * sc.height
    d_rgba = rng.normal(size=(hw, 4)).astype(np.float32)
    d_dist = (0.1 * rng.normal(size=hw)).astype(np.float32)
    for cam_index in (1, 6):
        pose = tracer_pose(sc.camera(cam_index, 10))
        out = []
        for mode in (7, 5, 0):  # default (screens + hit words, quarter-warp walk) / hit words without the forward screens / neither
            cfg = nat.default_config()
            cfg.kernel_degree = degree
            cfg.subtile_culling = mode
            ctx = nat.Context(cfg, 0)
            out.append(_host_frame(ctx, sc, pose, d_rgba, d_dist))
            ctx.close()
        (rgba1, dist1, hits1, dp1, ds1), (rgba5, dist5, hits5, dp5, ds5), (rgba0, dist0, hits0, dp0, ds0) = out
        assert hits0.sum() > 0
        for rgba_, dist_, hits_ in ((rgba5, dist5, hits5), (rgba0, dist0, hits0)):
            assert np.array_equal(hits1, hits_), f"hit counts differ on {(hits1 != hits_).sum()} pixels"
            assert np.array_equal(rgba1.view(np.uint32), rgba_.view(np.uint32))
            assert np.array_equal(dist1.view(np.uint32), dist_.view(np.uint32))
        # the screens drop only pairs nobody accepts: same hit words, same gradients up to the order of the atomics (canonical sums are
        # mapped to pos / scale / quat after the reduction, so the order noise of the sums passes through three small linear maps)
        assert rel_l2(dp1, dp5) <= 1e-4 and rel_l2(ds1, ds5) <= 1e-5
        # hit words on / off: the backward re-tests every pair either way; the words only skip entries no pixel of the warp accepted in
        # the forward, whose arithmetic differs from the backward's in the last bits (scale folded into the rotation rows) -- a borderline pair
        # accepted by one and not the other is the only possible difference
        e_dp, e_ds = rel_l2(dp1, dp0), rel_l2(ds1, ds0)
        print(f"[hit words] {scene_name} deg{degree} cam{cam_index}: gradients with vs without the forward's hit words: rel-L2 {e_dp:.2e} / {e_ds:.2e}")
        assert e_dp <= 3e-4 and e_ds <= 3e-4


def test_work_counters_are_consistent():
    """Debug work counters (bench.py's roofline_fp32): reference pair tests >= executed tests >= hits, accepted pairs == the image's hit
    counts, screens only ever remove tests."""
    import b200_native as nat

    sc = scenes.scene_c2(n=60_000, width=400, height=400)
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    ro, rd = sc.rays()
    particles, sph, tro, trd = t(sc.particles), t(sc.sph), t(ro), t(rd)
    pose = tracer_pose(sc.camera(2, 10))
    res = {}
    for mode in (7, 5):
        cfg = nat.default_config()
        cfg.subtile_culling = mode
        ctx = nat.Context(cfg, 0)
        cam = nat.Camera()
        cam.width, cam.height = sc.width, sc.height
        cam.principal[:] = [sc.cx, sc.cy]
        cam.focal[:] = [sc.fx, sc.fy]
        cam.pose_start[:] = [float(v) for v in pose]
        cam.pose_end[:] = [float(v) for v in pose]
        rgba = torch.empty((sc.height, sc.width, 4), device=dev)
        dist = torch.empty((sc.height, sc.width, 1), device=dev)
        hits = torch.empty((sc.height, sc.width, 1), device=dev)
        vis = torch.empty((sc.n, 1), device=dev)
        s = torch.cuda.current_stream(dev).cuda_stream
        ctx.forward(s, cam, sc.n, particles.data_ptr(), sph.data_ptr(), sc.sph_degree, tro.data_ptr(), trd.data_ptr(), rgba.data_ptr(), dist.data_ptr(),
                    hits.data_ptr(), vis.data_ptr())
        w = ctx.work_counters(particles.data_ptr(), tro.data_ptr(), trd.data_ptr())
        w["image_hits"] = int(hits.sum().item())
        w["I"] = ctx.stats()["I"]
        res[mode] = w
        print(f"[work] mode {mode}: {w}")
        assert w["tests_ref"] >= w["tests_exec"] >= w["hits"] > 0
        assert w["tests_ref"] <= 256 * w["I"]
        assert w["fwd_iters"] >= w["hit_iters"] > 0 and w["bwd_lanes"] <= 32 * w["hit_iters"]
        # accepted pairs >= composited hits (the t-range test and w > 0 only remove)
        assert w["hits"] >= w["image_hits"] and w["hits"] <= 1.01 * w["image_hits"] + 16
        assert 1.0 <= w["tests_exec"] / w["hits"]
        ctx.close()
    assert res[7]["tests_ref"] == res[5]["tests_ref"] and res[7]["hits"] == res[5]["hits"] and res[7]["hit_iters"] == res[5]["hit_iters"]
    assert res[7]["tests_exec"] < res[5]["tests_exec"] and res[5]["screens"] == 0
    assert abs(res[5]["tests_exec"] - res[5]["tests_ref"]) <= 0.001 * res[5]["tests_ref"]


def test_empty_and_offscreen_inputs():
    """Edge cases: zero particles, and particles all behind the camera (I = 0)."""
    _empty_and_offscreen_inputs(0)


def test_empty_offscreen_and_single_particle_inputs_sorted():
    """The same edge cases through the sorted variant (a k-buffer of 16 hits), and a single particle in view against the oracle's k-buffer."""
    _empty_and_offscreen_inputs(16)


def _empty_and_offscreen_inputs(k):
    import b200_native as nat

    sc = scenes.scene_c1(n=64)
    c2w = sc.camera(0, 4)
    ref = oracle_frame(sc, c2w)
    cfg = nat.default_config()
    cfg.k_buffer_size = k
    ctx = nat.Context(cfg, 0)
    cam = nat.Camera()
    cam.width, cam.height = sc.width, sc.height
    cam.principal[:] = [sc.cx, sc.cy]
    cam.focal[:] = [sc.fx, sc.fy]
    cam.pose_start[:] = [float(v) for v in ref["pose"]]
    cam.pose_end[:] = [float(v) for v in ref["pose"]]
    hw = sc.width * sc.height
    p = lambda a: a.ctypes.data  # noqa: E731
    ro, rd = np.ascontiguousarray(ref["ro"]), np.ascontiguousarray(ref["rd"])
    behind = sc.particles.copy()
    behind[:, 0:3] = behind[:, 0:3] * 0.05 + 3.0 * np.asarray(c2w)[:3, 3]  # beyond the camera, outside its frustum
    for parts in (np.zeros((0, 12), np.float32), behind):
        n = parts.shape[0]
        sph = np.zeros((max(n, 1), 48), np.float32)
        rgba, dist, hits, vis = (np.ones((hw, 4), np.float32), np.zeros(hw, np.float32), np.ones(hw, np.float32), np.ones(max(n, 1), np.float32))
        buf = parts if n else np.zeros((1, 12), np.float32)
        ctx.forward_host(cam, n, p(buf), p(sph), 3, p(ro), p(rd), p(rgba), p(dist), p(hits), p(vis))
        assert ctx.stats()["I"] == 0
        assert np.all(rgba == 0) and np.all(hits == 0) and np.all(dist == 0)
        dp, ds = np.ones((max(n, 1), 12), np.float32), np.ones((max(n, 1), 48), np.float32)
        ctx.backward_host(cam, n, p(buf), p(sph), 3, p(ro), p(rd), p(rgba), p(rgba), p(dist), p(dist), p(dp), p(ds))
        if n:
            assert np.all(dp == 0) and np.all(ds == 0)
    if k:
        _single_particle_kbuffer(ctx, cam, sc, ref, k)
    ctx.close()


def _single_particle_kbuffer(ctx, cam, sc, ref, k):
    """One particle in view, the largest of the scene in the frame: every ray holds at most one hit, which leaves the buffer in the drain."""
    from oracle import gut_oracle as go

    vis = np.flatnonzero(ref["pr"].tiles_count > 0)
    one = sc.particles[vis[np.argmax(ref["pr"].tiles_count[vis])]][None].copy()
    one[:, 3] = 0.9
    sph = np.ascontiguousarray(sc.sph[vis[:1]])
    cfg = go.default_config()
    pr = go.project(cfg, ref["cam"], one, sph, 3)
    bn = go.bin_tiles(cfg, ref["cam"], pr)
    rgba_ref, dist_ref, hits_ref = go.render_forward_kbuffer(cfg, ref["cam"], k, ref["ro"], ref["rd"], one, pr, bn)
    d_rgba, d_dist = ref["d_rgba"], ref["d_dist"]
    dp_ref, ds_ref = go.render_backward_kbuffer(cfg, ref["cam"], k, ref["ro"], ref["rd"], one, sph, 3, pr, bn, rgba_ref, dist_ref, d_rgba, d_dist)
    assert hits_ref.max() == 1 and hits_ref.sum() >= 16
    hw = sc.width * sc.height
    p = lambda a: a.ctypes.data  # noqa: E731
    ro, rd = np.ascontiguousarray(ref["ro"]), np.ascontiguousarray(ref["rd"])
    rgba, dist, hits, vis1 = (np.zeros((hw, 4), np.float32), np.zeros(hw, np.float32), np.zeros(hw, np.float32), np.zeros(1, np.float32))
    ctx.forward_host(cam, 1, p(one), p(sph), 3, p(ro), p(rd), p(rgba), p(dist), p(hits), p(vis1))
    mean_e, max_e, bad = image_error_report(f"single particle K={k} rgba", rgba.reshape(rgba_ref.shape), rgba_ref)
    assert mean_e <= 1e-5 and max_e <= 2e-2 and bad <= 3
    assert np.array_equal(hits.reshape(hits_ref.shape), hits_ref)
    dp, ds = np.zeros((1, 12), np.float32), np.zeros((1, 48), np.float32)
    ctx.backward_host(cam, 1, p(one), p(sph), 3, p(ro), p(rd), p(rgba), p(np.ascontiguousarray(d_rgba)), p(dist),
                      p(np.ascontiguousarray(d_dist)), p(dp), p(ds))
    errs = (rel_l2(dp, dp_ref), rel_l2(ds, ds_ref))
    print(f"[parity] single particle K={k}: {int(hits_ref.sum())} hit pixels, gradient rel-L2 {errs[0]:.2e} / {errs[1]:.2e} (bar 1e-3)")
    assert max(errs) <= 1e-3


def test_per_pixel_ray_origins_take_the_general_path():
    """Rays whose origins differ inside a tile must not use the common-origin fast path (render kernels pick it per tile).  Three bands of
    tiles: the frame's first-ray origin (forward UNIFORM, backward FAST: canonical sums relative to that origin), ANOTHER origin common to
    the tile (forward UNIFORM with exact hit words, backward GENERAL with the origin-offset correction terms), per-pixel jitter (both general)."""
    _per_pixel_ray_origins(0)


def test_per_pixel_ray_origins_sorted():
    """The same three bands through the sorted variant (a k-buffer of 16 hits), whose walk sets up every ray from its own origin, against the
    oracle's k-buffer."""
    _per_pixel_ray_origins(16)


def _per_pixel_ray_origins(k):
    import b200_native as nat
    from oracle import gut_oracle as go

    sc = scenes.scene_c1()
    c2w = sc.camera(4, 10)
    pose = scenes.pose7_from_c2w(c2w)
    ro, rd = sc.rays()
    rng = np.random.default_rng(3)
    ro = (ro + 0.02 * rng.normal(size=ro.shape)).astype(np.float32)
    ro[:, :32] = ro[0, 0, 0]                                              # tiles 0-1: the frame origin
    ro[:, 32:64] = ro[0, 0, 0] + np.array([0.03, -0.02, 0.05], np.float32)  # tiles 2-3: common to the tile, different from the frame's
    # columns 64..: per-pixel jitter
    cfg = go.default_config()
    ocam = go.make_camera(sc.width, sc.height, sc.fx, sc.fy, sc.cx, sc.cy, pose)
    pr = go.project(cfg, ocam, sc.particles, sc.sph, 3)
    bn = go.bin_tiles(cfg, ocam, pr)
    if k:
        rgba_ref, dist_ref, hits_ref = go.render_forward_kbuffer(cfg, ocam, k, ro, rd, sc.particles, pr, bn)
    else:
        rgba_ref, dist_ref, hits_ref = go.render_forward(cfg, ocam, ro, rd, sc.particles, pr, bn)
    d_rgba = rng.normal(size=rgba_ref.shape).astype(np.float32)
    d_dist = (0.1 * rng.normal(size=dist_ref.shape)).astype(np.float32)
    if k:
        dp_ref, ds_ref = go.render_backward_kbuffer(cfg, ocam, k, ro, rd, sc.particles, sc.sph, 3, pr, bn, rgba_ref, dist_ref, d_rgba, d_dist)
        from helpers import kbuffer_premises

        assert kbuffer_premises("jittered origins", cfg, ocam, k, ro, rd, sc.particles, pr, bn, hits_ref)["over_k"] > 0.05
    else:
        dp_ref, ds_ref = go.render_backward(cfg, ocam, ro, rd, sc.particles, sc.sph, 3, pr, bn, rgba_ref, dist_ref, d_rgba, d_dist)
    ncfg = nat.default_config()
    ncfg.k_buffer_size = k
    ctx = nat.Context(ncfg, 0)
    cam = nat.Camera()
    cam.width, cam.height = sc.width, sc.height
    cam.principal[:] = [sc.cx, sc.cy]
    cam.focal[:] = [sc.fx, sc.fy]
    cam.pose_start[:] = [float(v) for v in pose]
    cam.pose_end[:] = [float(v) for v in pose]
    n, hw = sc.n, sc.width * sc.height
    rgba, dist, hits, vis = (np.zeros((hw, 4), np.float32), np.zeros(hw, np.float32), np.zeros(hw, np.float32), np.zeros(n, np.float32))
    p = lambda a: a.ctypes.data  # noqa: E731
    ro_c, rd_c = np.ascontiguousarray(ro), np.ascontiguousarray(rd)
    ctx.forward_host(cam, n, p(sc.particles), p(sc.sph), 3, p(ro_c), p(rd_c), p(rgba), p(dist), p(hits), p(vis))
    mean_e, max_e, bad = image_error_report("jittered origins rgba", rgba.reshape(rgba_ref.shape), rgba_ref)
    assert mean_e <= 1e-5 and max_e <= 2e-2 and bad <= 3
    dp, ds = np.zeros((n, 12), np.float32), np.zeros((n, 48), np.float32)
    ctx.backward_host(cam, n, p(sc.particles), p(sc.sph), 3, p(ro_c), p(rd_c), p(rgba), p(d_rgba), p(dist), p(d_dist), p(dp), p(ds))
    assert float(np.mean(hits.reshape(hits_ref.shape) == hits_ref)) >= 0.999
    errs = (rel_l2(dp, dp_ref), rel_l2(ds, ds_ref))
    print(f"[parity] jittered origins K={k}: gradient rel-L2 d_particles {errs[0]:.2e}, d_sph {errs[1]:.2e} (bar 1e-3)")
    assert max(errs) <= 1e-3
    ctx.close()


def test_distorted_pinhole_takes_the_general_projection_path():
    """Non-zero OpenCV distortion coefficients: tile counts / keys stay bit-exact (cameraProjections.cuh:72-118)."""
    import b200_native as nat
    from oracle import gut_oracle as go

    sc = scenes.scene_c1()
    pose = scenes.pose7_from_c2w(sc.camera(5, 10))
    ocam = go.make_camera(sc.width, sc.height, sc.fx, sc.fy, sc.cx, sc.cy, pose)
    cam = nat.Camera()
    cam.width, cam.height = sc.width, sc.height
    cam.principal[:] = [sc.cx, sc.cy]
    cam.focal[:] = [sc.fx, sc.fy]
    cam.pose_start[:] = [float(v) for v in pose]
    cam.pose_end[:] = [float(v) for v in pose]
    for c in (ocam, cam):
        c.radial[:] = [0.05, -0.01, 0.002, 0.01, 0.0, 0.0]
        c.tangential[:] = [0.001, -0.0005]
        c.thin_prism[:] = [0.0003, 0.0, -0.0002, 0.0]
    ro, rd = sc.rays()
    cfg = go.default_config()
    pr, bn, rgba_ref, dist_ref, hits_ref = go.forward_all(cfg, ocam, ro, rd, sc.particles, sc.sph, 3)
    ctx = nat.Context(nat.default_config(), 0)
    n, hw = sc.n, sc.width * sc.height
    rgba, dist, hits, vis = (np.zeros((hw, 4), np.float32), np.zeros(hw, np.float32), np.zeros(hw, np.float32), np.zeros(n, np.float32))
    p = lambda a: a.ctypes.data  # noqa: E731
    ro_c, rd_c = np.ascontiguousarray(ro), np.ascontiguousarray(rd)
    ctx.forward_host(cam, n, p(sc.particles), p(sc.sph), 3, p(ro_c), p(rd_c), p(rgba), p(dist), p(hits), p(vis))
    assert np.array_equal(ctx.debug_copy(nat.DBG_TILES_COUNT), pr.tiles_count)
    assert np.array_equal(ctx.debug_copy(nat.DBG_SORTED_KEYS), bn.sorted_keys)
    assert np.array_equal(ctx.debug_copy(nat.DBG_SORTED_VALUES), bn.sorted_values)
    mean_e, max_e, bad = image_error_report("distorted pinhole rgba", rgba.reshape(rgba_ref.shape), rgba_ref)
    assert mean_e <= 1e-5 and max_e <= 2e-2 and bad <= 3
    ctx.close()


def test_error_conventions():
    """Failures surface as non-zero return codes / exceptions (the reference logs and drops its Status codes)."""
    import b200_native as nat

    ctx = nat.Context(nat.default_config(), 0)
    cam = nat.Camera()
    cam.width, cam.height = 32, 32
    buf = np.zeros((4, 64), np.float32)
    with pytest.raises(RuntimeError, match="forward context"):
        ctx.backward_host(cam, 1, buf.ctypes.data, buf.ctypes.data, 3, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data,
                          buf.ctypes.data, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data)
    bad = nat.default_config()
    bad.kernel_degree = 3
    ctx2 = nat.Context(bad, 0)
    with pytest.raises(RuntimeError, match="kernel_degree"):
        ctx2.forward_host(cam, 1, buf.ctypes.data, buf.ctypes.data, 3, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data,
                          buf.ctypes.data, buf.ctypes.data)
    cam.width = 0
    with pytest.raises(RuntimeError, match="resolution"):
        ctx.forward_host(cam, 1, buf.ctypes.data, buf.ctypes.data, 3, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data, buf.ctypes.data,
                         buf.ctypes.data, buf.ctypes.data)
    ctx.close()
    ctx2.close()


def test_backward_rejects_a_camera_other_than_the_forwards():
    """The backward replays the lists, the projection and the hit words of the immediately preceding forward: called with another view's
    camera (same resolution) it must fail, not mix two views silently (the reference uses the stale context, gutRenderer.cu:436-440)."""
    import b200_native as nat

    sc = scenes.scene_c1(n=200, width=64, height=64)
    ctx = nat.Context(nat.default_config(), 0)

    def camera(i):
        pose = tracer_pose(sc.camera(i, 10))
        cam = nat.Camera()
        cam.width, cam.height = sc.width, sc.height
        cam.principal[:] = [sc.cx, sc.cy]
        cam.focal[:] = [sc.fx, sc.fy]
        cam.pose_start[:] = [float(v) for v in pose]
        cam.pose_end[:] = [float(v) for v in pose]
        return cam

    n, hw = sc.n, sc.width * sc.height
    rgba, dist, hits, vis = (np.zeros((hw, 4), np.float32), np.zeros(hw, np.float32), np.zeros(hw, np.float32), np.zeros(n, np.float32))
    ro, rd = sc.rays()
    ro, rd = np.ascontiguousarray(ro), np.ascontiguousarray(rd)
    p = lambda a: a.ctypes.data  # noqa: E731
    ctx.forward_host(camera(1), n, p(sc.particles), p(sc.sph), 3, p(ro), p(rd), p(rgba), p(dist), p(hits), p(vis))
    dp, ds = np.zeros((n, 12), np.float32), np.zeros((n, 48), np.float32)
    d_rgba, d_dist = np.ones((hw, 4), np.float32), np.zeros(hw, np.float32)
    with pytest.raises(RuntimeError, match="differs from the immediately preceding forward"):
        ctx.backward_host(camera(2), n, p(sc.particles), p(sc.sph), 3, p(ro), p(rd), p(rgba), p(d_rgba), p(dist), p(d_dist), p(dp), p(ds))
    ctx.backward_host(camera(1), n, p(sc.particles), p(sc.sph), 3, p(ro), p(rd), p(rgba), p(d_rgba), p(dist), p(d_dist), p(dp), p(ds))
    assert np.abs(dp).sum() > 0
    ctx.close()


def test_compact_exchange_rebuilds_the_sh_gradient():
    """View-parallel exchange (gutb200_backward_compact + gutb200_sph_grad_from_views): the SH gradient rebuilt from the [N,4]
    radiance gradients of two views equals the sum of the two views' full [N,48] gradients, and d_particles is unchanged."""
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
    gen = torch.Generator(device=dev).manual_seed(7)
    full_dp, full_ds, gs, pos = [], [], [], []
    for view in (2, 7):
        pose = scenes.pose7_from_c2w(sc.camera(view, 10))
        d_rgba = torch.randn((H, W, 4), device=dev, generator=gen)
        d_dist = 0.05 * torch.randn((H, W, 1), device=dev, generator=gen)
        rgba, dst, hits, vis = raster.trace(0, 3, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose)
        dp, ds = raster.trace_bwd(0, 3, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose, rgba, d_rgba, dst, d_dist)
        full_dp.append(dp.clone())
        full_ds.append(ds.clone())
        rgba, dst, hits, vis = raster.trace(0, 3, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose)
        dp2, g = raster.trace_bwd_compact(0, 3, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose, rgba, d_rgba, dst, d_dist)
        assert rel_l2(dp2.cpu().numpy(), dp.cpu().numpy()) <= 2e-5  # atomics order only (through the per-particle maps of G8)
        gs.append(g.clone())
        pos.append(raster.sensor_position(sensor, pose, pose, W, H))
    assert np.allclose(pos[0], np.asarray(sc.camera(2, 10))[:3, 3], atol=1e-5)
    ds_sum = (full_ds[0] + full_ds[1]).cpu().numpy()
    rebuilt = raster.sph_grad_from_views(3, particles, np.stack(pos), torch.stack(gs)).cpu().numpy()
    assert np.abs(ds_sum).max() > 0
    assert rel_l2(rebuilt, ds_sum) <= 2e-6
    assert np.abs(rebuilt - ds_sum).max() <= 1e-5 * max(1.0, float(np.abs(ds_sum).max()))
    # a single view reproduces that view's rows (no summation: bit pattern of basis x g)
    one = raster.sph_grad_from_views(3, particles, pos[1][None], gs[1][None]).cpu().numpy()
    assert rel_l2(one, full_ds[1].cpu().numpy()) <= 1e-6


def _wide_angle_scene(model):
    import dataclasses

    base = scenes.scene_c1()
    f = 0.9 * base.width
    if model == "fisheye":
        return dataclasses.replace(base, fx=f, fy=f, fisheye=(0.05, -0.01, 0.002, -0.0003, 0.6))
    a1, a3 = 1.0 / f, 0.04 / f ** 3
    ft = dict(reference_poly=0 if model == "ftheta_bw" else 1, bw=[0.0, a1, 0.0, a3, 0.0, 0.0], fw=[0.0, f, 0.0, -0.04 * f, 0.0, 0.0],
              cde=[1.0, 0.001, -0.002], max_angle=0.6, principal=(base.width / 2.0 - 0.5, base.height / 2.0 - 0.5))
    return dataclasses.replace(base, fx=1.0, fy=1.0, ftheta=ft)


@pytest.mark.parametrize("cam_index,model", [(1, "fisheye"), (4, "fisheye"), (2, "ftheta_bw"), (5, "ftheta_fw")])
def test_fisheye_camera_parity(cam_index, model):
    """OpenCV fisheye (cameraProjections.cuh:120-146) and f-theta (:148-198) sensors with rays of the same camera.  The projections
    call atan2f, which is not correctly rounded on either side (CUDA <= 2 ulp, glibc <= 1 ulp), so the integer artefacts are compared
    per particle instead of bit for bit as a whole: tile counts equal on >= 99.9 % of the particles, depth bits (no atan2f involved)
    exactly equal.  (ftheta_fw: the rays come from the backward polynomial while the projection uses the forward one, which is only
    its low-order inverse -- both sides see the same inconsistency.)"""
    sc = _wide_angle_scene(model)
    c2w = sc.camera(cam_index, 10)
    ref = oracle_frame(sc, c2w, seed=cam_index, pose=tracer_pose(c2w))
    assert ref["pr"].tiles_count.sum() > 500  # (rejections by the valid cone are pinned on the CPU: tests/test_oracle_vs_ref.py)
    tr, g, out, dbg = _run(sc, c2w, ref)
    same = dbg["count"] == ref["pr"].tiles_count
    print(f"[parity] {model} cam{cam_index}: tile counts equal on {same.mean() * 100:.3f} % of the particles")
    assert same.mean() >= 0.999
    assert np.array_equal(dbg["depth"].view(np.uint32)[same & (dbg["count"] > 0)], ref["pr"].depth.view(np.uint32)[same & (dbg["count"] > 0)])
    if same.all():
        assert np.array_equal(dbg["keys"], ref["bn"].sorted_keys) and np.array_equal(dbg["vals"], ref["bn"].sorted_values)
    rgba = torch.cat([out["pred_features"], out["pred_opacity"]], -1)[0].detach().cpu().numpy()
    P = rgba.shape[0] * rgba.shape[1]
    mean_e, max_e, bad = image_error_report(f"{model} cam{cam_index} rgba", rgba, ref["rgba"])
    assert mean_e <= 1e-5 and bad <= max(3, int(2e-4 * P)) + 16 * int((~same).sum())
    if same.all():
        dp = ref["dp"]
        errs = dict(pos=rel_l2(g.positions.grad.cpu().numpy(), dp[:, 0:3]), dns=rel_l2(g._dns.grad.cpu().numpy(), dp[:, 3:4]),
                    quat=rel_l2(g._rot.grad.cpu().numpy(), dp[:, 4:8]), scl=rel_l2(g._scl.grad.cpu().numpy(), dp[:, 8:11]),
                    sph=rel_l2(g._sph.grad.cpu().numpy(), ref["ds"]))
        print("[parity] %s cam%d gradient rel-L2:" % (model, cam_index), {k: f"{v:.2e}" for k, v in errs.items()})
        assert max(errs.values()) <= 1e-3


@pytest.mark.parametrize("kind", [1, 4])
def test_rolling_shutter_parity(kind):
    """Rolling shutter (projectPointWithShutter, cameraProjections.cuh:218-257; pinned on the CPU by
    test_rolling_shutter_projection_bit_identical): sensor moving between shutter open and close, 5 pose / projection iterations per sigma
    point.  The pose interpolation calls acosf / sinf (not correctly rounded on either side), so tile counts are compared per particle
    (>= 99.9 % equal); the image is rendered with the mid-exposure pose on both sides."""
    import b200_native as nat
    from oracle import gut_oracle as go

    sc = scenes.scene_c1()
    p0 = scenes.pose7_from_c2w(sc.camera(1, 40))
    p1 = scenes.pose7_from_c2w(sc.camera(2, 40))
    cfg = go.default_config()
    ocam = go.make_camera(sc.width, sc.height, sc.fx, sc.fy, sc.cx, sc.cy, p0, p1, rolling_shutter=kind)
    ro, rd = sc.rays()
    pr, bn, rgba_ref, dist_ref, hits_ref = go.forward_all(cfg, ocam, ro, rd, sc.particles, sc.sph, 3)
    glob = go.project(cfg, go.make_camera(sc.width, sc.height, sc.fx, sc.fy, sc.cx, sc.cy, p0, p1), sc.particles, sc.sph, 3)
    assert not np.array_equal(glob.tiles_count, pr.tiles_count)  # the shutter matters for this motion

    ctx = nat.Context(nat.default_config(), 0)
    cam = nat.Camera()
    cam.width, cam.height = sc.width, sc.height
    cam.principal[:] = [sc.cx, sc.cy]
    cam.focal[:] = [sc.fx, sc.fy]
    cam.pose_start[:] = [float(v) for v in p0]
    cam.pose_end[:] = [float(v) for v in p1]
    cam.rolling_shutter = kind
    n, hw = sc.n, sc.width * sc.height
    rgba, dist, hits, vis = (np.zeros((hw, 4), np.float32), np.zeros(hw, np.float32), np.zeros(hw, np.float32), np.zeros(n, np.float32))
    p = lambda a: a.ctypes.data  # noqa: E731
    ro_c, rd_c = np.ascontiguousarray(ro), np.ascontiguousarray(rd)
    ctx.forward_host(cam, n, p(sc.particles), p(sc.sph), 3, p(ro_c), p(rd_c), p(rgba), p(dist), p(hits), p(vis))
    count = ctx.debug_copy(nat.DBG_TILES_COUNT)
    depth = ctx.debug_copy(nat.DBG_DEPTH)
    same = count == pr.tiles_count
    print(f"[parity] rolling shutter {kind}: tile counts equal on {same.mean() * 100:.3f} % of the particles")
    assert same.mean() >= 0.999
    vis_same = same & (count > 0)
    assert np.array_equal(depth.view(np.uint32)[vis_same], pr.depth.view(np.uint32)[vis_same])
    mean_e, max_e, bad = image_error_report(f"rolling shutter {kind} rgba", rgba.reshape(rgba_ref.shape), rgba_ref)
    assert mean_e <= 1e-5 and bad <= max(3, int(2e-4 * hw)) + 16 * int((~same).sum())
    ctx.close()

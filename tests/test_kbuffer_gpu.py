"""GPU parity of the sorted (k-buffer) 3DGUT variant (3dgrut_b200/csrc/gut_render_kbuffer.cu, the walk in kbuffer_walk.cuh, the CANON = false
instantiations of G8 in gut_render.cu) against the oracle's k-buffer forward and backward (oracle/gut_oracle.c:
gut_oracle_render_forward_kbuffer / _backward_kbuffer), through the C ABI's host entry points.

Bars (DESIGN.md section 5, as the unsorted path): tile counts, depth bits, sorted keys and values, ranges and visibility BIT-EXACT (the binning
is shared with K = 0); RGBA / distance mean |diff| <= 1e-5, at most max(3, 2e-4 P) pixels above 1e-4, max <= 2e-2; hit counts equal on
>= 99.9 % of the pixels; gradients rel-L2 <= 1e-3 per tensor.  On the dense frames (tile lists of thousands of entries) the gradient bar is the
yardstick rule of test_gut_headline_parity_gpu.py with the k-buffer oracle in float32 vs float64 on the same lists as the yardstick, and the
image's max |diff| and pixel count follow the same rule (_check_image_dense: only C2 at K = 16 is above the plain bar).  Every case
prints and asserts what it exercises (kbuffer_premises): the longest tile list, rays with more than K accepted hits (the buffer flushes before
the list ends) and rays that stop below min_transmittance at a flush and while the buffer drains."""
import dataclasses

import numpy as np
import pytest

import scenes
from helpers import image_error_report, kbuffer_premises, oracle_camera, rel_l2, tracer_pose
from oracle import gut_oracle as go
from test_gut_off_default_gpu import _check_gradients, _check_image, _check_integers

pytestmark = pytest.mark.gpu  # K = 1 .. 16, kernel degrees 2 / 4
torch = pytest.importorskip("torch")


def native_camera(ocam):
    """The C ABI camera with every field of the oracle's camera (pinhole, fisheye, distortion, rolling shutter)."""
    import b200_native as nat

    cam = nat.Camera()
    for name, _ in nat.Camera._fields_:
        v = getattr(ocam, name)
        if hasattr(v, "__len__"):
            getattr(cam, name)[:] = list(v)
        else:
            setattr(cam, name, v)
    return cam


def kbuffer_oracle(sc, ocam, k, settings, deg, seed, ro=None, rd=None, with_f64=False):
    """The oracle's k-buffer forward + backward on go.default_config() with `settings` applied; with_f64 adds the float64 evaluation on
    the same lists (dp_64, ds_64: the yardstick of the dense frames)."""
    cfg = go.default_config()
    for a, b in settings.items():
        setattr(cfg, a, b)
    if ro is None:
        ro, rd = sc.rays()
    pr = go.project(cfg, ocam, sc.particles, sc.sph, deg)
    bn = go.bin_tiles(cfg, ocam, pr)
    rgba, dist, hits = go.render_forward_kbuffer(cfg, ocam, k, ro, rd, sc.particles, pr, bn)
    rng = np.random.default_rng(seed)
    d_rgba = rng.normal(size=rgba.shape).astype(np.float32)
    d_dist = (0.1 * rng.normal(size=dist.shape)).astype(np.float32)
    dp, ds = go.render_backward_kbuffer(cfg, ocam, k, ro, rd, sc.particles, sc.sph, deg, pr, bn, rgba, dist, d_rgba, d_dist)
    out = dict(cfg=cfg, ro=ro, rd=rd, pr=pr, bn=bn, rgba=rgba, dist=dist, hits=hits, d_rgba=d_rgba, d_dist=d_dist, dp=dp, ds=ds)
    if with_f64:
        r64, d64, _ = go.render_forward_kbuffer(cfg, ocam, k, ro, rd, sc.particles, pr, bn, f64=True)
        out["rgba_64"], out["dist_64"] = r64, d64
        out["dp_64"], out["ds_64"] = go.render_backward_kbuffer(cfg, ocam, k, ro, rd, sc.particles, sc.sph, deg, pr, bn, r64, d64, d_rgba,
                                                                d_dist, f64=True)
    return out


def native_host(sc, ncam, settings, deg, ro, rd, d_rgba, d_dist):
    """Forward + backward through gutb200_forward_host / backward_host with `settings` applied to nat.default_config()."""
    import b200_native as nat

    cfg = nat.default_config()
    for a, b in settings.items():
        setattr(cfg, a, b)
    ctx = nat.Context(cfg, 0)
    n, hw = sc.n, sc.width * sc.height
    rgba, dist, hits, vis = (np.zeros((hw, 4), np.float32), np.zeros(hw, np.float32), np.zeros(hw, np.float32), np.zeros(n, np.float32))
    p = lambda a: a.ctypes.data  # noqa: E731
    ro, rd = np.ascontiguousarray(ro, np.float32), np.ascontiguousarray(rd, np.float32)
    d_rgba, d_dist = np.ascontiguousarray(d_rgba, np.float32), np.ascontiguousarray(d_dist, np.float32)
    ctx.forward_host(ncam, n, p(sc.particles), p(sc.sph), deg, p(ro), p(rd), p(rgba), p(dist), p(hits), p(vis))
    out = {a: ctx.debug_copy(b) for a, b in dict(count=nat.DBG_TILES_COUNT, keys=nat.DBG_SORTED_KEYS, vals=nat.DBG_SORTED_VALUES,
                                                 ranges=nat.DBG_TILE_RANGES, depth=nat.DBG_DEPTH).items()}
    dp, ds = np.zeros((n, 12), np.float32), np.zeros((n, 48), np.float32)
    ctx.backward_host(ncam, n, p(sc.particles), p(sc.sph), deg, p(ro), p(rd), p(rgba), p(d_rgba), p(dist), p(d_dist), p(dp), p(ds))
    ctx.close()
    out.update(rgba=rgba.reshape(sc.height, sc.width, 4), dist=dist.reshape(sc.height, sc.width, 1), hits=hits.reshape(sc.height, sc.width, 1),
               vis=vis, dp=dp, ds=ds)
    return out


def _dense_model(model):
    from test_gut_headline_parity_gpu import _dense

    return _dense(model)


def _frame(name):
    """(scene, oracle camera, dense) of the named frame.  The C1 frames have their Gaussians doubled in size, so that the per-ray hit order
    differs from the depth order of the lists and every ray accepts more than K hits."""
    if name in ("c1", "c1_ragged"):
        sc = scenes.scene_c1() if name == "c1" else scenes.scene_c1(width=75, height=53)
        sc.particles[:, 8:11] *= 2.0
        c2w = sc.camera(3 if name == "c1" else 5, 10)
        return sc, oracle_camera(sc, c2w, tracer_pose(c2w))[0], False
    if name == "dense":
        sc = scenes.scene_c2(n=60_000, width=256, height=256)
    elif name == "c2":  # the workload of the sorted paper configuration: BASELINE configs[1]
        sc = scenes.scene_c2()
        c2w = sc.camera(3, 100)
        return sc, oracle_camera(sc, c2w, tracer_pose(c2w))[0], True
    elif name == "fisheye":
        sc = _dense_model("fisheye")
    elif name == "rolling":  # OpenCV pinhole with every distortion term and a top-to-bottom rolling shutter
        sc = _dense_model("pinhole_distorted")
        p0, p1 = scenes.pose7_from_c2w(sc.camera(1, 40)), scenes.pose7_from_c2w(sc.camera(2, 40))
        ocam = go.make_camera(sc.width, sc.height, sc.fx, sc.fy, sc.cx, sc.cy, p0, p1, rolling_shutter=1)
        ocam.radial[:] = [0.05, -0.01, 0.002, 0.01, 0.0, 0.0]
        ocam.tangential[:] = [0.001, -0.0005]
        ocam.thin_prism[:] = [0.0003, 0.0, -0.0002, 0.0]
        return sc, ocam, True
    else:
        raise ValueError(name)
    c2w = sc.camera(2, 10)
    return sc, oracle_camera(sc, c2w, tracer_pose(c2w))[0], True


def _check_case(frame, k, degree):
    sc, ocam, dense = _frame(frame)
    settings = dict(kernel_degree=degree)
    ref = kbuffer_oracle(sc, ocam, k, settings, 3, seed=k + degree, with_f64=dense)
    label = f"kbuffer {frame} K={k} deg={degree}"
    pre = kbuffer_premises(label, ref["cfg"], ocam, k, ref["ro"], ref["rd"], sc.particles, ref["pr"], ref["bn"], ref["hits"])
    assert pre["over_k"] > 0.05, "too few rays flush their buffer before the list ends"
    assert pre["longest"] > (256 if dense else 32), "the lists must span several 32-entry batches of the walk"
    if frame == "c1" and k > 1:  # (K = 1 drains a single hit)
        assert pre["at_flush"] > 0 and pre["in_drain"] > 0, "rays must stop both at a flush and while the buffer drains"
    if frame == "c1":  # K > 1: the sorted variant really differs from K = 0 on this scene; K = 1 flushes in list order, as K = 0 composites
        base = go.render_forward(ref["cfg"], ocam, ref["ro"], ref["rd"], sc.particles, ref["pr"], ref["bn"])[0]
        diff = float(np.abs(base - ref["rgba"]).max())
        print(f"[kbuffer] {label}: oracle image max |K - unsorted| {diff:.2e}")
        assert diff <= 1e-6 if k == 1 else diff > 1e-3
    got = native_host(sc, native_camera(ocam), dict(settings, k_buffer_size=k), 3, ref["ro"], ref["rd"], ref["d_rgba"], ref["d_dist"])
    if frame in ("fisheye", "rolling"):
        # atan2f / the pose interpolation are not correctly rounded on either side: tile counts compared per particle and the image bar
        # widened by the differing particles, as test_gut_headline_parity_gpu.py does for these camera models
        same = got["count"] == ref["pr"].tiles_count
        print(f"[kbuffer] {label}: tile counts equal on {same.mean() * 100:.4f} % of the particles")
        assert same.mean() >= 0.999
        P = sc.width * sc.height
        mean_e, max_e, bad = image_error_report(f"{label} rgba", got["rgba"], ref["rgba"])
        assert mean_e <= 1e-5 and bad <= max(3, int(2e-4 * P)) + 16 * int((~same).sum())
        if not same.all():
            return
        assert np.array_equal(got["vals"], ref["bn"].sorted_values)
    else:
        _check_integers(label, got, ref)
        if dense:
            _check_image_dense(label, got, ref)
        else:
            _check_image(label, got["rgba"], got["dist"], got["hits"], ref)
    _check_gradients(label, got["dp"], got["ds"], ref)
    assert np.all(got["dp"][:, 11] == 0)


def _check_image_dense(label, got, ref):
    """The image bar with the yardstick rule of the gradients: on a frame where the oracle itself, float32 against float64 on the same lists,
    exceeds the max |diff| or the pixel count of the bar, the bar becomes 1.5 x that spread (printed); the mean bar stays.  With a k-buffer,
    two hits whose distances agree to the last bits can leave the buffer in either order under two valid float32 evaluations, which moves
    the pixel by up to alpha_1 alpha_2 |c_1 - c_2| -- beyond the 2e-2 of an accept flip (C2 at K = 16: max 2.8e-2, 157 pixels)."""
    P = got["rgba"].shape[0] * got["rgba"].shape[1]
    for key, scale in (("rgba", 1.0), ("dist", max(1.0, float(np.abs(ref["dist"]).max())))):
        atol = 1e-4 * scale
        _, y_max, y_bad = image_error_report(f"{label} {key} yardstick (oracle f32 vs f64)", ref[key], ref[key + "_64"], atol=atol)
        mean_e, max_e, bad = image_error_report(f"{label} {key}", got[key], ref[key], atol=atol)
        bad_bar = max(max(3, int(2e-4 * P)), int(1.5 * y_bad))
        max_bar = max(2e-2 * scale, 1.5 * y_max) if key == "rgba" else float("inf")
        print(f"[kbuffer] {label} {key} bar: mean <= {1e-5 * scale:.1e}, max <= {max_bar:.3e}, pixels > {atol:g} <= {bad_bar}")
        assert mean_e <= 1e-5 * scale and max_e <= max_bar and bad <= bad_bar, key
    same = float(np.mean(got["hits"] == ref["hits"]))
    print(f"[kbuffer] {label}: hit counts equal on {same * 100:.4f} % of the pixels (bar 99.9 %)")
    assert same >= 0.999


@pytest.mark.parametrize("k,degree", [(1, 2), (3, 2), (4, 2), (16, 2), (16, 4)])
def test_kbuffer_forward_and_gradients(k, degree):
    """The C1 frame: K = 1 (every new hit flushes the previous one), odd K, and K = 16 = kMaxK."""
    _check_case("c1", k, degree)


@pytest.mark.parametrize("frame,k,degree", [("c1_ragged", 16, 2), ("c1_ragged", 16, 4), ("dense", 4, 2), ("dense", 4, 4), ("dense", 16, 2),
                                            ("dense", 16, 4), ("c2", 16, 2), ("fisheye", 16, 2), ("rolling", 16, 2)])
def test_kbuffer_frames(frame, k, degree):
    """c1_ragged: partial tiles and partially filled warps (75x53).  dense: 60k Gaussians on 256x256, tile lists of thousands of entries.
    c2: 300k Gaussians on 800x800, the workload of configs/paper/3dgut/sorted_*.yaml.  fisheye / rolling: the dense scene through the OpenCV
    fisheye model and through a distorted pinhole with a rolling shutter."""
    _check_case(frame, k, degree)


def test_kbuffer_outputs_prefilled_with_nan_are_all_written():
    """K = 16 through the device-pointer entry points on a ragged frame, every output buffer filled with NaN first: forward, backward and
    backward_compact write every pixel and every gradient row (zeros where nothing is hit), and agree with the host entry points."""
    import b200_native as nat

    sc, ocam, _ = _frame("c1_ragged")
    sc = dataclasses.replace(sc, particles=np.concatenate([sc.particles, sc.particles[:5] + np.array([0, 0, 500] + [0] * 9, np.float32)]),
                             sph=np.concatenate([sc.sph, sc.sph[:5]]))  # five particles far off-screen: their rows must be written too
    cam = native_camera(ocam)
    cfg = nat.default_config()
    cfg.k_buffer_size = 16
    ctx = nat.Context(cfg, 0)
    dev = torch.device("cuda", 0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)  # noqa: E731
    ro, rd = sc.rays()
    particles, sph, tro, trd = t(sc.particles), t(sc.sph), t(ro), t(rd)
    h, w, n = sc.height, sc.width, sc.n
    nan = float("nan")
    rgba, dist, hits = (torch.full((h, w, 4), nan, device=dev), torch.full((h, w, 1), nan, device=dev), torch.full((h, w, 1), nan, device=dev))
    vis = torch.full((n, 1), nan, device=dev)
    s = torch.cuda.current_stream(dev).cuda_stream
    ctx.forward(s, cam, n, particles.data_ptr(), sph.data_ptr(), 3, tro.data_ptr(), trd.data_ptr(), rgba.data_ptr(), dist.data_ptr(),
                hits.data_ptr(), vis.data_ptr())
    torch.cuda.synchronize()
    for a in (rgba, dist, hits, vis):
        assert not torch.isnan(a).any()
    assert float(hits.max()) > 16 and float(vis[-5:].abs().max()) == 0
    rng = np.random.default_rng(4)
    d_rgba, d_dist = t(rng.normal(size=(h, w, 4))), t(0.1 * rng.normal(size=(h, w, 1)))
    dp, ds, dp_c, g = (torch.full((n, 12), nan, device=dev), torch.full((n, 48), nan, device=dev), torch.full((n, 12), nan, device=dev),
                       torch.full((n, 4), nan, device=dev))
    ctx.backward(s, cam, n, particles.data_ptr(), sph.data_ptr(), 3, tro.data_ptr(), trd.data_ptr(), rgba.data_ptr(), d_rgba.data_ptr(),
                 dist.data_ptr(), d_dist.data_ptr(), dp.data_ptr(), ds.data_ptr())
    ctx.backward_compact(s, cam, n, particles.data_ptr(), sph.data_ptr(), 3, tro.data_ptr(), trd.data_ptr(), rgba.data_ptr(), d_rgba.data_ptr(),
                         dist.data_ptr(), d_dist.data_ptr(), dp_c.data_ptr(), g.data_ptr())
    torch.cuda.synchronize()
    for a in (dp, ds, dp_c, g):
        assert not torch.isnan(a).any()
        assert float(a[-5:].abs().max()) == 0
    assert float(dp.abs().max()) > 0 and rel_l2(dp_c.cpu().numpy(), dp.cpu().numpy()) <= 2e-5
    host = native_host(sc, cam, dict(k_buffer_size=16), 3, ro, rd, d_rgba.cpu().numpy(), d_dist.cpu().numpy())
    assert np.array_equal(rgba.cpu().numpy().view(np.uint32), host["rgba"].view(np.uint32))
    assert np.array_equal(hits.cpu().numpy(), host["hits"])
    e = max(rel_l2(dp.cpu().numpy(), host["dp"]), rel_l2(ds.cpu().numpy(), host["ds"]))
    print(f"[kbuffer] NaN-prefilled device path vs host path: image bit-identical, gradients rel-L2 {e:.2e} (float atomics; bar 1e-5)")
    assert e <= 1e-5
    ctx.close()

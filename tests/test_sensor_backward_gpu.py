"""The 3DGUT backward through every non-pinhole sensor the projection takes -- OpenCV pinhole with k1, k2, p1, p2, OpenCV fisheye, f-theta
with either polynomial as the reference, and rolling shutters read out in each of the four directions -- against the oracle on the very
tile lists the GPU walked, for the unsorted render, the k-buffer and NHT features; and one fused training step through each COLMAP sensor.

The projections call atan2f (and the shutter's pose interpolation acosf / sinf), which are not correctly rounded on either side, so the GPU's
lists may differ from the oracle's by a particle here and there.  Each case therefore checks the projection on its own and the render on the
GPU's lists (helpers.gpu_binning):
  * lists: tile counts equal on >= 99.9 % of the particles, depth bits exact where the counts agree, and the projected centre (within
    1e-3 px) and conic and opacity (within 1e-3 relative) of every particle visible on both sides, all but max(2, 0.1 %) of them.  The
    tile counts alone miss a fraction of a pixel; the centres do not;
  * render, on the GPU's lists with the oracle's radiance (helpers.projection_for_lists): image and distance within the bars of
    test_gut_parity_gpu.py, hit counts equal on >= 99.9 % of the pixels, and the five gradient tensors within the yardstick rule of
    test_gut_headline_parity_gpu.py (err <= max(1e-3, 1.5 x the oracle's float32-vs-float64 spread on the same lists) and <= 1e-3 once
    the ten particles of the largest spread are left out).  Nothing is skipped when a tile count differs."""
import math

import numpy as np
import pytest

import helpers
from helpers import SENSORS, check_gradients, gpu_binning, nudged_configs, oracle_on_lists, output_grads, projection_for_lists, sensor_frame
from oracle import gut_oracle as go
from test_gut_off_default_gpu import _check_image

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

PATHS = ("unsorted", "kbuffer8", "nht")


def _gpu_lists(ctx):
    import b200_native as nat

    return dict(count=ctx.debug_copy(nat.DBG_TILES_COUNT), depth=ctx.debug_copy(nat.DBG_DEPTH), proj=ctx.debug_copy(nat.DBG_PROJ),
                bn=gpu_binning(ctx))


def _check_lists(label, got, pr):
    """The GPU's projection against the oracle's, particle by particle."""
    count, proj = got["count"], got["proj"]
    same = count == pr.tiles_count
    both = (count > 0) & (pr.tiles_count > 0)
    d_pos = np.abs(proj[:, 0:2] - pr.proj_pos).max(1)
    conic = pr.conic_opacity
    d_conic = np.abs(proj[:, 4:7] - conic[:, 0:3]).max(1) / np.maximum(np.abs(conic[:, [0, 2]]).max(1), 1e-30)
    d_op = np.abs(proj[:, 7] - conic[:, 3]) / np.maximum(conic[:, 3], 1e-30)
    off = both & ((d_pos > 1e-3) | (d_conic > 1e-3) | (d_op > 1e-3))
    print(f"[sensor] {label}: tile counts equal on {same.mean() * 100:.3f} % of the {len(same)} particles; of the {int(both.sum())} visible "
          f"on both sides, {int(off.sum())} project off the oracle (largest centre difference {d_pos[both].max():.2e} px)")
    assert same.mean() >= 0.999
    ok = same & (count > 0)
    assert np.array_equal(got["depth"].view(np.uint32)[ok], pr.depth.view(np.uint32)[ok])
    assert both.sum() > 500 and off.sum() <= max(2, int(1e-3 * both.sum()))
    assert len(got["bn"].sorted_values) == int(count.astype(np.int64).sum())


def _sh_case(sc, cam, ro, rd, k, d_rgba, d_dist):
    import b200_native as nat

    cfg = nat.default_config()
    cfg.k_buffer_size = k
    ctx = nat.Context(cfg, 0)
    ncam = nat.Camera.from_buffer_copy(bytes(cam))
    n, hw = sc.n, cam.width * cam.height
    rgba, dist, hits, vis = (np.zeros((hw, 4), np.float32), np.zeros(hw, np.float32), np.zeros(hw, np.float32), np.zeros(n, np.float32))
    p = lambda a: a.ctypes.data  # noqa: E731
    ro, rd = np.ascontiguousarray(ro, np.float32), np.ascontiguousarray(rd, np.float32)
    ctx.forward_host(ncam, n, p(sc.particles), p(sc.sph), 3, p(ro), p(rd), p(rgba), p(dist), p(hits), p(vis))
    got = _gpu_lists(ctx)
    dp, ds = np.zeros((n, 12), np.float32), np.zeros((n, 48), np.float32)
    ctx.backward_host(ncam, n, p(sc.particles), p(sc.sph), 3, p(ro), p(rd), p(rgba), p(d_rgba), p(dist), p(d_dist), p(dp), p(ds))
    ctx.close()
    shape = (cam.height, cam.width)
    got.update(rgba=rgba.reshape(*shape, 4), dist=dist.reshape(*shape, 1), hits=hits.reshape(*shape, 1), dp=dp, ds=ds)
    return got


@pytest.mark.parametrize("d_dist", ["random", "zero"])
@pytest.mark.parametrize("path", PATHS)
@pytest.mark.parametrize("sensor", SENSORS)
def test_backward_on_the_gpu_lists(sensor, path, d_dist):
    """d_dist "zero": the backward as training calls it (no loss term reads the distance)."""
    sc, cam, ro, rd = sensor_frame(sensor)
    cfg = go.default_config()
    pr = go.project(cfg, cam, sc.particles, sc.sph, 3)
    label = f"{sensor} {path} d_dist={d_dist}"
    seed = SENSORS.index(sensor)
    if path == "nht":
        from test_nht_render_gpu import _Gpu

        import nht_render_oracle as nro

        feats = np.random.default_rng(seed).uniform(-math.pi / 2, math.pi / 2, (sc.n, 48)).astype(np.float32)
        d_out, dd = output_grads((cam.height, cam.width, nro.NHT_OUT + 1), seed, d_dist)
        g = _Gpu(sc, int(cfg.kernel_degree), cam, feats, False, ro, rd).forward()
        got = _gpu_lists(g.ctx)
        got.update(rgba=g.out.cpu().numpy(), dist=g.dist.cpu().numpy(), hits=g.hits.cpu().numpy())
        got["dp"], got["ds"] = g.backward(d_out, dd)
        _check_lists(label, got, pr)
        pr_g = projection_for_lists(pr, got["count"], cam, sc.particles, sc.sph, 3)
        r64, r32, lo, hi = (nro.frame(c, cam, sc.particles, feats, ro, rd, go, d_out=d_out, d_dist=dd, device="cuda", dtype=dt, pr=pr_g,
                                      bn=got["bn"])
                            for c, dt in ((cfg, torch.float64), (cfg, torch.float32), *((c, torch.float64) for c in nudged_configs(cfg))))
        # the float64 oracle is the reference; its float32 evaluation and its nudged thresholds on the same lists give its spread
        ref = dict(rgba=r64["out"], dist=r64["dist"], hits=r64["hits"], dp=r64["dp"], ds=r64["df"],
                   spreads=[(r["dp"], r["df"]) for r in (r32, lo, hi)])
    else:
        k = 8 if path == "kbuffer8" else 0
        d_rgba, dd = output_grads((cam.height, cam.width, 4), seed, d_dist)
        got = _sh_case(sc, cam, ro, rd, k, d_rgba, dd)
        _check_lists(label, got, pr)
        pr_g = projection_for_lists(pr, got["count"], cam, sc.particles, sc.sph, 3)
        ref = oracle_on_lists(cfg, cam, ro, rd, sc.particles, sc.sph, 3, pr_g, got["bn"], d_rgba, dd, k=k, spreads=True)
    _check_image(label, got["rgba"], got["dist"], got["hits"], ref)
    check_gradients(label, got["dp"], got["ds"], (ref["dp"], ref["ds"]), ref["spreads"])
    assert np.abs(got["dp"][:, 0:11]).max() > 0 and np.abs(got["ds"]).max() > 0
    assert np.all(got["dp"][:, 11] == 0)


# ---------------------------------------------------------------------------------------------------------------------------------
# one fused training step through each COLMAP sensor


def _with_dataset_views(hz, sensor):
    """Point a training-step harness (C1, 96x96, six orbit views) at a COLMAP `sensor`, its rays, sensor and poses built by scene_data from
    the camera's COLMAP parameters, as the trainer builds a view."""
    import scene_data

    model, params = helpers.colmap_sensor(sensor, hz.W, hz.H, hz.sc.fx)
    cam = scene_data.colmap_camera(model, params, hz.W, hz.H, 1).to(hz.dev)
    split = scene_data.Split([cam], [0] * 6, np.stack([hz.sc.camera(i, 6) for i in range(6)]), [f"{i}.png" for i in range(6)])
    views = [split.view(i) for i in range(6)]
    hz.rays_o, hz.rays_d, hz.sensor = views[0][:3]
    hz.views = [v[3] for v in views]
    return hz


@pytest.mark.parametrize("features", ["sh", "nht"])
@pytest.mark.parametrize("sensor", ["opencv", "fisheye"])
def test_training_step_matches_autograd(sensor, features):
    """test_loss_terms_step_gpu.py::test_one_step_matches_autograd (SH, random background, mask, regularisers) and
    test_nht_train_step_gpu.py::test_one_step_matches_autograd (NHT, white background, mask, regularisers) with a distorted or fisheye
    camera: the Adam first moment after one fused step against autograd through Tracer.render, with those tests' bars."""
    if features == "sh":
        from test_loss_terms_step_gpu import _Harness, _step_against_autograd

        hz = _with_dataset_views(_Harness("gut"), sensor)
        errs, got_loss, want_loss = _step_against_autograd(hz, "random", True, 0.01, 0.02)
        floor, _, _ = _step_against_autograd(hz, "black", False, 0.0, 0.0)
        assert abs(got_loss - want_loss) <= 1e-5, (got_loss, want_loss)
    else:
        from test_nht_train_step_gpu import _Harness, _step_against_autograd

        hz = _with_dataset_views(_Harness("gut"), sensor)
        errs, floor, got_loss, want_loss = _step_against_autograd(hz, True)
        assert abs(got_loss - want_loss) <= 1e-5 * max(1.0, abs(want_loss)), (got_loss, want_loss)
    for k, err in errs.items():
        bar = max(1e-5, 2.0 * floor[k])
        print(f"[sensor step] {sensor} {features} {k}: exp_avg / (1 - b1) vs autograd rel-L2 {err:.2e} (bar {bar:.2e})")
        assert err <= bar, k

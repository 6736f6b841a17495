"""The tile-sample method of tests/test_full_scale_parity_gpu.py, pinned on C1 (ragged 134x118 frame) and the dense 60k frame: the 3DGUT
oracle cut down to a sample of the tiles (helpers.restrict_to_tiles: every other tile's list emptied, the particles no kept list names
dropped)
- forwards to the full frame's image, distance and hit counts on the sampled pixels, bit for bit;
- differentiates to the full frame's backward whose output gradients are zero off the sampled pixels: equal within rel-L2 1e-6 at the
  kept particles (the backward sums per-thread float64 accumulators, and OpenMP hands the tiles to threads in a different grouping),
  and every other particle's gradient is exactly zero."""
import functools

import numpy as np
import pytest

import scenes
from helpers import oracle_camera, output_grads, rel_l2, restrict_to_tiles, tile_pixels, tile_sample
from oracle import gut_oracle as go

SCENES = {
    "c1": lambda: scenes.scene_c1(width=134, height=118),
    "dense60k": lambda: scenes.scene_c2(n=60_000, width=256, height=256),
}
SAMPLE = {"c1": dict(heaviest=4, k=8), "dense60k": dict(heaviest=16, k=48)}


@functools.lru_cache(maxsize=None)
def _frame(name):
    sc = SCENES[name]()
    c2w = sc.camera(2, 10)
    cfg = go.default_config()
    cam, _ = oracle_camera(sc, c2w)
    ro, rd = sc.rays()
    pr, bn, rgba, dist, hits = go.forward_all(cfg, cam, ro, rd, sc.particles, sc.sph, sc.sph_degree)
    tiles = tile_sample(bn.ranges, sc.height, sc.width, seed=3, **SAMPLE[name])
    gx, gy = (sc.width + 15) // 16, (sc.height + 15) // 16
    assert len(tiles) < gx * gy, "a sample, not the whole frame"
    return sc, cfg, cam, ro, rd, pr, bn, (rgba, dist, hits), tiles


@pytest.mark.parametrize("name", list(SCENES))
def test_cut_forward_is_the_full_frame_on_the_sampled_tiles(name):
    sc, cfg, cam, ro, rd, pr, bn, full, tiles = _frame(name)
    rows, particles, sph, spr, sbn = restrict_to_tiles(sc.particles, sc.sph, pr, bn, tiles)
    assert 0 < len(rows) < sc.n
    cut = go.render_forward(cfg, cam, ro, rd, particles, spr, sbn)
    on = tile_pixels(tiles, sc.height, sc.width)
    assert full[2][on].sum() > 0 and full[2][~on].sum() > 0  # the sample is hit, and so is the rest of the frame
    for what, a, b in zip(("rgba", "dist", "hits"), full, cut):
        assert np.array_equal(a[on].view(np.uint32), b[on].view(np.uint32)), what
        assert not b[~on].any(), what  # nothing is drawn off the sample


@pytest.mark.parametrize("d_dist", ["random", "zero"])
@pytest.mark.parametrize("name", list(SCENES))
def test_cut_backward_is_the_masked_full_frame_backward(name, d_dist):
    sc, cfg, cam, ro, rd, pr, bn, (rgba, dist, _), tiles = _frame(name)
    on = tile_pixels(tiles, sc.height, sc.width)[..., None]
    d_rgba, dd = output_grads(rgba.shape, seed=4, d_dist=d_dist)
    d_rgba, dd = d_rgba * on, dd * on
    rows, particles, sph, spr, sbn = restrict_to_tiles(sc.particles, sc.sph, pr, bn, tiles)
    for f64 in (False, True):
        dp, ds = go.render_backward(cfg, cam, ro, rd, sc.particles, sc.sph, sc.sph_degree, pr, bn, rgba, dist, d_rgba, dd, f64=f64)
        cp, cs = go.render_backward(cfg, cam, ro, rd, particles, sph, sc.sph_degree, spr, sbn, rgba, dist, d_rgba, dd, f64=f64)
        off = np.ones(sc.n, bool)
        off[rows] = False
        assert not dp[off].any() and not ds[off].any()
        e = max(rel_l2(cp, dp[rows]), rel_l2(cs, ds[rows]))
        print(f"[tile-sample] {name} d_dist={d_dist} f64={f64}: {len(tiles)} tiles, {len(rows)} of {sc.n} particles, cut vs full "
              f"backward rel-L2 {e:.2e}")
        assert np.abs(dp[rows]).max() > 0 and e <= 1e-6

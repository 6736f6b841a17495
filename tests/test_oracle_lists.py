"""The helpers that run the oracle on tile lists made elsewhere (helpers.binning_from_lists, projection_for_lists, oracle_on_lists), pinned
on the CPU: fed the oracle's own lists, they reproduce go.forward_all and go.render_backward bit for bit, and the radiance they supply for
particles the oracle does not count is the one its projection computes.  The GPU tests run them on the GPU's lists
(test_sensor_backward_gpu.py), so that a gradient is compared on the very lists the kernels walked."""
import dataclasses

import numpy as np
import pytest

import helpers
from oracle import gut_oracle as go


@pytest.mark.parametrize("sensor", ["opencv", "fisheye", "ftheta_bw", "rs3"])
@pytest.mark.parametrize("k", [0, 8])
def test_own_lists_through_the_helpers_reproduce_the_oracle(sensor, k):
    sc, cam, ro, rd = helpers.sensor_frame(sensor, 64, 48)
    cfg = go.default_config()
    pr, bn, rgba, dist, hits = go.forward_all(cfg, cam, ro, rd, sc.particles, sc.sph, 3)
    assert len(bn.sorted_values) > 200
    d_rgba, d_dist = helpers.output_grads(rgba.shape, seed=1)
    if k:
        rgba, dist, hits = go.render_forward_kbuffer(cfg, cam, k, ro, rd, sc.particles, pr, bn)
        dp, ds = go.render_backward_kbuffer(cfg, cam, k, ro, rd, sc.particles, sc.sph, 3, pr, bn, rgba, dist, d_rgba, d_dist)
    else:
        dp, ds = go.render_backward(cfg, cam, ro, rd, sc.particles, sc.sph, 3, pr, bn, rgba, dist, d_rgba, d_dist)
    lists = helpers.binning_from_lists(bn.sorted_keys, bn.sorted_values, bn.ranges)
    got = helpers.oracle_on_lists(cfg, cam, ro, rd, sc.particles, sc.sph, 3, helpers.projection_for_lists(pr, pr.tiles_count, cam, sc.particles,
                                                                                                         sc.sph, 3),
                                  lists, d_rgba, d_dist, k=k, with_f64=False)
    for key, want in dict(rgba=rgba, dist=dist, hits=hits, dp=dp, ds=ds).items():
        assert np.array_equal(got[key].view(np.uint32), want.view(np.uint32)), key


def test_radiance_of_particles_only_other_lists_count():
    """A projection whose counts say no tile sees a third of the visible particles (as the oracle's does where the GPU's atan2f put a
    particle on a tile and its own did not): projection_for_lists with the true counts restores their radiance bit for bit."""
    sc, cam, ro, rd = helpers.sensor_frame("fisheye", 64, 48)
    cfg = go.default_config()
    pr = go.project(cfg, cam, sc.particles, sc.sph, 3)
    vis = np.flatnonzero(pr.tiles_count > 0)
    hidden = vis[::3]
    assert hidden.size > 50
    counts, rgb = pr.tiles_count.copy(), pr.rgb.copy()
    counts[hidden], rgb[hidden] = 0, 0.0
    got = helpers.projection_for_lists(dataclasses.replace(pr, tiles_count=counts, rgb=rgb), pr.tiles_count, cam, sc.particles, sc.sph, 3)
    assert np.array_equal(got.tiles_count, pr.tiles_count)
    assert np.array_equal(got.rgb.view(np.uint32), pr.rgb.view(np.uint32))

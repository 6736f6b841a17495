"""The ray-sample method of tests/test_grt_headline_parity_gpu.py, pinned on C1 (1k Gaussians, 128x128) for both proxy primitives:
the brute-force 3DGRT oracle treats each ray on its own, so on a seeded sample of the rays
- its forward equals the full-frame forward at those rays bit for bit;
- its backward equals the full-frame backward whose output gradient is zero on every other ray (up to the order of the per-thread
  float64 accumulators, which OpenMP sums in a different grouping);
- the hit lists the NHT oracle composites over are the full frame's lists of those rays."""
import numpy as np
import pytest

import grt_ico_oracle as gio
import scenes
from helpers import ray_sample, rel_l2

torch = pytest.importorskip("torch")
import grt_nht_oracle as gno  # noqa: E402

PRIMS = {"instances": dict(degree=4, clamping=True), "icosahedron": dict(degree=2, clamping=False)}


def _setup(prim):
    sc = scenes.scene_c1(n=1000, seed=42, width=128, height=128)
    c2w = np.asarray(sc.camera(1, 10), np.float32)
    cfg = gio.paper_config(PRIMS[prim]["degree"])
    ro, rd = sc.rays()
    ro, rd = ro[0].reshape(-1, 3), rd[0].reshape(-1, 3)
    idx = ray_sample(sc.height, sc.width, 2048, 9)
    return sc, c2w, cfg, ro, rd, idx, dict(clamping=PRIMS[prim]["clamping"], primitive=prim)


def test_sample_has_the_edge_rays_and_is_sorted():
    idx = ray_sample(822, 1237, 4096, 0)
    assert np.all(np.diff(idx) > 0)
    flat = set(idx.tolist())
    assert all((821 * 1237 + x) in flat for x in range(1237)) and all((y * 1237 + 1236) in flat for y in range(822))
    assert 4096 <= len(idx) <= 4096 + 1237 + 822 - 1
    assert np.array_equal(idx, ray_sample(822, 1237, 4096, 0))


@pytest.mark.parametrize("prim", list(PRIMS))
def test_sampled_forward_is_the_full_frame_at_the_sample(prim):
    sc, c2w, cfg, ro, rd, idx, kw = _setup(prim)
    full = gio.grt_trace(cfg, sc.particles, sc.sph, 3, ro, rd, c2w, **kw)
    part = gio.grt_trace(cfg, sc.particles, sc.sph, 3, ro[idx], rd[idx], c2w, **kw)
    assert full[3].sum() > 4 * sc.width * sc.height  # a scene the rays actually cross
    for name, a, b in zip(("rgb", "alpha", "dist", "hits"), full[:4], part[:4]):
        assert np.array_equal(a[idx].view(np.uint32), b.view(np.uint32)), name
    # the sample's visible particles are among the full frame's
    assert np.all(full[4][part[4] != 0] != 0) and (part[4] != 0).sum() > 0


@pytest.mark.parametrize("prim", list(PRIMS))
def test_masked_full_frame_backward_is_the_sampled_backward(prim):
    sc, c2w, cfg, ro, rd, idx, kw = _setup(prim)
    R = ro.shape[0]
    rgb, alpha, dist, _, _ = gio.grt_trace(cfg, sc.particles, sc.sph, 3, ro, rd, c2w, **kw)
    rng = np.random.default_rng(2)
    g = (rng.normal(size=(len(idx), 3)).astype(np.float32), rng.normal(size=len(idx)).astype(np.float32),
         (0.1 * rng.normal(size=len(idx))).astype(np.float32))
    masked = [np.zeros((R, 3), np.float32), np.zeros(R, np.float32), np.zeros(R, np.float32)]
    for m, v in zip(masked, g):
        m[idx] = v
    dp_full, ds_full = gio.grt_trace_bwd(cfg, sc.particles, sc.sph, 3, ro, rd, c2w, rgb, alpha, dist, *masked, **kw)
    dp, ds = gio.grt_trace_bwd(cfg, sc.particles, sc.sph, 3, ro[idx], rd[idx], c2w, rgb[idx], alpha[idx], dist[idx], *g, **kw)
    assert np.abs(dp).max() > 0 and np.abs(ds).max() > 0
    for name, a, b in (("d_particles", dp_full, dp), ("d_sph", ds_full, ds)):
        err = rel_l2(a, b)
        print(f"[sample] {prim} {name}: masked full frame vs sampled rays rel-L2 {err:.2e}")
        assert err <= 1e-6


@pytest.mark.parametrize("prim", list(PRIMS))
def test_nht_lists_of_the_sample_are_the_full_frame_lists(prim):
    sc, c2w, cfg, ro, rd, idx, kw = _setup(prim)
    full = gno.trace_lists(cfg, sc.particles, ro, rd, c2w, f64=True, **kw)
    part = gno.trace_lists(cfg, sc.particles, ro[idx], rd[idx], c2w, f64=True, **kw)
    assert part["count"].max() > 8
    assert np.array_equal(full["count"][idx], part["count"]) and np.array_equal(full["last"][idx], part["last"])
    L = part["pid"].shape[1]
    assert np.all(full["count"][idx] <= L)
    for k in ("pid", "key", "alpha", "depth"):
        assert np.array_equal(full[k][idx][:, :L], part[k]), k

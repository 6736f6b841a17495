"""The binning stages between `project` and `render` (gut_binning.cu): the shared-memory and the L2 path of the per-tile sort, the
grid-wide tile scan, and the buffers a context reuses from frame to frame (grow-only key buffers, per-tile counters, hit words).

Every sorted list must equal the reference's order, (depth bits, particle index) ascending, whichever path sorted it, and a context
that has rendered other frames before must give exactly what a fresh context gives."""
import numpy as np
import pytest

import scenes
from helpers import rel_l2, tracer_pose

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

STAGE_KEYS = 4096  # tile lists up to this length are sorted in shared memory (kStageKeys, gut_binning.cu)


def _camera(sc, pose):
    import b200_native as nat

    cam = nat.Camera()
    cam.width, cam.height = sc.width, sc.height
    cam.principal[:] = [sc.cx, sc.cy]
    cam.focal[:] = [sc.fx, sc.fy]
    cam.pose_start[:] = [float(v) for v in pose]
    cam.pose_end[:] = [float(v) for v in pose]
    return cam


def _frame(ctx, sc, pose, backward=True, seed=5):
    """Forward (+ backward with seeded output gradients) through the host entry points; the frame's outputs and binning artefacts."""
    import b200_native as nat

    cam = _camera(sc, pose)
    n, hw = sc.n, sc.width * sc.height
    rgba, dist, hits, vis = (np.zeros((hw, 4), np.float32), np.zeros(hw, np.float32), np.zeros(hw, np.float32), np.zeros(n, np.float32))
    p = lambda a: a.ctypes.data  # noqa: E731
    ro, rd = sc.rays()
    ro, rd = np.ascontiguousarray(ro), np.ascontiguousarray(rd)
    particles, sph = np.ascontiguousarray(sc.particles), np.ascontiguousarray(sc.sph)
    ctx.forward_host(cam, n, p(particles), p(sph), sc.sph_degree, p(ro), p(rd), p(rgba), p(dist), p(hits), p(vis))
    out = dict(rgba=rgba, dist=dist, hits=hits, vis=vis, ranges=ctx.debug_copy(nat.DBG_TILE_RANGES),
               values=ctx.debug_copy(nat.DBG_SORTED_VALUES), depth=ctx.debug_copy(nat.DBG_DEPTH))
    if backward:
        rng = np.random.default_rng(seed)
        d_rgba = rng.normal(size=(hw, 4)).astype(np.float32)
        d_dist = (0.1 * rng.normal(size=hw)).astype(np.float32)
        dp, ds = np.zeros((n, 12), np.float32), np.zeros((n, 48), np.float32)
        ctx.backward_host(cam, n, p(particles), p(sph), sc.sph_degree, p(ro), p(rd), p(rgba), p(d_rgba), p(dist), p(d_dist), p(dp), p(ds))
        out.update(dp=dp, ds=ds)
    return out


def _check_lists_sorted(out):
    """Every tile's list is (depth bits, particle) ascending, without duplicates; returns the list lengths."""
    ranges, vals, dbits = out["ranges"], out["values"], out["depth"].view(np.uint32)
    lengths = (ranges[:, 1] - ranges[:, 0]).astype(np.int64)
    for t in np.nonzero(lengths)[0]:
        v = vals[ranges[t, 0]:ranges[t, 1]]
        want = v[np.lexsort((v, dbits[v]))]
        assert np.array_equal(v, want), f"tile {t} ({len(v)} entries) is not in (depth bits, particle) order"
        assert len(np.unique(v)) == len(v), f"tile {t} lists a particle twice"
    return lengths


def _assert_same_frame(a, b, what, grads=True):
    for k in ("rgba", "dist", "hits", "vis", "ranges", "values"):
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), f"{what}: {k} differs"
    if grads:  # float atomics: equal up to their order
        assert rel_l2(a["dp"], b["dp"]) <= 1e-4 and rel_l2(a["ds"], b["ds"]) <= 1e-4, what


def _dense_c2(width, height):
    # C2's 300k Gaussians on a quarter of the pixels: the tiles of the object's core hold several times C2's longest lists
    return scenes.scene_c2(width=width, height=height)


def test_both_sort_paths_in_one_frame():
    import b200_native as nat

    sc = _dense_c2(200, 200)
    ctx = nat.Context(nat.default_config(), 0)
    out = _frame(ctx, sc, tracer_pose(sc.camera(3, 10)), backward=False)
    ctx.close()
    lengths = _check_lists_sorted(out)
    print(f"[binning] tiles {len(lengths)}, longest list {lengths.max()}, "
          f"{int(((lengths > 0) & (lengths <= STAGE_KEYS)).sum())} lists in shared memory, {int((lengths > STAGE_KEYS).sum())} through the L2")
    assert (lengths > STAGE_KEYS).any() and ((lengths > 0) & (lengths <= STAGE_KEYS)).any()
    assert int(lengths.sum()) == len(out["values"])


def test_cloned_particles_sort_by_index_on_both_paths():
    """Runs of equal depth bits (cloned Gaussians) are ordered by particle index in shared memory and in the L2 path alike."""
    import b200_native as nat

    base = _dense_c2(200, 200)
    rng = np.random.default_rng(3)
    pick = rng.choice(base.n, 20_000, replace=False)
    particles = np.concatenate([base.particles, base.particles[pick]])
    sph = np.concatenate([base.sph, base.sph[pick]])
    perm = rng.permutation(len(particles))  # clones spread over the index range
    sc = scenes.Scene(base.name, base.width, base.height, base.fx, base.fy, particles[perm], sph[perm], base.sph_degree, base.camera_radius)
    ctx = nat.Context(nat.default_config(), 0)
    out = _frame(ctx, sc, tracer_pose(sc.camera(3, 10)), backward=False)
    ctx.close()
    lengths = _check_lists_sorted(out)
    assert (lengths > STAGE_KEYS).any() and ((lengths > 0) & (lengths <= STAGE_KEYS)).any()


def test_scene_growth_past_the_headroom_regrows_and_matches_a_fresh_context():
    """A frame whose lists exceed the key buffers (grown with 12.5 % head-room) is binned again after the buffers grew."""
    import b200_native as nat

    full = _dense_c2(320, 320)
    small = scenes.Scene(full.name, full.width, full.height, full.fx, full.fy, full.particles[: full.n // 2], full.sph[: full.n // 2],
                         full.sph_degree, full.camera_radius)
    pose = tracer_pose(full.camera(3, 10))
    ctx = nat.Context(nat.default_config(), 0)
    first = _frame(ctx, small, pose)
    i_small = ctx.stats()["I"]
    grown = _frame(ctx, full, pose)
    i_full = ctx.stats()["I"]
    assert i_full > i_small * 1.125 + 64, (i_small, i_full)
    again = _frame(ctx, small, pose)
    ctx.close()
    fresh = nat.Context(nat.default_config(), 0)
    ref_full = _frame(fresh, full, pose)
    fresh.close()
    _check_lists_sorted(grown)
    _assert_same_frame(grown, ref_full, "grown frame vs fresh context")
    _assert_same_frame(again, first, "small frame after the grown one vs before it")


def test_resolution_change_between_frames_leaves_nothing_stale():
    """Per-tile counters and hit words of a frame with more (or fewer) tiles must not leak into the next frame."""
    import b200_native as nat

    def at(w, h):
        sc = _dense_c2(w, h)
        return sc, tracer_pose(sc.camera(6, 10))

    shapes = [(320, 240), (480, 400), (200, 160), (480, 400)]
    ctx = nat.Context(nat.default_config(), 0)
    seen = [_frame(ctx, *at(w, h)) for w, h in shapes]
    ctx.close()
    for (w, h), out in zip(shapes, seen):
        fresh = nat.Context(nat.default_config(), 0)
        ref = _frame(fresh, *at(w, h))
        fresh.close()
        _check_lists_sorted(out)
        _assert_same_frame(out, ref, f"{w}x{h} after other resolutions vs fresh context")


def test_backward_after_early_termination_in_every_tile():
    """Dense opaque scene: every tile's forward stops before the end of its list.  The backward that walks the forward's hit words
    must give the gradients of the backward that re-tests every entry (subtile_culling bit 2 off)."""
    import b200_native as nat

    base = scenes.scene_c2(n=120_000, width=256, height=256)
    particles = base.particles.copy()
    particles[:, 3] = 0.99           # density: opaque
    particles[:, 8:11] *= 6.0        # scales: large, overlapping
    sc = scenes.Scene(base.name, base.width, base.height, base.fx, base.fy, particles, base.sph, base.sph_degree, base.camera_radius)
    pose = tracer_pose(sc.camera(2, 10))
    outs = {}
    for mode in (7, 3):
        cfg = nat.default_config()
        cfg.subtile_culling = mode
        ctx = nat.Context(cfg, 0)
        outs[mode] = _frame(ctx, sc, pose)
        ctx.close()
    a, b = outs[7], outs[3]
    lengths = (a["ranges"][:, 1] - a["ranges"][:, 0]).astype(np.int64)
    alpha = a["rgba"][:, 3]
    # every covered tile ends opaque, with far fewer accepted entries per pixel than the list holds: the forward stopped early
    assert (lengths > 0).sum() > 0.5 * len(lengths)
    assert float(np.median(alpha[alpha > 0])) > 0.99
    assert float(a["hits"].max()) < float(lengths.max())
    for k in ("rgba", "dist", "hits"):
        assert np.array_equal(a[k].view(np.uint32), b[k].view(np.uint32)), k
    e_dp, e_ds = rel_l2(a["dp"], b["dp"]), rel_l2(a["ds"], b["ds"])
    print(f"[hit words] early-terminating scene: gradients with vs without the forward's hit words: rel-L2 {e_dp:.2e} / {e_ds:.2e}")
    assert e_dp <= 3e-4 and e_ds <= 3e-4

"""The per-tile sort (gut_binning.cu) at the list shapes its bucket pass has to get right, and the warp-flattened placement of the pairs
(gut_project.cu) against the projection's own tile counts.

A slice of at most 4096 keys is sorted by one counting pass over equal-width depth buckets and a rank inside each bucket; a slice whose
fullest bucket holds too many keys (equal depths, tight clusters) goes through the radix passes instead, and so does every longer slice.
Each case places seeded Gaussians so that every one of them covers exactly one tile, with the depths the case needs, and checks that the
tile's list holds exactly those Gaussians in (depth bits, particle index) order -- the reference's order."""
import numpy as np
import pytest

import scenes
from helpers import tracer_pose

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

STAGE_KEYS = 4096   # kStageKeys, gut_binning.cu: longer lists are sorted through the L2
GRID_X = 8          # tiles per row of the synthetic frames
FX = 200.0


def _camera(sc, pose):
    import b200_native as nat

    cam = nat.Camera()
    cam.width, cam.height = sc.width, sc.height
    cam.principal[:] = [sc.cx, sc.cy]
    cam.focal[:] = [sc.fx, sc.fy]
    cam.pose_start[:] = [float(v) for v in pose]
    cam.pose_end[:] = [float(v) for v in pose]
    return cam


def _tile_scene(lists, seed=0):
    """One tile per entry of `lists` (camera-space depths z of its Gaussians), row-major on a GRID_X-wide grid.  Every Gaussian sits on
    the ray through its tile's centre pixel with a footprint of about one pixel, so it lands in its tile only.  Returns the scene, the
    camera pose and, per tile, the indices of its Gaussians; the particles are shuffled so that a tile's indices are spread out."""
    rng = np.random.default_rng(seed)
    gy = (len(lists) + GRID_X - 1) // GRID_X
    width, height = 16 * GRID_X, 16 * gy
    pos, owner = [], []
    for t, z in enumerate(lists):
        z = np.asarray(z, np.float64)
        u, v = 16 * (t % GRID_X) + 8.5, 16 * (t // GRID_X) + 8.5   # the tile's centre in the projection's pixel convention
        pos.append(np.stack([(u - width / 2.0) * z / FX, (v - height / 2.0) * z / FX, z], 1))
        owner.append(np.full(len(z), t))
    pos, owner = np.concatenate(pos), np.concatenate(owner)
    n = len(pos)
    scl = np.repeat((pos[:, 2] / FX)[:, None], 3, 1)   # about one pixel
    quat = np.tile([1.0, 0.0, 0.0, 0.0], (n, 1))
    particles = scenes._pack(pos, np.full(n, 0.9), quat, scl)
    sph = scenes._sph(rng, n, 0.2, 0.8, 0.1)
    perm = rng.permutation(n)
    particles, sph, owner = particles[perm], sph[perm], owner[perm]
    sc = scenes.Scene("tile_sort_cases", width, height, FX, FX, particles, sph, 3, 1.0)
    members = [np.nonzero(owner == t)[0].astype(np.uint32) for t in range(len(lists))]
    return sc, tracer_pose(np.eye(4)), members


def _bin(ctx, sc, pose):
    """Forward through the host entry points; the frame's tile ranges, sorted values, depths and per-particle tile counts."""
    import b200_native as nat

    cam = _camera(sc, pose)
    n, hw = sc.n, sc.width * sc.height
    rgba, dist, hits, vis = (np.zeros((hw, 4), np.float32), np.zeros(hw, np.float32), np.zeros(hw, np.float32), np.zeros(n, np.float32))
    p = lambda a: a.ctypes.data  # noqa: E731
    ro, rd = (np.ascontiguousarray(a) for a in sc.rays())
    particles, sph = np.ascontiguousarray(sc.particles), np.ascontiguousarray(sc.sph)
    ctx.forward_host(cam, n, p(particles), p(sph), sc.sph_degree, p(ro), p(rd), p(rgba), p(dist), p(hits), p(vis))
    return dict(ranges=ctx.debug_copy(nat.DBG_TILE_RANGES).astype(np.int64), values=ctx.debug_copy(nat.DBG_SORTED_VALUES),
                depth=ctx.debug_copy(nat.DBG_DEPTH), counts=ctx.debug_copy(nat.DBG_TILES_COUNT), rgba=rgba, hits=hits)


def _want(ids, dbits):
    return ids[np.lexsort((ids, dbits[ids]))]


def _check_tiles(out, members):
    """Tile t lists exactly members[t], in (depth bits, particle) order; every other tile is empty."""
    ranges, vals, dbits = out["ranges"], out["values"], out["depth"].view(np.uint32)
    for t, ids in enumerate(members):
        got = vals[ranges[t, 0]:ranges[t, 1]]
        assert len(got) == len(ids), f"tile {t}: {len(got)} entries, {len(ids)} Gaussians placed there"
        assert np.array_equal(got, _want(ids, dbits)), f"tile {t} ({len(ids)} entries) is not its Gaussians in (depth bits, particle) order"
    assert int((ranges[len(members):, 1] - ranges[len(members):, 0]).sum()) == 0


def _uniform(rng, k, lo=1.0, hi=10.0):
    return rng.uniform(lo, hi, k)


def _cases():
    rng = np.random.default_rng(11)
    sizes = [1, 31, 32, 33, 2047, 4095, 4096, 4097]
    lists = [_uniform(rng, k) for k in sizes]
    names = [f"{k} keys" for k in sizes]
    lists += [np.full(40, 3.0), np.full(700, 3.0)]                          # equal depths: one bucket, ranked / over-full
    names += ["40 equal depths", "700 equal depths"]
    lists.append(np.concatenate([1.0 + 1e-6 * rng.random(900), 100.0 + 1e-4 * rng.random(900)]))   # two tight clusters far apart
    names.append("two tight clusters")
    lists.append(np.exp(rng.uniform(np.log(0.3), np.log(1.0e4), 3000)))   # depths over more than four decades
    names.append("wide depth range")
    for k in (1500, 2600):                                                 # every depth twice: clones, broken by index (both paths)
        z = _uniform(rng, k)
        lists.append(np.concatenate([z, z]))
        names.append(f"{k} cloned pairs")
    return lists, names


def test_sorted_lists_at_every_list_shape():
    import b200_native as nat

    lists, names = _cases()
    sc, pose, members = _tile_scene(lists)
    ctx = nat.Context(nat.default_config(), 0)
    out = _bin(ctx, sc, pose)
    ctx.close()
    lengths = out["ranges"][:, 1] - out["ranges"][:, 0]
    print("[tile sort] " + ", ".join(f"{nm}: {int(lengths[t])}" for t, nm in enumerate(names)))
    assert (lengths[: len(lists)] > STAGE_KEYS).sum() == 2 and lengths[7] == STAGE_KEYS + 1   # 4097 keys and 2 x 2600 take the L2 path
    _check_tiles(out, members)
    assert np.array_equal(out["counts"], np.ones(sc.n, np.uint32))


def test_global_z_order_sorts_by_view_depth():
    """Under global_z_order the key is the view-space z (positive: the projection drops everything closer than 0.2)."""
    import b200_native as nat

    lists, _ = _cases()
    sc, pose, members = _tile_scene(lists, seed=1)
    cfg = nat.default_config()
    cfg.global_z_order = 1
    ctx = nat.Context(cfg, 0)
    out = _bin(ctx, sc, pose)
    ctx.close()
    assert (out["depth"] > 0.0).all()
    _check_tiles(out, members)


def test_context_that_rendered_other_frames_matches_a_fresh_one():
    import b200_native as nat

    lists, _ = _cases()
    sc, pose, members = _tile_scene(lists, seed=2)
    ctx = nat.Context(nat.default_config(), 0)
    other = scenes.scene_c2(n=100_000, width=320, height=240)
    _bin(ctx, other, tracer_pose(other.camera(4, 10)))
    sc_b, pose_b, _ = _tile_scene(_cases()[0][::-1], seed=3)
    _bin(ctx, sc_b, pose_b)
    used = _bin(ctx, sc, pose)
    ctx.close()
    fresh_ctx = nat.Context(nat.default_config(), 0)
    fresh = _bin(fresh_ctx, sc, pose)
    fresh_ctx.close()
    _check_tiles(used, members)
    for k in ("ranges", "values", "rgba", "hits"):
        assert np.array_equal(used[k].view(np.uint32), fresh[k].view(np.uint32)), k


def test_every_projected_pair_is_placed_once():
    """Dense C2 Gaussians with footprints of one to hundreds of tiles: every particle appears in exactly as many tile lists as the
    projection counted for it (the placement's culling test must agree with the projection's, cell for cell), once per tile."""
    import b200_native as nat

    sc = scenes.scene_c2(width=200, height=200)
    particles = sc.particles.copy()
    particles[::97, 8:11] *= 40.0   # some footprints far larger than a warp's 32 cells
    sc = scenes.Scene(sc.name, sc.width, sc.height, sc.fx, sc.fy, particles, sc.sph, sc.sph_degree, sc.camera_radius)
    ctx = nat.Context(nat.default_config(), 0)
    out = _bin(ctx, sc, tracer_pose(sc.camera(3, 10)))
    ctx.close()
    ranges, vals, counts, dbits = out["ranges"], out["values"], out["counts"], out["depth"].view(np.uint32)
    n = sc.n
    assert counts.max() > 32
    assert np.array_equal(np.bincount(vals, minlength=n), counts.astype(np.int64))
    for t in np.nonzero(ranges[:, 1] > ranges[:, 0])[0]:
        v = vals[ranges[t, 0]:ranges[t, 1]]
        assert np.array_equal(v, _want(np.unique(v), dbits)), f"tile {t}"

"""Oracle parity AT FULL SCALE: the C3 workload (scenes.scene_c3(): 6M Gaussians at 1237x822, bench.py's configs[2], the one the 1 -> 8
GPU scaling curve is named on) through 3DGUT, and C5 (scenes.scene_c5(): the same generator at 5M) through 3DGRT, camera rays and the
C5_MIRROR reflections of the hybrid.  The headline tests (test_gut_headline_parity_gpu.py, test_grt_headline_parity_gpu.py) stop at 400k
Gaussians, where no tile list is longer than the shared-memory sort's 4096 keys; at C3 three quarters of the tiles are, the render and
backward kernels walk tens of staged batches per tile and the key buffers grow to ~2.8e7 entries.  Also here, small and cheap: an LBVH
driven to its deepest shape (the traversal stack), and the view-parallel SH gradient rebuilt from 32 and 64 views at 6M particles.

3DGUT: the integer artefacts of the WHOLE frame (tile counts, depth bits, sorted keys and values, tile ranges, visibility, I and V)
bit-exact against the oracle's projection and binning.  The oracle's render and backward cost O(pixels x list length), so they run on a
sample of the tiles (helpers.tile_sample: the 16 heaviest lists, the ragged last row and column, 48 seeded others) over a frame cut down to
it (helpers.restrict_to_tiles, pinned by tests/test_oracle_tile_sample.py); the GPU renders and differentiates the whole frame, with the
output gradients zero off the sampled pixels.  Bars as test_gut_headline_parity_gpu.py: images and distances on the sampled pixels, hit
counts equal on >= 99.9 % of them, per gradient tensor err <= max(1e-3, 1.5 x yardstick) (yardstick = the oracle in fp32 vs fp64 on the
same lists) and err <= 1e-3 once the ten particles with the largest yardstick error are removed.

3DGRT: the brute-force oracle is O(N) per ray; at 5M Gaussians it needs ~1 core-second per ray and pass, so RAYS_5M rays per frame (sized
to the host's cores) plus a strided sample of the last row and column.  Bars, ray sampling and the zero output gradient off the sample are
those of test_grt_headline_parity_gpu.py."""
import os
import time

import numpy as np
import pytest

import scenes
from helpers import (image_error_report, oracle_camera, output_grads, rel_l2, restrict_to_tiles, tile_pixels, tile_sample,
                     tracer_pose)
from oracle import gut_oracle as go

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import grt_ico_oracle as gio  # noqa: E402
from test_grt_headline_parity_gpu import _check_outputs, _finite, _Frame, _Gpu, _sh_oracle, _split  # noqa: E402
from test_gut_headline_parity_gpu import _native_camera  # noqa: E402

CORES = len(os.sched_getaffinity(0))
C3_CAMERAS = (1, 6)  # of the 10-camera orbit
RAYS_5M = min(1024, 16 * CORES)  # sampled rays per 5M-Gaussian 3DGRT frame: ~2 to 3 minutes of oracle time on any core count
EDGE_RAYS = 16                   # of the last row, and of the last column
GRADS = ("pos", "dns", "quat", "scl", "feat")


@pytest.fixture(scope="module")
def c3():
    t0 = time.perf_counter()
    sc = scenes.scene_c3()
    print(f"\n[full-scale] C3: {sc.n} Gaussians at {sc.width}x{sc.height}, generated in {time.perf_counter() - t0:.1f} s")
    return sc


@pytest.fixture(scope="module")
def c5():
    t0 = time.perf_counter()
    sc = scenes.scene_c5()
    print(f"\n[full-scale] C5: {sc.n} Gaussians at {sc.width}x{sc.height}, generated in {time.perf_counter() - t0:.1f} s")
    return sc


def _check_grads(label, got, ref, other):
    """got / ref / other: dicts of the five gradient tensors (GPU, oracle fp32, oracle fp64) over the same particles."""
    fmt = lambda d: {k: f"{v:.2e}" for k, v in d.items()}  # noqa: E731
    errs = {k: rel_l2(got[k], ref[k]) for k in GRADS}
    yard = {k: rel_l2(ref[k], other[k]) for k in GRADS}
    n = ref["pos"].shape[0]
    e2 = np.zeros(n)
    for k in GRADS:
        a, b = np.asarray(ref[k], np.float64).reshape(n, -1), np.asarray(other[k], np.float64).reshape(n, -1)
        e2 += ((a - b) ** 2).sum(1) / max(float((b ** 2).sum()), 1e-300)
    keep = np.ones(n, bool)
    keep[np.argsort(-e2)[:10]] = False
    robust = {k: rel_l2(got[k][keep], ref[k][keep]) for k in GRADS}
    print(f"[full-scale] {label} gradient rel-L2 vs oracle:", fmt(errs))
    print(f"[full-scale] {label} yardstick (oracle fp32 vs fp64, same lists):", fmt(yard))
    print(f"[full-scale] {label} gradient rel-L2 without the oracle's 10 flip particles:", fmt(robust))
    for k in GRADS:
        assert errs[k] <= max(1e-3, 1.5 * yard[k]), (k, errs[k], yard[k])
        assert robust[k] <= 1e-3, (k, robust[k])


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. 3DGUT on C3 at 6M


def _gut_forward(ctx, cam, sc, ro, rd):
    hw, p = sc.width * sc.height, (lambda a: a.ctypes.data)
    out = dict(rgba=np.zeros((hw, 4), np.float32), dist=np.zeros(hw, np.float32), hits=np.zeros(hw, np.float32),
               vis=np.zeros(sc.n, np.float32))
    before = ctx.launch_count()
    ctx.forward_host(cam, sc.n, p(sc.particles), p(sc.sph), sc.sph_degree, p(ro), p(rd), p(out["rgba"]), p(out["dist"]), p(out["hits"]),
                     p(out["vis"]))
    out["launches"] = ctx.launch_count() - before
    return out


def _gut_integers(ctx):
    import b200_native as nat

    return dict(count=ctx.debug_copy(nat.DBG_TILES_COUNT), depth=ctx.debug_copy(nat.DBG_DEPTH).view(np.uint32),
                keys=ctx.debug_copy(nat.DBG_SORTED_KEYS), values=ctx.debug_copy(nat.DBG_SORTED_VALUES),
                ranges=ctx.debug_copy(nat.DBG_TILE_RANGES), stats=ctx.stats())


@pytest.mark.parametrize("cam_index", C3_CAMERAS)
def test_c3_full_scale_matches_the_oracle(c3, cam_index):
    """C3, one orbit camera: whole-frame integer artefacts bit-exact; image, distance, hit counts and the backward (random d_dist, and
    d_dist = 0 as every training step calls it) on the sampled tiles."""
    import b200_native as nat

    sc, label = c3, f"c3 cam{cam_index}"
    c2w = sc.camera(cam_index, 10)
    pose = tracer_pose(c2w)
    cfg = go.default_config()
    ocam, _ = oracle_camera(sc, c2w, pose)
    ro, rd = (np.ascontiguousarray(a) for a in sc.rays())
    t0 = time.perf_counter()
    pr = go.project(cfg, ocam, sc.particles, sc.sph, sc.sph_degree)
    t1 = time.perf_counter()
    bn = go.bin_tiles(cfg, ocam, pr)
    t2 = time.perf_counter()
    lens = bn.ranges[:, 1].astype(np.int64) - bn.ranges[:, 0]
    tiles = tile_sample(bn.ranges, sc.height, sc.width, seed=cam_index)
    long_tiles = int((lens > 4096).sum())
    print(f"\n[full-scale] {label}: I={len(bn.sorted_keys)} V={int((pr.tiles_count > 0).sum())} longest tile list {int(lens.max())} "
          f"(batches of 256: {int(np.ceil(lens.max() / 256))}), {long_tiles} of {len(lens)} tiles over 4096 keys; oracle projection "
          f"{t1 - t0:.1f} s, binning {t2 - t1:.1f} s ({CORES} cores)")
    s = lens[tiles]
    print(f"[full-scale] {label}: {len(tiles)} sampled tiles, {int((s > 4096).sum())} of them over 4096 keys, "
          f"{int(((s > 0) & (s <= 4096)).sum())} non-empty at most 4096")
    assert long_tiles >= 2500 and lens.max() >= 12_000
    assert (s > 4096).any() and ((s > 0) & (s <= 4096)).any(), "the sample takes both sort paths"

    ctx = nat.Context(nat.default_config(), 0)
    cam = _native_camera(sc, pose)
    got = _gut_forward(ctx, cam, sc, ro, rd)
    gi = _gut_integers(ctx)
    assert np.array_equal(gi["count"], pr.tiles_count)
    assert np.array_equal(gi["depth"], pr.depth.view(np.uint32))
    assert np.array_equal(gi["keys"], bn.sorted_keys)
    assert np.array_equal(gi["values"], bn.sorted_values)
    assert np.array_equal(gi["ranges"], bn.ranges)
    assert np.array_equal(got["vis"].view(np.int32) != 0, pr.visibility != 0)
    assert gi["stats"]["I"] == len(bn.sorted_keys) and gi["stats"]["V"] == int((pr.tiles_count > 0).sum())
    del gi

    t0 = time.perf_counter()
    rows, particles, sph, spr, sbn = restrict_to_tiles(sc.particles, sc.sph, pr, bn, tiles)
    del bn
    rgba, dist, hits = go.render_forward(cfg, ocam, ro, rd, particles, spr, sbn)
    rgba64, dist64, _ = go.render_forward(cfg, ocam, ro, rd, particles, spr, sbn, f64=True)
    on = tile_pixels(tiles, sc.height, sc.width)
    H, W, P = sc.height, sc.width, int(on.sum())
    mean_e, max_e, bad = image_error_report(f"{label} rgba ({P} sampled pixels)", got["rgba"].reshape(H, W, 4)[on][:, None], rgba[on][:, None])
    assert mean_e <= 1e-5 and max_e <= 2e-2 and bad <= max(3, int(2e-4 * P))
    dscale = max(1.0, float(np.abs(dist[on]).max()))
    mean_e, max_e, bad = image_error_report(f"{label} dist", got["dist"].reshape(H, W, 1)[on][:, None], dist[on][:, None], atol=1e-4 * dscale)
    assert mean_e <= 1e-5 * dscale and bad <= max(3, int(2e-4 * P))
    same_hits = float(np.mean(got["hits"].reshape(H, W, 1)[on] == hits[on]))
    print(f"[full-scale] {label}: hit counts equal on {same_hits * 100:.4f} % of the sampled pixels, oracle hits per pixel mean "
          f"{float(hits[on].mean()):.1f}")
    assert same_hits >= 0.999

    off = np.ones(sc.n, bool)
    off[rows] = False
    p = lambda a: a.ctypes.data  # noqa: E731
    for mode in ("random", "zero"):
        d_rgba, d_dist = output_grads(rgba.shape, seed=cam_index, d_dist=mode)
        d_rgba, d_dist = np.ascontiguousarray(d_rgba * on[..., None]), np.ascontiguousarray(d_dist * on[..., None])
        dp32, ds32 = go.render_backward(cfg, ocam, ro, rd, particles, sph, sc.sph_degree, spr, sbn, rgba, dist, d_rgba, d_dist)
        dp64, ds64 = go.render_backward(cfg, ocam, ro, rd, particles, sph, sc.sph_degree, spr, sbn, rgba64, dist64, d_rgba, d_dist, f64=True)
        dp, ds = np.zeros((sc.n, 12), np.float32), np.zeros((sc.n, 48), np.float32)
        ctx.backward_host(cam, sc.n, p(sc.particles), p(sc.sph), sc.sph_degree, p(ro), p(rd), p(got["rgba"]), p(d_rgba), p(got["dist"]),
                          p(d_dist), p(dp), p(ds))
        print(f"[full-scale] {label} d_dist={mode}: {len(rows)} particles in the sampled lists")
        assert not dp[off].any() and not ds[off].any(), "a gradient on a particle no sampled pixel reads"
        assert np.all(dp[:, 11] == 0)
        _check_grads(f"{label} d_dist={mode}", _split(dp[rows], ds[rows]), _split(dp32, ds32), _split(dp64, ds64))
    print(f"[full-scale] {label}: oracle render + 2 backwards on the sample, fp32 and fp64: {time.perf_counter() - t0:.1f} s")
    ctx.close()


def test_c3_second_camera_in_a_reused_context_matches_a_fresh_context(c3):
    """Camera B rendered after camera A in the same context (grown key buffers, scratch and tile state left by A) is bit-identical to
    camera B in a fresh context: integer artefacts, image, distance, hit counts and visibility."""
    import b200_native as nat

    sc = c3
    ro, rd = (np.ascontiguousarray(a) for a in sc.rays())
    cams = [_native_camera(sc, tracer_pose(sc.camera(i, 10))) for i in C3_CAMERAS]
    ctx = nat.Context(nat.default_config(), 0)
    a = _gut_forward(ctx, cams[0], sc, ro, rd)
    b = _gut_forward(ctx, cams[1], sc, ro, rd)
    bi = _gut_integers(ctx)
    again = _gut_forward(ctx, cams[1], sc, ro, rd)  # B once more: nothing left to grow
    fresh_ctx = nat.Context(nat.default_config(), 0)
    fresh = _gut_forward(fresh_ctx, cams[1], sc, ro, rd)
    fi = _gut_integers(fresh_ctx)
    print(f"\n[full-scale] c3 reuse: launches per frame A {a['launches']}, B after A {b['launches']}, B again {again['launches']}, B fresh "
          f"{fresh['launches']}; camera A regrew the key buffers: {a['launches'] > again['launches']}, camera B after A: "
          f"{b['launches'] > again['launches']}; I of B {bi['stats']['I']}")
    for k in ("count", "depth", "keys", "values", "ranges"):
        assert np.array_equal(bi[k], fi[k]), k
    assert bi["stats"] == fi["stats"]
    for k in ("rgba", "dist", "hits", "vis"):
        assert np.array_equal(b[k].view(np.uint32), fresh[k].view(np.uint32)), k
        assert np.array_equal(again[k].view(np.uint32), fresh[k].view(np.uint32)), k
    ctx.close()
    fresh_ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. 3DGRT on C5 at 5M


def _ray_sample_5m(height, width, k, seed, among=None):
    """Sorted flat indices: k seeded rays (drawn from `among` when given) plus EDGE_RAYS evenly spaced rays of the last row and of the
    last column, corner included (drawn from `among` as well)."""
    rng = np.random.default_rng(seed)
    pool = np.arange(height * width) if among is None else among
    row = (height - 1) * width + np.linspace(0, width - 1, EDGE_RAYS).round().astype(np.int64)
    col = np.linspace(0, height - 1, EDGE_RAYS).round().astype(np.int64) * width + width - 1
    edge = np.intersect1d(np.concatenate([row, col]), pool)
    return np.unique(np.concatenate([rng.choice(pool, size=k, replace=False), edge]))


def _check_grt_frame(fr):
    ref = _sh_oracle(fr)
    h = ref[""]["hits"]
    print(f"[full-scale] {fr.label}: N={fr.particles.shape[0]}, {len(fr.idx)} rays compared (RAYS_5M={RAYS_5M}, {CORES} cores), oracle "
          f"hits per ray mean {h.mean():.2f} max {int(h.max())}, {100 * np.mean(h > 0):.1f} % of the rays hit; oracle wall time "
          f"{ref['secs']:.1f} s")
    assert np.mean(h > 0) > 0.5
    g = _Gpu(fr)
    g.counters(fr.label)
    got = g.trace()
    _check_outputs(fr.label, got, ref[""], fr.idx)
    dp, ds = g.trace_bwd(fr.idx, *ref["grads_in"])
    _finite(fr.label, dp, ds)
    assert np.all(dp[:, 11] == 0)
    _check_grads(fr.label, _split(dp, ds), ref[""]["grads"], ref["64"]["grads"])
    g.ctx.close()


def test_c5_camera_rays_match_the_oracle(c5):
    """C5 camera 1 of 10: the LBVH over 5M particles, the whole frame traced and differentiated on the GPU."""
    sc = c5
    ro, rd = sc.rays()
    fr = _Frame("c5 cam1", sc.particles, sc.sph, ro[0], rd[0], np.asarray(sc.camera(1, 10), np.float32),
                _ray_sample_5m(sc.height, sc.width, RAYS_5M, 1), 1)
    _check_grt_frame(fr)


def test_c5_mirror_rays_match_the_oracle(c5):
    """The hybrid's secondary rays: C5 camera 1's rays reflected off scenes.C5_MIRROR (hybrid.mirror_rays, world space), traced through
    the same kind of 5M-particle BVH; compared on rays that hit the mirror."""
    import hybrid

    sc = c5
    ro, rd = sc.rays()
    c2w = torch.from_numpy(np.asarray(sc.camera(1, 10), np.float32))[None]
    o, d, hit = hybrid.mirror_rays(torch.from_numpy(ro), torch.from_numpy(rd), c2w, scenes.C5_MIRROR["plane_point"],
                                   scenes.C5_MIRROR["plane_normal"])
    hit = hit.numpy().reshape(-1)
    print(f"\n[full-scale] c5 mirror: {100 * hit.mean():.1f} % of the camera rays hit the mirror")
    assert hit.mean() > 0.5
    fr = _Frame("c5 cam1 mirror", sc.particles, sc.sph, o[0].numpy(), d[0].numpy(), np.eye(4, dtype=np.float32),
                _ray_sample_5m(sc.height, sc.width, RAYS_5M, 2, among=np.flatnonzero(hit)), 2)
    _check_grt_frame(fr)


# ---------------------------------------------------------------------------------------------------------------------------------
# 3. LBVH depth


def _deep_tree_frame():
    """Particles whose Morton codes split ONE bit per tree level.  The morton key quantises the proxy centre to a 1024^3 grid over the
    scene box; two anchor pairs pin that box to 1024 cells a side.  64 particles sit in cell (512, 512, 512), and for each bit j = 8..0 and
    each axis four more sit 2^j cells out along that axis: geometrically shrinking distances towards the cluster, each group one Morton
    bit below the previous one, so the Karras tree descends 27 levels towards the cluster (then 5 more over its 32 leaves, whose equal
    codes are split by index) with a group subtree beside every level.  The 48 x 48 parallel rays come from the low corner along the
    diagonal through the cluster: every ray crosses every group's box, and the subtree towards the cluster is the nearer child at every
    level, so the walk holds one pending group per level on its stack.  All proxies have radius 250 cells; every hit is accepted well above
    min_alpha and no ray falls below min_transmittance, so the oracle accepts every particle near the rays."""
    cfg = go.grt_config()
    dens = 0.03
    probe = np.zeros((1, 12), np.float32)
    probe[0, 3], probe[0, 4], probe[0, 8:11] = dens, 1.0, 1.0
    cell = float(go.grt_proxies(cfg, probe)[0][0, 0]) / 250.0
    rng = np.random.default_rng(12)
    # m copies spaced evenly along the diagonal: inside their cell, and tens of float ulps apart in t along every ray (the k-nearest
    # query resumes strictly beyond the last hit's t, so hits at one float t would be an artefact of the scene)
    along = lambda m: (np.arange(m) / m - 0.5)[:, None] * np.full(3, 0.4)  # noqa: E731
    pos, color = [250.1 + along(2), 773.9 + along(2)], [np.full(2, 0), np.full(2, 1)]
    pos.append(512.3 + 0.75 * along(64))  # the lower half of the cell: apart from the nearest groups along the rays
    color.append(np.full(64, 2))
    for j in range(8, -1, -1):
        for axis in range(3):
            c = np.full(3, 512.5)
            c[axis] += 2.0 ** j
            pos.append(c + 0.25 * along(4) + 0.06 * (axis - 1))  # the three axes' groups meet the diagonal at one t: shifted apart
            color.append(np.full(4, 3 + j))  # one colour per distance: hits that could swap order along a ray look alike
    pos, color = np.concatenate(pos) * cell, np.concatenate(color)
    n = len(pos)
    particles = np.zeros((n, 12), np.float32)
    particles[:, 0:3], particles[:, 3], particles[:, 4], particles[:, 8:11] = pos, dens, 1.0, 1.0
    palette = rng.uniform(0.2, 2.0, (color.max() + 1, 3))
    sph = np.zeros((n, 48), np.float32)
    sph[:, 0:3] = palette[color]
    # parallel rays along +(1,1,1) from 2000 cells before the cluster, through a 40 x 40 cell square around it: every ray sees the
    # particles at the same spacing in t as the central one
    u = np.ones(3) / np.sqrt(3.0)
    e1 = np.array([1.0, -1.0, 0.0]) / np.sqrt(2.0)
    e2 = np.cross(u, e1)
    s = np.linspace(-20.0, 20.0, 48)
    ro = np.full(3, 512.5) - 2000.0 * u + s[:, None, None] * e1 + s[None, :, None] * e2
    rd = np.broadcast_to(u, ro.shape)
    return _Frame("deep LBVH", particles, sph, (ro * cell).astype(np.float32), rd.astype(np.float32), np.eye(4, dtype=np.float32),
                  np.arange(48 * 48), 12)


def test_deepest_lbvh_loses_no_hit():
    """Every hit the brute-force oracle accepts on every ray of the deep-tree scene is found: the traversal stack holds the pending
    subtree of every level (a stack too short for the tree drops subtrees without a signal and shows up here as missing hits)."""
    fr = _deep_tree_frame()
    ro, rd = fr.ro.reshape(-1, 3), fr.rd.reshape(-1, 3)
    t0 = time.perf_counter()
    rgb, alpha, dist, hits, vis = gio.grt_trace(fr.cfg, fr.particles, fr.sph, 3, ro, rd, fr.c2w, clamping=fr.clamping, primitive=fr.prim)
    ref = dict(rgb=rgb, alpha=alpha[:, 0], dist=dist[:, 0], hits=hits[:, 0], vis=vis[:, 0] != 0)
    print(f"\n[full-scale] {fr.label}: N={len(fr.particles)}, {len(ro)} rays, oracle hits per ray min {int(ref['hits'].min())} mean "
          f"{ref['hits'].mean():.1f}, {int(ref['vis'].sum())} particles accepted, final transmittance min {1 - float(alpha.max()):.3f}; "
          f"oracle {time.perf_counter() - t0:.2f} s")
    assert ref["hits"].min() >= 64 and 1 - float(alpha.max()) > 2e-3  # every ray crosses the cluster and none stops early
    g = _Gpu(fr)
    g.counters(fr.label)
    got = g.trace()
    _check_outputs(fr.label, got, ref, fr.idx)
    missing = np.flatnonzero(ref["vis"] & ~got["vis"])
    assert missing.size == 0, f"particles accepted by the oracle and never hit on the GPU: {missing[:20]}"
    g.ctx.close()


# ---------------------------------------------------------------------------------------------------------------------------------
# 4. the view-parallel SH gradient from 32 and 64 views


def _sh_basis64(deg, d):
    """[M, 16] real SH basis of unit directions d [M, 3] in float64, zero beyond (deg + 1)^2 (sh_basis16, hit_math.cuh)."""
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    b = np.zeros((len(d), 16))
    b[:, 0] = 0.28209479177387814
    if deg > 0:
        b[:, 1], b[:, 2], b[:, 3] = -0.4886025119029199 * y, 0.4886025119029199 * z, -0.4886025119029199 * x
    if deg > 1:
        xx, yy, zz = x * x, y * y, z * z
        b[:, 4], b[:, 5] = 1.0925484305920792 * x * y, -1.0925484305920792 * y * z
        b[:, 6] = 0.31539156525252005 * (2 * zz - xx - yy)
        b[:, 7], b[:, 8] = -1.0925484305920792 * x * z, 0.5462742152960396 * (xx - yy)
    if deg > 2:
        b[:, 9] = -0.5900435899266435 * y * (3 * xx - yy)
        b[:, 10] = 2.890611442640554 * x * y * z
        b[:, 11] = -0.4570457994644658 * y * (4 * zz - xx - yy)
        b[:, 12] = 0.3731763325901154 * z * (2 * zz - 3 * xx - 3 * yy)
        b[:, 13] = -0.4570457994644658 * x * (4 * zz - xx - yy)
        b[:, 14] = 1.445305721320277 * z * (xx - yy)
        b[:, 15] = -0.5900435899266435 * x * (xx - 3 * yy)
    return b


@pytest.mark.parametrize("views", [32, 64])
@pytest.mark.parametrize("deg", [3, 1])
def test_sph_grad_from_views_at_full_scale(c3, views, deg):
    """gutb200_sph_grad_from_views over the 6M C3 particles with `views` seeded [N,4] radiance gradients (~30 % of the (view, particle)
    rows exactly zero: the kernel's skip branch) at the C3 orbit's camera positions, against a float64 evaluation on 100k seeded rows and
    the last 256; rel-L2 <= 1e-6, and nothing beyond the (deg + 1)^2 active coefficients."""
    import b200_native as nat

    sc = c3
    n, dev = sc.n, torch.device("cuda", 0)
    vp = np.stack([np.asarray(sc.camera(v, views), np.float32)[:3, 3] for v in range(views)])
    gen = torch.Generator(device=dev).manual_seed(100 * views + deg)
    g_all = torch.randn((views, n, 4), device=dev, generator=gen)
    g_all *= (torch.rand((views, n, 1), device=dev, generator=gen) >= 0.3)
    particles = torch.from_numpy(sc.particles).to(dev)
    d_sph = torch.full((n, 48), float("nan"), device=dev)
    ctx = nat.Context(nat.default_config(), 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    ctx.sph_grad_from_views(stream, n, particles.data_ptr(), deg, vp, g_all.data_ptr(), d_sph.data_ptr())
    torch.cuda.synchronize()
    rows = np.unique(np.concatenate([np.random.default_rng(views + deg).choice(n - 256, 100_000, replace=False), np.arange(n - 256, n)]))
    rows_t = torch.from_numpy(rows).to(dev)
    g = g_all[:, rows_t].cpu().numpy().astype(np.float64)
    got = d_sph[rows_t].cpu().numpy()
    zero = float((g[..., :3] == 0).all(-1).mean())
    t0 = time.perf_counter()
    pos = sc.particles[rows, 0:3].astype(np.float64)
    want = np.zeros((len(rows), 16, 3))
    for v in range(views):
        vec = pos - vp[v].astype(np.float64)
        b = _sh_basis64(deg, vec / np.linalg.norm(vec, axis=1, keepdims=True))
        want += b[:, :, None] * g[v, :, None, 0:3]
    err = rel_l2(got, want.reshape(-1, 48))
    print(f"\n[full-scale] sph_grad_from_views views={views} deg={deg}: {100 * zero:.1f} % zero rows, {len(rows)} rows compared, rel-L2 "
          f"vs float64 {err:.2e} (bar 1e-6); float64 reference {time.perf_counter() - t0:.1f} s")
    assert 0.25 <= zero <= 0.35
    assert np.isfinite(got).all() and err <= 1e-6
    assert np.all(got.reshape(-1, 16, 3)[:, (deg + 1) ** 2:] == 0)
    small = torch.zeros((65, 1000, 4), device=dev)
    with pytest.raises(RuntimeError, match="views 65 out of range"):
        ctx.sph_grad_from_views(stream, 1000, particles.data_ptr(), deg, np.zeros((65, 3), np.float32), small.data_ptr(), d_sph.data_ptr())
    ctx.close()

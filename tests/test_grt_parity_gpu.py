"""GPU parity of the 3DGRT path (LBVH + ordered tracing + adjoint) against the brute-force CPU oracle.

Tolerances (DESIGN.md sections 5, 9): RGB / alpha / distance mean |diff| <= 1e-5, |diff| <= 1e-4 on all but
max(3, 2e-4 * P) rays, max <= 2e-2 (isolated accept-test flips); hit counts equal on >= 99.9 % of rays;
gradients rel-L2 <= 1e-3 per tensor."""
import numpy as np
import pytest

import scenes
from helpers import image_error_report, packet_share, permute_pixels, rel_l2, shuffled_pixels, unpermute_pixels
from oracle import gut_oracle as go

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


class _Gaussians:
    def __init__(self, sc, device):
        p = torch.from_numpy(sc.particles).to(device)
        self.positions = p[:, 0:3].clone().requires_grad_(True)
        self.density = p[:, 3:4].clone().requires_grad_(True)
        self.rotation = p[:, 4:8].clone().requires_grad_(True)
        self.scale = p[:, 8:11].clone().requires_grad_(True)
        self._sph = torch.from_numpy(sc.sph).to(device).requires_grad_(True)
        self.n_active_features = sc.sph_degree
        self.num_gaussians = sc.n
        ident = lambda t: t  # noqa: E731  (parameters here are already post-activation)
        self.rotation_activation = self.scale_activation = self.density_activation = ident

    def get_rotation(self):
        return self.rotation

    def get_scale(self):
        return self.scale

    def get_density(self):
        return self.density

    def get_features(self):
        return self._sph


class _Batch:
    def __init__(self, sc, c2w, device, rays=None):
        ro, rd = sc.rays() if rays is None else rays
        self.rays_ori = torch.from_numpy(ro).to(device)
        self.rays_dir = torch.from_numpy(rd).to(device)
        self.T_to_world = torch.from_numpy(np.asarray(c2w, np.float32))[None].to(device)


@pytest.mark.parametrize("cam_index,size", [(1, (128, 128)), (6, (128, 128)), (3, (75, 53))])
def test_c4_like_forward_and_gradients(cam_index, size):
    """size (75, 53): ragged image -- partially filled 8x4 ray blocks (lanes without a ray take part in the packet votes)."""
    import threedgrt_tracer

    sc = scenes.scene_c1(width=size[0], height=size[1])
    c2w = np.asarray(sc.camera(cam_index, 10), np.float32)
    cfg = go.grt_config()
    ro, rd = sc.rays()
    rgb, alpha, dist, hits, vis = go.grt_trace(cfg, sc.particles, sc.sph, 3, ro[0], rd[0], c2w)
    rng = np.random.default_rng(cam_index)
    d_rgb = rng.normal(size=rgb.shape).astype(np.float32)
    d_alpha = rng.normal(size=alpha.shape).astype(np.float32)
    d_dist = (0.1 * rng.normal(size=alpha.shape)).astype(np.float32)
    dp, ds = go.grt_trace_bwd(cfg, sc.particles, sc.sph, 3, ro[0], rd[0], c2w, rgb, alpha, dist, d_rgb, d_alpha, d_dist)

    dev = torch.device("cuda", 0)
    tr = threedgrt_tracer.Tracer({"render": {"min_transmittance": 0.001}})
    g = _Gaussians(sc, dev)
    tr.build_acc(g, rebuild=True)
    kscl, bb = go.grt_proxies(cfg, sc.particles)
    assert np.allclose(tr.tracer_wrapper.native_context(dev).scene_aabb(), bb, rtol=1e-5, atol=1e-5)
    out = tr.render(g, _Batch(sc, c2w, dev), train=True)
    loss = (out["pred_features"] * torch.from_numpy(d_rgb[None]).to(dev)).sum() + (out["pred_opacity"] * torch.from_numpy(d_alpha[None]).to(dev)).sum() \
        + (out["pred_dist"] * torch.from_numpy(d_dist[None]).to(dev)).sum()
    loss.backward()
    torch.cuda.synchronize()
    P = sc.width * sc.height
    got = torch.cat([out["pred_features"], out["pred_opacity"]], -1)[0].detach().cpu().numpy()
    mean_e, max_e, bad = image_error_report(f"grt cam{cam_index} rgba", got, np.concatenate([rgb, alpha], -1))
    assert mean_e <= 1e-5 and max_e <= 2e-2 and bad <= max(3, int(2e-4 * P))
    mean_e, max_e, bad = image_error_report(f"grt cam{cam_index} dist", out["pred_dist"][0].detach().cpu().numpy(), dist[..., 0:1],
                                            atol=1e-4 * max(1.0, float(np.abs(dist[..., 0]).max())))
    assert mean_e <= 1e-4 and bad <= max(3, int(2e-4 * P))
    assert float(np.mean(out["hits_count"][0].detach().cpu().numpy() == hits)) >= 0.999
    got_vis = out["mog_visibility"].detach().cpu().numpy().view(np.int32).reshape(-1) != 0
    assert np.mean(got_vis == (vis.reshape(-1) != 0)) >= 0.999
    errs = dict(pos=rel_l2(g.positions.grad.cpu().numpy(), dp[:, 0:3]), dns=rel_l2(g.density.grad.cpu().numpy(), dp[:, 3:4]),
                quat=rel_l2(g.rotation.grad.cpu().numpy(), dp[:, 4:8]), scl=rel_l2(g.scale.grad.cpu().numpy(), dp[:, 8:11]),
                sph=rel_l2(g._sph.grad.cpu().numpy(), ds))
    print("[parity] grt cam%d gradient rel-L2:" % cam_index, {k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) <= 1e-3


def test_grt_edge_cases_empty_single_and_missing_rays():
    import b200_native as nat

    dev = torch.device("cuda", 0)
    ctx = nat.GrtContext(nat.grt_default_config(), 0)
    s = torch.cuda.current_stream(dev).cuda_stream
    sc = scenes.scene_c1(n=1, width=32, height=24)
    ro, rd = sc.rays()
    c2w = np.asarray(sc.camera(0, 4), np.float32)
    r2w = np.ascontiguousarray(c2w[:3, :4])
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    tro, trd = t(ro), t(rd)
    R = sc.width * sc.height
    for n in (0, 1):
        parts = sc.particles[:n]
        P = t(parts if n else np.zeros((1, 12), np.float32))
        S = t(sc.sph[:n] if n else np.zeros((1, 48), np.float32))
        # keep the four SoA tensors alive until the build has run (a temporary's block is recycled by the caching allocator as soon
        # as .data_ptr() returns, which would make pos / rot / scl / dns alias)
        soa = [P[:, 0:3].contiguous(), P[:, 4:8].contiguous(), P[:, 8:11].contiguous(), P[:, 3:4].contiguous()]
        ctx.build_bvh(s, n, *[a.data_ptr() for a in soa])
        rgb, alpha, dist, hits, vis = (torch.ones((R, 3), device=dev), torch.ones(R, device=dev), torch.ones((R, 2), device=dev),
                                       torch.ones(R, device=dev), torch.ones(max(n, 1), device=dev))
        ctx.trace(s, n, P.data_ptr(), S.data_ptr(), 3, 1e-3, 1, sc.height, sc.width, tro.data_ptr(), trd.data_ptr(), r2w.ctypes.data,
                  rgb.data_ptr(), alpha.data_ptr(), dist.data_ptr(), hits.data_ptr(), vis.data_ptr())
        torch.cuda.synchronize()
        if n == 0:
            assert float(rgb.abs().max()) == 0 and float(alpha.abs().max()) == 0 and float(hits.max()) == 0
        else:
            ref = go.grt_trace(go.grt_config(), parts, sc.sph[:1], 3, ro[0], rd[0], c2w)
            assert np.abs(rgb.cpu().numpy().reshape(ref[0].shape) - ref[0]).max() <= 1e-4
            assert np.array_equal(hits.cpu().numpy().reshape(ref[3].shape), ref[3])
    ctx.close()


def test_hybrid_primary_raster_plus_traced_secondary():
    """BASELINE config 5: 3DGUT primary + 3DGRT secondary on the same Gaussians; each pass matches its oracle and the
    gradients of the composite reach the parameters through both tracers."""
    import hybrid
    import threedgrt_tracer
    import threedgut_tracer
    from test_gut_parity_gpu import _Batch as GutBatch

    sc = scenes.scene_c1(n=400, width=64, height=48)
    c2w = np.asarray(sc.camera(2, 9), np.float32)
    dev = torch.device("cuda", 0)
    g = _Gaussians(sc, dev)
    g.positions.grad = None
    batch = GutBatch(sc, c2w, dev)
    batch.T_to_world = batch.T_to_world.to(dev)
    gut = threedgut_tracer.Tracer({})
    grt = threedgrt_tracer.Tracer({"render": {"min_transmittance": 0.001}})
    out = hybrid.render_hybrid(gut, grt, g, batch, train=True)
    # secondary pass against the brute-force oracle on the same reflected rays
    sec_o, sec_d, hit = hybrid.mirror_rays(batch.rays_ori, batch.rays_dir, batch.T_to_world, (0.0, 0.0, -1.2), (0.0, 0.0, 1.0))
    ref = go.grt_trace(go.grt_config(), sc.particles, sc.sph, 3, sec_o[0].cpu().numpy(), sec_d[0].cpu().numpy(), np.eye(4, dtype=np.float32))
    mean_e, max_e, bad = image_error_report("hybrid secondary rgb", out["pred_secondary"][0].detach().cpu().numpy(), ref[0])
    assert mean_e <= 1e-5 and max_e <= 2e-2 and bad <= 3
    assert float(hit.float().mean()) > 0.05
    out["pred_features_hybrid"].sum().backward()
    assert g.positions.grad is not None and float(g.positions.grad.abs().sum()) > 0 and torch.isfinite(g._sph.grad).all()


def _grt_frame(sc, c2w, d_out, perm=None):
    """One forward + backward through the Tracer; returns numpy (rgba + dist, hits, grads).  perm: the rays are traced in that pixel
    order (shuffled_pixels), and the image and hits are returned in the camera's order."""
    import threedgrt_tracer

    dev = torch.device("cuda", 0)
    tr = threedgrt_tracer.Tracer({"render": {"min_transmittance": 0.001}})
    g = _Gaussians(sc, dev)
    tr.build_acc(g, rebuild=True)
    rays = None if perm is None else tuple(permute_pixels(a, perm) for a in sc.rays())
    out = tr.render(g, _Batch(sc, c2w, dev, rays), train=True)
    img = torch.cat([out["pred_features"], out["pred_opacity"], out["pred_dist"]], -1)
    (img * torch.from_numpy(d_out if perm is None else permute_pixels(d_out, perm)).to(dev)).sum().backward()
    torch.cuda.synchronize()
    grads = [t.grad.detach().cpu().numpy() for t in (g.positions, g.density, g.rotation, g.scale, g._sph)]
    img, hits = img[0].detach().cpu().numpy(), out["hits_count"][0].detach().cpu().numpy()
    return (img, hits, grads) if perm is None else (unpermute_pixels(img, perm), unpermute_pixels(hits, perm), grads)


@pytest.mark.parametrize("switch,off", [pytest.param("shuffled", None, id="shuffled"), ("GRTB200_HITCAP", "0"), ("GRTB200_HITCAP", "8")])
def test_traversal_variants_give_the_same_image(switch, off, monkeypatch):
    """The walk changes HOW the tree is traversed, not which hits a ray finds: "shuffled" traces the same rays in a seeded pixel order,
    so that every warp fails the coherence vote and takes the per-lane walk where the camera's order takes the packet walk.  The
    hit-list cache changes how the backward finds the forward's hits (HITCAP=0: re-trace like the reference, HITCAP=8: nearly every ray
    overflows its list and takes the re-trace fallback).  The same rays through either variant must give the same image, hit counts and
    gradients."""
    sc = scenes.scene_c2(n=60_000, width=256, height=256)
    c2w = np.asarray(sc.camera(2, 10), np.float32)
    rng = np.random.default_rng(0)
    d_out = rng.normal(size=(1, sc.height, sc.width, 5)).astype(np.float32)
    img1, hits1, g1 = _grt_frame(sc, c2w, d_out)
    if switch == "shuffled":
        perm = shuffled_pixels(sc.height, sc.width)
        ro, rd = sc.rays()
        assert packet_share(sc.particles, sc.sph, c2w, ro, rd) >= 0.9
        assert packet_share(sc.particles, sc.sph, c2w, permute_pixels(ro, perm), permute_pixels(rd, perm)) <= 0.1
        img0, hits0, g0 = _grt_frame(sc, c2w, d_out, perm)
    else:
        monkeypatch.setenv(switch, off)
        img0, hits0, g0 = _grt_frame(sc, c2w, d_out)
    assert hits1.sum() > 0
    # not bit-identical: a hit whose t* lies before its box entry (ray clipping a corner of the proxy) survives or not depending on
    # which node boxes got culled by the shrinking 16th-hit bound -- the same ambiguity OptiX has; hence the standard tolerances
    P = sc.width * sc.height
    print(f"[variants] {switch}: hit counts differ on {(hits1 != hits0).sum()} of {P} rays")
    assert (hits1 != hits0).mean() <= 1e-3
    mean_e, max_e, bad = image_error_report(f"{switch}: image", img1, img0, atol=1e-4)
    assert mean_e <= 1e-6 and max_e <= 2e-2 and bad <= max(3, int(2e-4 * P))
    for name, a, b in zip(("positions", "density", "rotation", "scale", "sph"), g1, g0):
        err = rel_l2(a, b)
        print(f"[variants] {switch}: d_{name} rel-L2 {err:.3e}")
        assert err <= 1e-3


def _raw_trace_vs_oracle(sc, ro, rd, label):
    """Rays straight through the C ABI (identity ray-to-world) against the brute-force oracle."""
    import b200_native as nat

    dev = torch.device("cuda", 0)
    H, W = ro.shape[:2]
    r2w = np.ascontiguousarray(np.eye(4, dtype=np.float32)[:3, :4])
    cfg = go.grt_config()
    rgb_ref, alpha_ref, dist_ref, hits_ref, vis_ref = go.grt_trace(cfg, sc.particles, sc.sph, 3, ro, rd, np.eye(4, dtype=np.float32))
    assert hits_ref.sum() > 100
    ctx = nat.GrtContext(nat.grt_default_config(), 0)
    s = torch.cuda.current_stream(dev).cuda_stream
    P = torch.from_numpy(sc.particles).to(dev)
    S = torch.from_numpy(sc.sph).to(dev)
    soa = [P[:, 0:3].contiguous(), P[:, 4:8].contiguous(), P[:, 8:11].contiguous(), P[:, 3:4].contiguous()]  # named: must outlive the build
    ctx.build_bvh(s, sc.n, *[a.data_ptr() for a in soa])
    R = H * W
    tro, trd = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)
    rgb, alpha, dist, hits, vis = (torch.zeros((R, 3), device=dev), torch.zeros(R, device=dev), torch.zeros((R, 2), device=dev),
                                   torch.zeros(R, device=dev), torch.zeros(sc.n, device=dev))
    ctx.trace(s, sc.n, P.data_ptr(), S.data_ptr(), 3, 1e-3, 1, H, W, tro.data_ptr(), trd.data_ptr(), r2w.ctypes.data, rgb.data_ptr(),
              alpha.data_ptr(), dist.data_ptr(), hits.data_ptr(), vis.data_ptr())
    torch.cuda.synchronize()
    got_hits = hits.cpu().numpy().reshape(hits_ref.shape)
    print(f"[axis] {label}: hits {int(got_hits.sum())} vs oracle {int(hits_ref.sum())}, per-ray agreement {np.mean(got_hits == hits_ref):.5f}")
    assert got_hits.sum() > 100 and float(np.mean(got_hits == hits_ref)) >= 0.999
    mean_e, max_e, bad = image_error_report(label + " rgb", rgb.cpu().numpy().reshape(rgb_ref.shape), rgb_ref)
    assert mean_e <= 1e-5 and bad <= 3
    ctx.close()
    return got_hits, hits_ref


def test_axis_parallel_rays_reach_the_geometry():
    """Rays with exactly zero direction components (orthographic bundles): the inverse direction is infinite there, which the one-FMA
    slab test of the node boxes must survive (it used to produce NaN and cull everything)."""
    sc = scenes.scene_c1()
    H = W = 48
    ys, xs = np.meshgrid(np.linspace(-1.4, 1.4, H, dtype=np.float32), np.linspace(-1.4, 1.4, W, dtype=np.float32), indexing="ij")
    ro = np.stack([xs, ys, np.full_like(xs, -4.0)], -1).astype(np.float32)       # orthographic: origins on a plane,
    rd = np.broadcast_to(np.array([0, 0, 1], np.float32), ro.shape).copy()        # all directions exactly +z
    _raw_trace_vs_oracle(sc, ro, rd, "orthographic bundle")


@pytest.mark.parametrize("axis", [0, 1, 2])
def test_axis_aligned_pinhole_centre_row_and_column(axis):
    """An axis-aligned pinhole camera with an odd resolution: the centre column has d.x == 0, the centre row d.y == 0 and the centre pixel
    both -- ordinary inputs for the reference (OptiX).  Looking along each world axis in turn."""
    sc = scenes.scene_c1()
    H = W = 49
    f = 60.0
    u = (np.arange(W, dtype=np.float32) - (W // 2)) / np.float32(f)
    v = (np.arange(H, dtype=np.float32) - (H // 2)) / np.float32(f)
    vv, uu = np.meshgrid(v, u, indexing="ij")
    d = np.stack([uu, vv, np.ones_like(uu)], -1).astype(np.float32)
    d /= np.linalg.norm(d, axis=-1, keepdims=True)
    d = d.astype(np.float32)
    d[:, W // 2, 0] = 0.0
    d[H // 2, :, 1] = 0.0
    perm = [(0, 1, 2), (2, 0, 1), (1, 2, 0)][axis]  # which world axis the camera looks along
    rd = np.ascontiguousarray(d[..., list(perm)])
    o = np.zeros(3, np.float32)
    o[perm.index(2)] = -4.0
    ro = np.broadcast_to(o, rd.shape).copy()
    assert (rd == 0).sum() >= H + W
    got, ref = _raw_trace_vs_oracle(sc, ro, rd, f"axis-aligned pinhole (look axis {perm.index(2)})")
    # the degenerate rows / columns themselves, not just the bulk
    assert np.array_equal(got.reshape(H, W)[H // 2], ref.reshape(H, W)[H // 2]) or np.mean(got.reshape(H, W)[H // 2] == ref.reshape(H, W)[H // 2]) >= 0.95
    assert np.mean(got.reshape(H, W)[:, W // 2] == ref.reshape(H, W)[:, W // 2]) >= 0.95

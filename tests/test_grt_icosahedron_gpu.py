"""GPU checks of 3DGRT with the reference's icosahedron proxies (`primitive_type: icosahedron`, the paper configurations
configs/paper/3dgrt/base_ours.yaml and base_ours_reference.yaml) against the brute-force oracle that intersects the
reference's world-space triangles (tests/grt_ico_oracle.py).  Tolerances are those of test_grt_parity_gpu.py."""
import numpy as np
import pytest

import grt_ico_oracle as gio
import scenes
from helpers import image_error_report, rel_l2
from test_grt_parity_gpu import _Batch, _Gaussians

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

# render blocks of configs/paper/3dgrt/base_ours.yaml (degree 4) and base_ours_reference.yaml (degree 2)
PAPER = {
    4: {"method": "3dgrt", "pipeline_type": "reference", "backward_pipeline_type": "referenceBwd", "particle_kernel_degree": 4,
        "particle_kernel_density_clamping": False, "particle_kernel_min_response": 0.0113, "particle_kernel_min_alpha": 1.0 / 255.0,
        "particle_kernel_max_alpha": 0.99, "particle_radiance_sph_degree": 3, "primitive_type": "icosahedron", "min_transmittance": 0.001,
        "max_consecutive_bvh_update": 15, "enable_normals": False, "enable_hitcounts": False, "enable_kernel_timings": False},
}
PAPER[2] = dict(PAPER[4], particle_kernel_degree=2)


def _tracer(degree):
    import threedgrt_tracer

    return threedgrt_tracer.Tracer({"render": dict(PAPER[degree])})


@pytest.mark.parametrize("degree", [4, 2])
@pytest.mark.parametrize("cam_index,size", [(1, (128, 128)), (6, (128, 128)), (3, (75, 53))])
def test_icosahedron_forward_and_gradients(degree, cam_index, size):
    """The rays whose forward differs by more than 1e-4 (at most max(3, 2e-4 * P): hit-order swaps of near-equal entry t, rays
    grazing an edge) get no upstream gradient in either backward, so that the gradient tolerance measures the adjoint."""
    sc = scenes.scene_c1(width=size[0], height=size[1])
    c2w = np.asarray(sc.camera(cam_index, 10), np.float32)
    cfg = gio.paper_config(degree)
    ro, rd = sc.rays()
    kw = dict(clamping=False, primitive="icosahedron")
    rgb, alpha, dist, hits, vis = gio.grt_trace(cfg, sc.particles, sc.sph, 3, ro[0], rd[0], c2w, **kw)

    dev = torch.device("cuda", 0)
    tr = _tracer(degree)
    g = _Gaussians(sc, dev)
    tr.build_acc(g, rebuild=True)
    _, bb = gio.grt_proxies(cfg, sc.particles, **kw)
    assert np.allclose(tr.tracer_wrapper.native_context(dev).scene_aabb(), bb, rtol=1e-5, atol=1e-5)
    out = tr.render(g, _Batch(sc, c2w, dev), train=True)
    img = torch.cat([out["pred_features"], out["pred_opacity"], out["pred_dist"]], -1)[0].detach().cpu().numpy()
    ref = np.concatenate([rgb, alpha, dist[..., 0:1]], -1)
    keep = (np.abs(img - ref).max(-1, keepdims=True) <= 1e-4).astype(np.float32)
    rng = np.random.default_rng(cam_index)
    d_rgb = rng.normal(size=rgb.shape).astype(np.float32) * keep
    d_alpha = rng.normal(size=alpha.shape).astype(np.float32) * keep
    d_dist = (0.1 * rng.normal(size=alpha.shape)).astype(np.float32) * keep
    dp, ds = gio.grt_trace_bwd(cfg, sc.particles, sc.sph, 3, ro[0], rd[0], c2w, rgb, alpha, dist, d_rgb, d_alpha, d_dist, **kw)
    loss = (out["pred_features"] * torch.from_numpy(d_rgb[None]).to(dev)).sum() + (out["pred_opacity"] * torch.from_numpy(d_alpha[None]).to(dev)).sum() \
        + (out["pred_dist"] * torch.from_numpy(d_dist[None]).to(dev)).sum()
    loss.backward()
    torch.cuda.synchronize()
    P = sc.width * sc.height
    assert hits.sum() > P and (1.0 - keep).sum() <= max(3, int(2e-4 * P))
    got = torch.cat([out["pred_features"], out["pred_opacity"]], -1)[0].detach().cpu().numpy()
    mean_e, max_e, bad = image_error_report(f"ico d{degree} cam{cam_index} rgba", got, np.concatenate([rgb, alpha], -1))
    assert mean_e <= 1e-5 and max_e <= 2e-2 and bad <= max(3, int(2e-4 * P))
    mean_e, max_e, bad = image_error_report(f"ico d{degree} cam{cam_index} dist", out["pred_dist"][0].detach().cpu().numpy(), dist[..., 0:1],
                                            atol=1e-4 * max(1.0, float(np.abs(dist[..., 0]).max())))
    assert mean_e <= 1e-4 and bad <= max(3, int(2e-4 * P))
    assert float(np.mean(out["hits_count"][0].detach().cpu().numpy() == hits)) >= 0.999
    got_vis = out["mog_visibility"].detach().cpu().numpy().view(np.int32).reshape(-1) != 0
    assert np.mean(got_vis == (vis.reshape(-1) != 0)) >= 0.999
    errs = dict(pos=rel_l2(g.positions.grad.cpu().numpy(), dp[:, 0:3]), dns=rel_l2(g.density.grad.cpu().numpy(), dp[:, 3:4]),
                quat=rel_l2(g.rotation.grad.cpu().numpy(), dp[:, 4:8]), scl=rel_l2(g.scale.grad.cpu().numpy(), dp[:, 8:11]),
                sph=rel_l2(g._sph.grad.cpu().numpy(), ds))
    print(f"[ico] degree {degree} cam{cam_index} gradient rel-L2:", {k: f"{v:.2e}" for k, v in errs.items()})
    assert max(errs.values()) <= 1e-3


def _frame(sc, c2w, d_out, degree=4):
    dev = torch.device("cuda", 0)
    tr = _tracer(degree)
    g = _Gaussians(sc, dev)
    tr.build_acc(g, rebuild=True)
    out = tr.render(g, _Batch(sc, c2w, dev), train=True)
    img = torch.cat([out["pred_features"], out["pred_opacity"], out["pred_dist"]], -1)
    (img * torch.from_numpy(d_out).to(dev)).sum().backward()
    torch.cuda.synchronize()
    grads = [t.grad.detach().cpu().numpy() for t in (g.positions, g.density, g.rotation, g.scale, g._sph)]
    return img[0].detach().cpu().numpy(), out["hits_count"][0].detach().cpu().numpy(), grads


@pytest.fixture(scope="module")
def c2_frame():
    sc = scenes.scene_c2(n=60_000, width=256, height=256)
    c2w = np.asarray(sc.camera(2, 10), np.float32)
    d_out = np.random.default_rng(0).normal(size=(1, sc.height, sc.width, 5)).astype(np.float32)
    return sc, c2w, d_out, _frame(sc, c2w, d_out)


def test_retrace_gives_the_replayed_gradients(c2_frame, monkeypatch):
    """GRTB200_HITCAP=0: the backward re-traces every ray (icosahedron candidates, entry-t order, stop before the last processed
    entry t) instead of replaying the forward's lists; the same hits in the same order give the same gradients."""
    sc, c2w, d_out, (img1, hits1, g1) = c2_frame
    monkeypatch.setenv("GRTB200_HITCAP", "0")
    img0, hits0, g0 = _frame(sc, c2w, d_out)
    assert hits1.sum() > 0 and np.array_equal(hits1, hits0)
    for name, a, b in zip(("positions", "density", "rotation", "scale", "sph"), g1, g0):
        err = rel_l2(a, b)
        print(f"[ico] re-trace vs replay d_{name} rel-L2 {err:.3e}")
        assert err <= 1e-5


@pytest.mark.parametrize("switch,off", [("GRTB200_PACKET", "0"), ("GRTB200_LEAF", "1"), ("GRTB200_SIZE_LEVELS", "0")])
def test_traversal_variants_give_the_same_image(c2_frame, switch, off, monkeypatch):
    sc, c2w, d_out, (img1, hits1, g1) = c2_frame
    monkeypatch.setenv(switch, off)
    img0, hits0, g0 = _frame(sc, c2w, d_out)
    P = sc.width * sc.height
    print(f"[ico] {switch}: hit counts differ on {(hits1 != hits0).sum()} of {P} rays")
    assert (hits1 != hits0).mean() <= 1e-3
    mean_e, max_e, bad = image_error_report(f"ico {switch}: image", img1, img0, atol=1e-4)
    assert mean_e <= 1e-6 and max_e <= 2e-2 and bad <= max(3, int(2e-4 * P))
    for name, a, b in zip(("positions", "density", "rotation", "scale", "sph"), g1, g0):
        assert rel_l2(a, b) <= 1e-3


def _raw_trace(parts, sph, ro, rd, degree=4):
    """Rays straight through the C ABI with an identity ray-to-world: (rgb [R,3], alpha [R], hits [R], visibility [N])."""
    import b200_native as nat

    dev = torch.device("cuda", 0)
    cfg = nat.grt_default_config()
    cfg.kernel_degree, cfg.density_clamping, cfg.primitive = degree, 0, nat.GRT_PRIMITIVES["icosahedron"]
    ctx = nat.GrtContext(cfg, 0)
    s = torch.cuda.current_stream(dev).cuda_stream
    n = parts.shape[0]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)  # noqa: E731
    P = t(parts if n else np.zeros((1, 12)))
    S = t(sph if n else np.zeros((1, 48)))
    soa = [P[:, 0:3].contiguous(), P[:, 4:8].contiguous(), P[:, 8:11].contiguous(), P[:, 3:4].contiguous()]  # must outlive the build
    ctx.build_bvh(s, n, *[a.data_ptr() for a in soa])
    H, W = ro.shape[:2]
    R = H * W
    tro, trd = t(ro), t(rd)
    r2w = np.ascontiguousarray(np.eye(4, dtype=np.float32)[:3, :4])
    rgb, alpha, dist, hits, vis = (torch.ones((R, 3), device=dev), torch.ones(R, device=dev), torch.ones((R, 2), device=dev),
                                   torch.ones(R, device=dev), torch.ones(max(n, 1), device=dev))
    ctx.trace(s, n, P.data_ptr(), S.data_ptr(), 3, 1e-3, 1, H, W, tro.data_ptr(), trd.data_ptr(), r2w.ctypes.data, rgb.data_ptr(),
              alpha.data_ptr(), dist.data_ptr(), hits.data_ptr(), vis.data_ptr())
    torch.cuda.synchronize()
    out = rgb.cpu().numpy(), alpha.cpu().numpy(), hits.cpu().numpy(), vis.cpu().numpy().view(np.int32)[:n]
    ctx.close()
    return out


def test_ray_origin_inside_the_proxy_gpu():
    sc = scenes.scene_c1(n=50, seed=3)
    parts = sc.particles[:1].copy()
    parts[0, 3] = 0.8
    cfg = gio.paper_config(4)
    kscl, _ = gio.grt_proxies(cfg, parts, clamping=False)
    d = np.array([0.3, -0.2, 0.93], np.float32)
    d /= np.linalg.norm(d)
    inside = (parts[0, 0:3] - 0.3 * float(kscl[0].min()) * d).astype(np.float32)
    outside = (parts[0, 0:3] - 5.0 * float(kscl[0].max()) * d).astype(np.float32)
    ro = np.stack([inside, outside]).reshape(1, 2, 3)
    rd = np.stack([d, d]).reshape(1, 2, 3)
    rgb, alpha, hits, vis = _raw_trace(parts, sc.sph[:1], ro, rd)
    ref = gio.grt_trace(cfg, parts, sc.sph[:1], 3, ro, rd, np.eye(4, dtype=np.float32), clamping=False, primitive="icosahedron")
    assert hits.tolist() == [0.0, 1.0] and ref[3].reshape(-1).tolist() == [0.0, 1.0]
    assert float(alpha[0]) == 0.0 and float(np.abs(rgb[0]).max()) == 0.0
    assert np.abs(rgb[1] - ref[0].reshape(-1, 3)[1]).max() <= 1e-4


def test_axis_parallel_rays_reach_the_geometry():
    sc = scenes.scene_c1()
    H = W = 48
    ys, xs = np.meshgrid(np.linspace(-1.4, 1.4, H, dtype=np.float32), np.linspace(-1.4, 1.4, W, dtype=np.float32), indexing="ij")
    ro = np.stack([xs, ys, np.full_like(xs, -4.0)], -1).astype(np.float32)
    rd = np.broadcast_to(np.array([0, 0, 1], np.float32), ro.shape).copy()
    rgb, alpha, hits, vis = _raw_trace(sc.particles, sc.sph, ro, rd)
    ref = gio.grt_trace(gio.paper_config(4), sc.particles, sc.sph, 3, ro, rd, np.eye(4, dtype=np.float32), clamping=False,
                        primitive="icosahedron")
    got_hits = hits.reshape(ref[3].shape)
    print(f"[ico] orthographic bundle: hits {int(got_hits.sum())} vs oracle {int(ref[3].sum())}")
    assert ref[3].sum() > 100 and float(np.mean(got_hits == ref[3])) >= 0.999
    mean_e, max_e, bad = image_error_report("ico orthographic rgb", rgb.reshape(ref[0].shape), ref[0])
    assert mean_e <= 1e-5 and bad <= 3


def test_empty_scene_and_single_particle():
    sc = scenes.scene_c1(n=50, width=32, height=24)
    ro, rd = sc.rays()
    c2w = np.asarray(sc.camera(0, 4), np.float32)
    wo = (ro[0].reshape(-1, 3) @ c2w[:3, :3].T + c2w[:3, 3]).reshape(1, sc.height, sc.width, 3).astype(np.float32)
    wd = (rd[0].reshape(-1, 3) @ c2w[:3, :3].T).reshape(1, sc.height, sc.width, 3).astype(np.float32)
    rgb, alpha, hits, _ = _raw_trace(sc.particles[:0], sc.sph[:0], wo[0], wd[0])
    assert float(np.abs(rgb).max()) == 0 and float(np.abs(alpha).max()) == 0 and float(hits.max()) == 0
    # one particle on the centre pixel's ray
    parts = sc.particles[:1].copy()
    c = wo[0, sc.height // 2, sc.width // 2], wd[0, sc.height // 2, sc.width // 2]
    parts[0, 0:3] = c[0] + 3.0 * c[1] / np.linalg.norm(c[1])
    parts[0, 3] = 0.8
    parts[0, 8:11] = 0.3
    rgb, alpha, hits, vis = _raw_trace(parts, sc.sph[:1], wo[0], wd[0])
    ref = gio.grt_trace(gio.paper_config(4), parts, sc.sph[:1], 3, wo[0], wd[0], np.eye(4, dtype=np.float32), clamping=False,
                        primitive="icosahedron")
    assert ref[3].sum() > 20 and np.array_equal(hits.reshape(ref[3].shape), ref[3]) and int(vis[0]) == 1
    assert np.abs(rgb.reshape(ref[0].shape) - ref[0]).max() <= 1e-4


def test_short_fit_with_the_paper_config():
    """30 Adam steps through Tracer.build_acc (rebuild=False: the update path of max_consecutive_bvh_update) + Tracer.render
    pull perturbed Gaussians towards renders of the unperturbed ones."""
    sc = scenes.scene_c1(n=400, width=64, height=48)
    dev = torch.device("cuda", 0)
    tr = _tracer(2)
    cams = [np.asarray(sc.camera(i, 6), np.float32) for i in range(3)]
    target = _Gaussians(sc, dev)
    with torch.no_grad():
        tr.build_acc(target, rebuild=True)
        refs = [tr.render(target, _Batch(sc, c, dev))["pred_features"].detach() for c in cams]
    rng = np.random.default_rng(0)
    pert = sc.particles.copy()
    pert[:, 0:3] += rng.normal(0, 0.02, (sc.n, 3)).astype(np.float32)
    pert[:, 3] = np.clip(pert[:, 3] * rng.uniform(0.6, 1.4, sc.n), 0.02, 0.95).astype(np.float32)
    sc_p = scenes.Scene(sc.name, sc.width, sc.height, sc.fx, sc.fy, pert, sc.sph, sc.sph_degree, sc.camera_radius)
    g = _Gaussians(sc_p, dev)
    opt = torch.optim.Adam([{"params": [g.positions], "lr": 2e-3}, {"params": [g.density], "lr": 2e-2}, {"params": [g._sph], "lr": 1e-2}])
    losses = []
    for it in range(30):
        tr.build_acc(g, rebuild=(it == 0))
        opt.zero_grad()
        loss = sum(torch.nn.functional.l1_loss(tr.render(g, _Batch(sc, cams[k], dev), train=True)["pred_features"], refs[k]) for k in range(3))
        loss.backward()
        opt.step()
        with torch.no_grad():
            g.density.clamp_(0.01, 0.99)
        losses.append(float(loss))
    print(f"[ico] short fit: loss {losses[0]:.4f} -> {losses[-1]:.4f}")
    assert all(np.isfinite(losses)) and losses[-1] < 0.8 * losses[0]
    assert tr.num_update_bvh > 0  # build_acc took the update path


@pytest.mark.parametrize("primitive", ["octahedron", "tetrahedron", "diamond", "trihexa", "trisurfel", "sphere", "custom"])
def test_unsupported_primitives_raise(primitive):
    import threedgrt_tracer

    with pytest.raises(NotImplementedError, match="instances, icosahedron"):
        threedgrt_tracer.Tracer({"render": dict(PAPER[4], primitive_type=primitive)})

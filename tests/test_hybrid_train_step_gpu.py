"""The 3DGRUT hybrid training step (train_step_hybrid.GaussianTrainStepHybrid) and the device code it adds: the mirror rays and the
composite against hybrid.py's torch expressions, the accumulating 3DGRT backward, one step against autograd through both reference-facing
tracers, reflectivity 0 against the 3DGUT step, render against hybrid.render_hybrid, short fits with and without densification, and two
ranks."""
import os

import numpy as np
import pytest

import scenes
from helpers import rel_l2

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

INSTANCES = {"render": {}}
# the 3DGRT paper config (base_ours.yaml) on the 3DGRT-only keys; the kernel is the 3DGUT pass's degree 2 either way
PAPER = {"render": {"primitive_type": "icosahedron", "particle_kernel_density_clamping": False, "max_consecutive_bvh_update": 15}}
CONFIGS = {"instances": INSTANCES, "icosahedron_paper": PAPER}
LRS = dict(positions=2e-3, density=0.05, rotation=1e-3, scale=5e-3, features_albedo=1e-2, features_specular=5e-4)


def _raw_from(particles, sph):
    dns = particles[:, 3:4].clamp(1e-4, 1 - 1e-4)
    return {"positions": particles[:, 0:3].clone(), "density": torch.log(dns / (1 - dns)), "rotation": particles[:, 4:8].clone(),
            "scale": torch.log(particles[:, 8:11]), "features_albedo": sph[:, 0:3].clone(), "features_specular": sph[:, 3:48].clone()}


class _Batch:
    """A gpu_batch for both reference-facing tracers: camera-space rays, T_to_world, the pinhole intrinsics of the scene."""

    def __init__(self, sc, rays_o, rays_d, c2w):
        from threedgut_tracer.tracer import ShutterType

        self.rays_ori, self.rays_dir, self.T_to_world = rays_o, rays_d, c2w.to(rays_o.device)
        self.intrinsics_OpenCVPinholeCameraModelParameters = dict(
            resolution=np.array([sc.width, sc.height]), shutter_type=ShutterType.GLOBAL, principal_point=np.array([sc.cx, sc.cy], np.float32),
            focal_length=np.array([sc.fx, sc.fy], np.float32), radial_coeffs=np.zeros(6, np.float32), tangential_coeffs=np.zeros(2, np.float32),
            thin_prism_coeffs=np.zeros(4, np.float32))


def _setup(n=600, size=96, dev=None):
    from threedgut_tracer.tracer import Tracer

    dev = dev or torch.device("cuda", 0)
    sc = scenes.scene_c1(n=n, width=size, height=size)
    ro, rd = sc.rays()
    rays_o, rays_d = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)
    P, S = torch.from_numpy(sc.particles).to(dev), torch.from_numpy(sc.sph).to(dev)
    poses = [torch.from_numpy(np.asarray(sc.camera(i, 6), np.float32))[None] for i in range(6)]  # host [1,4,4] camera-to-world
    sensor = Tracer._create_camera_parameters(_Batch(sc, rays_o, rays_d, poses[0]))[0]
    return sc, rays_o, rays_d, P, S, poses, sensor


def _capture_adam(step):
    seen = []
    real = step.optimizer.step

    def spy(d_particles, d_sph, visibility=None, **kw):
        seen.append((d_particles.clone(), d_sph.clone()))
        return real(d_particles, d_sph, visibility=visibility, **kw)

    step.optimizer.step = spy
    return seen


# ---------------------------------------------------------------------------------------------------------------------------------
# device code


@pytest.mark.parametrize("plane", ["floor", "tilted", "vertical"])
def test_rays_match_mirror_rays(plane):
    import hybrid
    import train_step_hybrid as th

    dev = torch.device("cuda", 0)
    sc = scenes.scene_c1(width=120, height=90)
    ro, rd = sc.rays()
    rays_o, rays_d = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)
    rays_o = rays_o + 0.05 * torch.randn_like(rays_o)  # non-zero camera-space origins exercise the whole transform
    # the tilted and the vertical plane pass through the scene centre, so that views 1 and 4 see part of the image reflect
    point, normal = {"floor": ((0.0, 0.0, -1.2), (0.0, 0.0, 1.0)), "tilted": ((0.0, 0.0, 0.0), (1.0, 0.0, 0.2)),
                     "vertical": ((0.0, 0.0, 0.0), (1.0, 0.0, 0.0))}[plane]
    partial = []
    for view in (1, 4):
        c2w = torch.from_numpy(np.asarray(sc.camera(view, 6), np.float32))[None]
        m = th.mirror_settings(dict(plane_point=point, plane_normal=normal))
        o, d, hit = th.hybrid_rays(rays_o, rays_d, c2w, m["plane_point"], m["plane_normal"])
        o2, d2, hit2 = th.hybrid_rays(rays_o, rays_d, c2w, m["plane_point"], m["plane_normal"])
        for a, b in ((o, o2), (d, d2), (hit, hit2)):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
        wo, wd, whit = hybrid.mirror_rays(rays_o, rays_d, c2w.to(dev), point, normal)
        got_hit, want_hit = hit.bool().cpu().numpy(), whit.reshape(-1).cpu().numpy()
        # rays at the boundary of the test: |denom| or |s| within 1e-6 of 0, recomputed from the reference's own terms
        R, t = c2w[0, :3, :3].to(dev), c2w[0, :3, 3].to(dev)
        wo_, wd_ = rays_o @ R.T + t, rays_d @ R.T
        n = torch.as_tensor(normal, dtype=torch.float32, device=dev)
        n = n / n.norm()
        denom = (wd_ * n).sum(-1).reshape(-1)
        s = ((torch.as_tensor(point, device=dev) - wo_) * n).sum(-1).reshape(-1) / torch.where(denom.abs() > 1e-8, denom, torch.full_like(denom, 1e-8))
        edge = ((denom.abs() <= 1e-6) | (s.abs() <= 1e-6)).cpu().numpy()
        diff = got_hit != want_hit
        print(f"[hybrid-rays] {plane} view {view}: hit fraction {got_hit.mean():.3f}, mask differences {int(diff.sum())} "
              f"(all at the boundary: {bool(np.all(edge[diff]))})")
        partial.append(0.0 < want_hit.mean() < 1.0)
        assert np.all(edge[diff])
        same = ~diff
        # `rays @ R.T` is a library matmul in mirror_rays: its last bit may differ from the kernel's sum, and the hit point o + s d moves by
        # that much over |denom| (the ray's condition number at the plane), so the relative bar scales with 1 / |denom| on hit rays
        cond = np.where(want_hit, 1.0 + 1.0 / np.maximum(denom.abs().cpu().numpy(), 1e-30), 1.0)[same]
        for name, got, want in (("origin", o, wo), ("direction", d, wd)):
            g, w = got.reshape(-1, 3).cpu().numpy()[same].astype(np.float64), want.reshape(-1, 3).cpu().numpy()[same].astype(np.float64)
            err = np.abs(g - w).max(1) / np.maximum(np.abs(w).max(1), 1.0)
            scaled = err / (cond if name == "origin" else 1.0)
            print(f"[hybrid-rays] {plane} view {view} {name}: max rel err {err.max():.2e}, over the condition number {scaled.max():.2e}")
            assert float(scaled.max()) <= 1e-6, (name, float(scaled.max()))
    assert plane == "floor" or any(partial)


def test_composite_forward_is_bit_identical_and_backward_matches_autograd():
    import train_step_hybrid as th

    dev = torch.device("cuda", 0)
    H, W, r = 37, 53, 0.3
    gen = torch.Generator(device=dev).manual_seed(5)
    rgba = torch.rand((H, W, 4), device=dev, generator=gen)
    rgba[::3, :, 3] = 0.0
    rgba[1::5, :, 3] = 1.0
    sec = torch.rand((1, H, W, 3), device=dev, generator=gen) * 1.7 - 0.2
    hit = (torch.rand((H * W,), device=dev, generator=gen) > 0.4).float()
    rgb = th.hybrid_composite(rgba, sec, hit, r)
    # render_hybrid's expression
    p_rgb, p_alpha = rgba[None, ..., :3], rgba[None, ..., 3:]
    want = p_rgb + r * (1.0 - p_alpha) * hit.view(1, H, W, 1) * sec
    assert torch.equal(rgb.view(torch.int32), want[0].contiguous().view(torch.int32))

    for with_alpha in (False, True):
        d_rgb = torch.randn((H, W, 3), device=dev, generator=gen)
        d_alpha = torch.randn((H, W, 1), device=dev, generator=gen) if with_alpha else None
        d_rgba, d_sec = th.hybrid_composite_bwd(rgba, sec, hit, r, d_rgb, d_alpha)
        a = rgba.clone().requires_grad_(True)
        s = sec.clone().requires_grad_(True)
        out = a[None, ..., :3] + r * (1.0 - a[None, ..., 3:]) * hit.view(1, H, W, 1) * s
        obj = (out[0] * d_rgb).sum() + ((a[..., 3:] * d_alpha).sum() if with_alpha else 0.0)
        obj.backward()
        for name, got, ref in (("d_rgba", d_rgba, a.grad), ("d_secondary", d_sec, s.grad)):
            err = float(((got - ref).abs() / ref.abs().clamp_min(1.0)).max())
            assert err <= 1e-6, (name, with_alpha, err)


@pytest.mark.parametrize("primitive", ["instances", "icosahedron"])
def test_accumulating_backward_adds_to_the_buffer(primitive):
    import threedgrt_tracer

    sc, rays_o, rays_d, P, S, poses, _ = _setup()
    dev = P.device
    ot = threedgrt_tracer.Tracer({"render": {"primitive_type": primitive}}).tracer_wrapper
    ot.set_replay(True, dev)
    ot.build_bvh_packed(P)
    rgb, alpha, dst, nrm, hits, vis = ot.trace(0, poses[2], rays_o, rays_d, P, S, 0, 3, 0.001)
    gen = torch.Generator(device=dev).manual_seed(9)
    d_rgb = torch.randn(rgb.shape, device=dev, generator=gen)
    d_alpha = torch.randn(alpha.shape, device=dev, generator=gen)
    zero1, zero3 = torch.zeros_like(alpha), torch.zeros_like(nrm)
    args = (0, poses[2], rays_o, rays_d, rgb, alpha, dst, nrm, P, S, d_rgb, d_alpha, zero1, zero3, 0, 3, 0.001)
    plain = [t.clone() for t in ot.trace_bwd(*args)]
    prefill = (torch.randn((sc.n, 12), device=dev, generator=gen), torch.randn((sc.n, 48), device=dev, generator=gen))
    buf = tuple(t.clone() for t in prefill)
    ot.trace_bwd(*args, out=buf, accumulate=True)
    assert float(plain[0].abs().max()) > 0 and float(plain[1].abs().max()) > 0
    for name, got, pre, g in zip(("d_particles", "d_sph"), buf, prefill, plain):
        err = rel_l2((got - pre).cpu().numpy(), g.cpu().numpy())
        err_sum = rel_l2(got.cpu().numpy(), (pre + g).cpu().numpy())
        print(f"[hybrid-accumulate] {primitive} {name}: rel-L2 {err:.2e} / {err_sum:.2e} (bar 1e-6)")
        assert err_sum <= 1e-6
    # the default still overwrites
    buf2 = tuple(t.clone() for t in prefill)
    ot.trace_bwd(*args, out=buf2)
    for got, g in zip(buf2, plain):
        assert rel_l2(got.cpu().numpy(), g.cpu().numpy()) <= 1e-6


# ---------------------------------------------------------------------------------------------------------------------------------
# one step against autograd


class _Gaussians:
    """Activated leaf tensors in the shape both Tracer.render / build_acc read them (identity activations)."""

    def __init__(self, particles, sph, deg):
        self.positions = particles[:, 0:3].clone().requires_grad_(True)
        self.density = particles[:, 3:4].clone().requires_grad_(True)
        self.rotation = particles[:, 4:8].clone().requires_grad_(True)
        self.scale = particles[:, 8:11].clone().requires_grad_(True)
        self._sph = sph.clone().requires_grad_(True)
        self.n_active_features = deg
        ident = lambda t: t  # noqa: E731
        self.rotation_activation = self.scale_activation = self.density_activation = ident

    def get_rotation(self):
        return self.rotation

    def get_scale(self):
        return self.scale

    def get_density(self):
        return self.density

    def get_features(self):
        return self._sph


class _SecondaryBatch:
    def __init__(self, o, d):
        self.rays_ori, self.rays_dir = o, d
        self.T_to_world = torch.eye(4, device=o.device, dtype=o.dtype)[None]


class _ImageLoss(torch.autograd.Function):
    """The step's loss on (rgb, primary alpha) as an autograd node: the composited, masked entry, or the plain one on black."""

    @staticmethod
    def forward(ctx, rgb, alpha, target, l1, ssim, background, mask):
        import losses

        if background is None and mask is None:
            loss, _, _, d_rgb = losses.image_loss_rgb(rgb.contiguous(), target, l1, ssim)
            d_alpha = torch.zeros_like(alpha)
        else:
            loss, _, _, d_rgb, d_alpha = losses.image_loss_rgb_alpha(rgb.contiguous(), alpha.contiguous(), target, l1, ssim, background=background,
                                                                     mask=mask)
        ctx.save_for_backward(d_rgb, d_alpha)
        return loss

    @staticmethod
    def backward(ctx, g):
        d_rgb, d_alpha = ctx.saved_tensors
        return g * d_rgb, g * d_alpha, None, None, None, None, None


CASES = [("instances", (1.0, 0.0), "black"), ("instances", (0.8, 0.2), "black"), ("icosahedron_paper", (1.0, 0.0), "black"),
         ("icosahedron_paper", (0.8, 0.2), "black"), ("instances", (0.8, 0.2), "white+mask")]


@pytest.mark.parametrize("config,weights,background", CASES)
def test_one_step_matches_autograd(config, weights, background):
    import hybrid
    import threedgrt_tracer
    import threedgut_tracer
    import train_step_hybrid as th

    sc, rays_o, rays_d, P, S, poses, sensor = _setup()
    dev = P.device
    H, W = sc.height, sc.width
    white = background != "black"
    mask = None
    if white:
        mask = (torch.rand((H, W), device=dev, generator=torch.Generator(device=dev).manual_seed(4)) > 0.2).float()
    step = th.GaussianTrainStepHybrid(_raw_from(P, S), LRS, conf=CONFIGS[config], lambda_l1=weights[0], lambda_ssim=weights[1],
                                      background="white" if white else "black")
    gen = torch.Generator(device=dev).manual_seed(3)
    target = (torch.rand((H, W, 3), device=dev, generator=gen) * 0.8).contiguous()
    particles, sph = step.activated()
    seen = _capture_adam(step)
    c2w = poses[1]
    step.step(rays_o, rays_d, sensor, c2w, target, mask=mask)
    d_particles, d_sph = seen[0]

    conf = th.hybrid_render_conf(CONFIGS[config])
    g = _Gaussians(particles, sph, 3)
    gut = threedgut_tracer.Tracer(conf)
    grt = threedgrt_tracer.Tracer(conf)
    primary = gut.render(g, _Batch(sc, rays_o, rays_d, c2w), train=True)
    m = th.mirror_settings()
    so, sd, hit = th.hybrid_rays(rays_o, rays_d, c2w, m["plane_point"], m["plane_normal"])  # the step's own secondary rays
    wo, wd, whit = hybrid.mirror_rays(rays_o, rays_d, c2w.to(dev), m["plane_point"], m["plane_normal"])
    assert int((whit.reshape(-1).float() != hit).sum()) <= 2
    grt.build_acc(g, rebuild=True)
    secondary = grt.render(g, _SecondaryBatch(so, sd), train=True)
    weight = m["reflectivity"] * (1.0 - primary["pred_opacity"]) * hit.view(1, H, W, 1)
    rgb = primary["pred_features"] + weight * secondary["pred_features"]
    alpha = primary["pred_opacity"]
    if weights[1] == 0.0 and not white:
        loss = weights[0] * (rgb[0] - target).abs().mean()
    else:
        loss = _ImageLoss.apply(rgb[0], alpha[0], target, weights[0], weights[1], (1.0, 1.0, 1.0) if white else None, mask)
    loss.backward()
    ref = {"positions": (g.positions.grad, d_particles[:, 0:3]), "density": (g.density.grad, d_particles[:, 3:4]),
           "rotation": (g.rotation.grad, d_particles[:, 4:8]), "scale": (g.scale.grad, d_particles[:, 8:11]), "sph": (g._sph.grad, d_sph)}
    print(f"[hybrid-train] {config} {weights} {background}: hit fraction {float(hit.mean()):.3f}")
    for name, (want, got) in ref.items():
        err = rel_l2(got.cpu().numpy(), want.cpu().numpy())
        print(f"[hybrid-train] {config} {weights} {background} {name}: rel-L2 {err:.2e} (bar 1e-5)")
        assert float(want.abs().max()) > 0 and err <= 1e-5, name
    assert float(d_particles[:, 11].abs().max()) == 0.0


def test_reflectivity_zero_gives_the_3dgut_steps_gradients():
    import train_step
    import train_step_hybrid as th
    from threedgut_tracer.tracer import Tracer

    sc, rays_o, rays_d, P, S, poses, sensor = _setup()
    gen = torch.Generator(device=P.device).manual_seed(7)
    target = (torch.rand((sc.height, sc.width, 3), device=P.device, generator=gen) * 0.8).contiguous()
    hyb = th.GaussianTrainStepHybrid(_raw_from(P, S), LRS, mirror=dict(reflectivity=0.0), lambda_l1=0.8, lambda_ssim=0.2)
    gut = [train_step.GaussianTrainStep(_raw_from(P, S), LRS, conf=th.hybrid_render_conf(None), lambda_l1=0.8, lambda_ssim=0.2) for _ in range(2)]
    a, b = _capture_adam(hyb), [_capture_adam(s) for s in gut]
    hyb.step(rays_o, rays_d, sensor, poses[3], target)
    for s in gut:
        s.step(rays_o, rays_d, sensor, Tracer._pose_from_c2w(poses[3][0]), target)
    for i, name in enumerate(("d_particles", "d_sph")):
        got, want, again = a[0][i].cpu().numpy(), b[0][0][i].cpu().numpy(), b[1][0][i].cpu().numpy()
        err, floor = rel_l2(got, want), rel_l2(again, want)
        # the 3DGUT backward sums its gradient rows with float atomics, so two runs of the same step differ by ~1e-6 already (`floor`)
        bar = 1e-6 + 2.0 * floor
        print(f"[hybrid-train] reflectivity 0 vs GaussianTrainStep {name}: rel-L2 {err:.2e}; GaussianTrainStep run to run {floor:.2e} "
              f"(bar {bar:.2e})")
        assert float(np.abs(want).max()) > 0 and err <= bar, name


def test_render_matches_render_hybrid():
    import hybrid
    import threedgrt_tracer
    import threedgut_tracer
    import train_step_hybrid as th

    sc, rays_o, rays_d, P, S, poses, sensor = _setup()
    conf = th.hybrid_render_conf(None)
    step = th.GaussianTrainStepHybrid(_raw_from(P, S), LRS)
    particles, sph = step.activated()
    g = _Gaussians(particles, sph, 3)
    gut, grt = threedgut_tracer.Tracer(conf), threedgrt_tracer.Tracer(conf)
    for view in (0, 2, 5):
        rgb, rgba, srgb, hit = step.render(rays_o, rays_d, sensor, poses[view])
        with torch.no_grad():
            want = hybrid.render_hybrid(gut, grt, g, _Batch(sc, rays_o, rays_d, poses[view]))
        assert torch.equal(rgba[..., :3], want["pred_features"][0]) and torch.equal(rgba[..., 3:], want["pred_opacity"][0])
        err = (rgb - want["pred_features_hybrid"][0]).abs().max(-1).values
        off = int((err > 1e-4).sum())
        print(f"[hybrid-render] view {view}: hit fraction {float(hit.mean()):.3f}, mean |d| {float(err.mean()):.2e}, max {float(err.max()):.2e}, "
              f"pixels > 1e-4: {off}")
        assert float(err.mean()) <= 1e-6 and off <= 5


# ---------------------------------------------------------------------------------------------------------------------------------
# fits


def _perturb(sc, P, S):
    gen = torch.Generator(device=P.device).manual_seed(0)
    P[:, 0:3] += 0.02 * torch.randn((sc.n, 3), device=P.device, generator=gen)
    P[:, 8:11] *= torch.exp(0.2 * torch.randn((sc.n, 3), device=P.device, generator=gen))
    S[:, 0:3] += 0.5 * torch.randn((sc.n, 3), device=P.device, generator=gen)
    return P, S


def _fit(start, steps, conf=INSTANCES, **kw):
    import train_step_hybrid as th

    sc, rays_o, rays_d, P, S, poses, sensor = _setup()
    truth = th.GaussianTrainStepHybrid(_raw_from(P, S), LRS, conf=conf)
    targets = [truth.render(rays_o, rays_d, sensor, p)[0].clone() for p in poses]
    P2, S2 = start(sc, P.clone(), S.clone())
    fit = th.GaussianTrainStepHybrid(_raw_from(P2, S2), LRS, conf=conf, **kw)

    def mean_loss():
        return float(np.mean([float((fit.render(rays_o, rays_d, sensor, p)[0] - t).abs().mean()) for p, t in zip(poses, targets)]))

    before, sizes = mean_loss(), []
    for it in range(steps):
        fit.step(rays_o, rays_d, sensor, poses[it % 6], targets[it % 6])
        sizes.append(fit.n)
    return sc, fit, before, mean_loss(), sizes


def test_short_fit_reduces_the_loss():
    sc, fit, before, after, _ = _fit(_perturb, 90, conf=PAPER)
    print(f"[hybrid-train] fit: mean L1 over 6 views {before:.5f} -> {after:.5f} after 90 steps, num_update_bvh {fit.num_update_bvh}")
    assert np.isfinite(after) and after < 0.6 * before
    assert fit.optimizer.steps == 90


def test_fit_with_gs_densification():
    import densify

    def start(sc, P, S):
        keep = torch.arange(sc.n, device=P.device) % 3 != 0
        P2, S2 = P[keep].clone(), S[keep].clone()
        P2[:, 8:11] *= 1.3
        return P2, S2

    conf = densify.DensifyConfig(clone_grad_threshold=2e-6, split_grad_threshold=2e-6, relative_size_threshold=0.03, prune_density_threshold=0.02,
                                 densify_start=10, densify_end=200, densify_frequency=30, prune_start=10, prune_end=200, prune_frequency=45,
                                 reset_start=-1, seed=1)
    sc, fit, before, after, sizes = _fit(start, 120, densify_conf=conf, scene_extent=3.0)
    n0 = sizes[0]
    print(f"[hybrid-train+densify] N {n0} -> {fit.n} (max {max(sizes)}), mean L1 {before:.5f} -> {after:.5f}")
    assert len(set(sizes)) > 1 and max(sizes) > n0
    assert fit.exchange.n == fit.n and fit.exchange.bucket.flat.numel() == 60 * fit.n
    assert np.isfinite(after) and after < 0.95 * before


def test_fit_with_mcmc_densification():
    import densify

    def start(sc, P, S):
        P, S = _perturb(sc, P, S)
        P[::9, 3] = 0.001
        return P, S

    conf = densify.MCMCConfig(relocate_start=5, relocate_frequency=20, add_start=5, add_frequency=20, perturb_start=0, noise_lr=5e3, seed=2)
    sc, fit, before, after, sizes = _fit(start, 90, conf=PAPER, densify_conf=conf, lambda_l1=0.8, lambda_ssim=0.2)
    print(f"[hybrid-train+mcmc] N {sc.n} -> {fit.n}, mean L1 {before:.5f} -> {after:.5f}")
    assert fit.n > sc.n and fit.exchange.n == fit.n and fit.optimizer.exp_avg["scale"].shape == (fit.n, 3)
    assert np.isfinite(after) and after < 0.8 * before


# ---------------------------------------------------------------------------------------------------------------------------------
# two ranks


def _rank_worker(rank, world, port, out_dir):
    import torch.distributed as dist

    import train_step_hybrid as th
    import view_parallel as vp

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        dev = torch.device("cuda", rank)
        sc, rays_o, rays_d, P, S, poses, sensor = _setup(dev=dev)
        targets = torch.from_numpy(np.load(os.path.join(out_dir, "targets.npy"))).to(dev)
        fit = th.GaussianTrainStepHybrid(_raw_from(*_perturb(sc, P.clone(), S.clone())), LRS, selective=True)
        for it in range(20):
            views = [vp.views_for_rank(it, r, world, 6)[0] for r in range(world)]
            positions = np.stack([np.asarray(poses[v][0, :3, 3], np.float32) for v in views])
            fit.step(rays_o, rays_d, sensor, poses[views[rank]], targets[views[rank]], all_sensor_positions=positions)
        torch.cuda.synchronize(dev)
        np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **{k: v.detach().cpu().numpy() for k, v in fit.params.items()})
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_stay_bit_identical(tmp_path):
    import torch.multiprocessing as mp

    import train_step_hybrid as th
    from test_grt_train_step_gpu import _free_port

    world = 2
    sc, rays_o, rays_d, P, S, poses, sensor = _setup()
    truth = th.GaussianTrainStepHybrid(_raw_from(P, S), LRS)
    targets = torch.stack([truth.render(rays_o, rays_d, sensor, p)[0] for p in poses])
    np.save(tmp_path / "targets.npy", targets.cpu().numpy())
    mp.spawn(_rank_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [np.load(tmp_path / f"rank{r}.npz") for r in range(world)]
    for k in outs[0].files:
        assert np.array_equal(outs[0][k], outs[1][k]), k

"""The 3DGRT training step (train_step_grt.GaussianTrainStepGRT) and the device code it adds: the packed BVH build, the image loss on the
3DGRT layout, the gradients it hands to Adam against Tracer.render + autograd, short fits with and without densification, and two ranks."""
import os
import socket

import numpy as np
import pytest

import scenes
from helpers import rel_l2
from train_step import raw_params

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

INSTANCES = {"render": {}}
# the 3DGRT paper configs (base_ours.yaml): icosahedron proxies, degree-2 kernel, no density clamping, BVH update cadence 15
PAPER = {"render": {"primitive_type": "icosahedron", "particle_kernel_degree": 2, "particle_kernel_density_clamping": False,
                    "max_consecutive_bvh_update": 15}}
CONFIGS = {"instances": INSTANCES, "icosahedron_paper": PAPER}
LRS = dict(positions=2e-3, density=0.05, rotation=1e-3, scale=5e-3, features_albedo=1e-2, features_specular=5e-4)


def _setup(n=600, size=96, dev=None):
    dev = dev or torch.device("cuda", 0)
    sc = scenes.scene_c1(n=n, width=size, height=size)
    ro, rd = sc.rays()
    rays_o, rays_d = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)
    P, S = torch.from_numpy(sc.particles).to(dev), torch.from_numpy(sc.sph).to(dev)
    poses = [torch.from_numpy(np.asarray(sc.camera(i, 6), np.float32))[None] for i in range(6)]  # host [1,4,4]
    return sc, rays_o, rays_d, P, S, poses


def _capture_adam(step):
    """Wrap the optimizer's step so that the (d_particles, d_sph) it is handed are copied out."""
    seen = []
    real = step.optimizer.step

    def spy(d_particles, d_sph, visibility=None):
        seen.append((d_particles.clone(), d_sph.clone()))
        return real(d_particles, d_sph, visibility=visibility)

    step.optimizer.step = spy
    return seen


# ---------------------------------------------------------------------------------------------------------------------------------
# device code


@pytest.mark.parametrize("primitive", ["instances", "icosahedron"])
@pytest.mark.parametrize("scene", ["c1", "c2_small"])
def test_packed_build_is_bit_identical(primitive, scene):
    import threedgrt_tracer

    dev = torch.device("cuda", 0)
    sc = scenes.scene_c1(width=128, height=96) if scene == "c1" else scenes.scene_c2(n=40_000, width=160, height=128)
    P, S = torch.from_numpy(sc.particles).to(dev), torch.from_numpy(sc.sph).to(dev)
    ro, rd = sc.rays()
    rays_o, rays_d = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)
    c2w = torch.from_numpy(np.asarray(sc.camera(2, 10), np.float32))[None]
    outs, boxes = [], []
    for packed in (False, True):
        ot = threedgrt_tracer.Tracer({"render": {"primitive_type": primitive}}).tracer_wrapper
        if packed:
            ot.build_bvh_packed(P)
        else:
            ot.build_bvh(P[:, 0:3].contiguous(), P[:, 4:8].contiguous(), P[:, 8:11].contiguous(), P[:, 3:4].contiguous())
        boxes.append(ot.native_context(dev).scene_aabb())
        rgb, alpha, dst, _, hits, vis = ot.trace(0, c2w, rays_o, rays_d, P, S, 0, 3, 0.001)
        outs.append([t.cpu().numpy() for t in (rgb, alpha, dst, hits, vis)])
    assert np.array_equal(boxes[0].view(np.uint32), boxes[1].view(np.uint32))
    assert float(outs[0][3].sum()) > 0
    for name, a, b in zip(("rgb", "alpha", "dist", "hits", "visibility"), *outs):
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), name


@pytest.mark.parametrize("size", [(96, 96), (800, 800), (61, 97)])
@pytest.mark.parametrize("weights", [(0.8, 0.2), (1.0, 0.0), (0.0, 1.0)])
def test_split_layout_loss_is_bit_identical(size, weights):
    import losses

    dev = torch.device("cuda", 0)
    h, w = size
    gen = torch.Generator(device=dev).manual_seed(h * 1000 + w)
    tgt = torch.rand((h, w, 3), device=dev, generator=gen)
    rgb = (tgt + 0.1 * torch.randn((1, h, w, 3), device=dev, generator=gen)).clamp(0, 1.2).contiguous()
    alpha = torch.rand((1, h, w, 1), device=dev, generator=gen)
    ref = losses.image_loss(torch.cat([rgb, alpha], -1).contiguous(), tgt, *weights)
    got = losses.image_loss_rgb(rgb, tgt, *weights)
    assert got[3].shape == (h, w, 3)
    assert torch.equal(got[3], ref[3][..., :3]) and bool((ref[3][..., 3] == 0).all())
    # Both entries add their per-block partial sums of |x - y| and of the SSIM map with atomicAdd, so the order of those additions (not
    # their terms) changes from run to run, in either entry alike; the scalars agree to that rounding (the absolute bar of test_loss_gpu.py).
    for name, a, b in zip(("loss", "l1", "ssim"), got[:3], ref[:3]):
        a, b = float(a), float(b)
        assert abs(a - b) <= 1e-6, (name, a, b)


# ---------------------------------------------------------------------------------------------------------------------------------
# one step against autograd


class _Gaussians:
    """Activated leaf tensors in the shape Tracer.render / build_acc read them (identity activations)."""

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


class _Batch:
    def __init__(self, rays_o, rays_d, c2w):
        self.rays_ori, self.rays_dir, self.T_to_world = rays_o, rays_d, c2w.to(rays_o.device)


class _ImageLoss(torch.autograd.Function):
    """lambda_l1 L1 + lambda_ssim (1 - SSIM) of the 3DGUT layout entry on cat(rgb, alpha), as an autograd node."""

    @staticmethod
    def forward(ctx, rgba, target, l1, ssim):
        import losses

        loss, _, _, d = losses.image_loss(rgba.contiguous(), target.contiguous(), l1, ssim)
        ctx.save_for_backward(d)
        return loss

    @staticmethod
    def backward(ctx, g):
        (d,) = ctx.saved_tensors
        return g * d, None, None, None


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("weights", [(1.0, 0.0), (0.8, 0.2)])
def test_one_step_matches_autograd(config, weights):
    import threedgrt_tracer
    import train_step_grt

    sc, rays_o, rays_d, P, S, poses = _setup()
    step = train_step_grt.GaussianTrainStepGRT(raw_params(P, S), LRS, conf=CONFIGS[config], lambda_l1=weights[0], lambda_ssim=weights[1])
    gen = torch.Generator(device=P.device).manual_seed(3)
    target = (torch.rand((sc.height, sc.width, 3), device=P.device, generator=gen) * 0.8).contiguous()
    particles, sph = step.activated()
    seen = _capture_adam(step)
    step.step(rays_o, rays_d, poses[1], target)
    d_particles, d_sph = seen[0]

    tracer = threedgrt_tracer.Tracer(CONFIGS[config])
    g = _Gaussians(particles, sph, 3)
    tracer.build_acc(g, rebuild=True)
    out = tracer.render(g, _Batch(rays_o, rays_d, poses[1]), train=True)
    rgb = out["pred_features"]
    if weights[1] == 0.0:
        loss = weights[0] * (rgb[0] - target).abs().mean()
    else:
        loss = _ImageLoss.apply(torch.cat([rgb, out["pred_opacity"]], -1)[0], target, *weights)
    loss.backward()
    ref = {"positions": (g.positions.grad, d_particles[:, 0:3]), "density": (g.density.grad, d_particles[:, 3:4]),
           "rotation": (g.rotation.grad, d_particles[:, 4:8]), "scale": (g.scale.grad, d_particles[:, 8:11]), "sph": (g._sph.grad, d_sph)}
    for name, (want, got) in ref.items():
        err = rel_l2(got.cpu().numpy(), want.cpu().numpy())
        print(f"[grt-train] {config} {weights} {name}: rel-L2 {err:.2e} (bar 1e-5)")
        assert float(want.abs().max()) > 0 and err <= 1e-5, name
    assert float(d_particles[:, 11].abs().max()) == 0.0


# ---------------------------------------------------------------------------------------------------------------------------------
# fits


def _fit_setup(config, raw_perturb, **kw):
    import train_step_grt

    sc, rays_o, rays_d, P, S, poses = _setup()
    truth = train_step_grt.GaussianTrainStepGRT(raw_params(P, S), LRS, conf=CONFIGS[config])
    targets = [truth.render(rays_o, rays_d, p)[0][0].clone() for p in poses]
    P2, S2 = raw_perturb(sc, P.clone(), S.clone())
    fit = train_step_grt.GaussianTrainStepGRT(raw_params(P2, S2), LRS, conf=CONFIGS[config], **kw)

    def mean_loss():
        return float(np.mean([float((fit.render(rays_o, rays_d, p)[0][0] - t).abs().mean()) for p, t in zip(poses, targets)]))

    return sc, fit, rays_o, rays_d, poses, targets, mean_loss


def _perturb(sc, P, S):
    gen = torch.Generator(device=P.device).manual_seed(0)
    P[:, 0:3] += 0.02 * torch.randn((sc.n, 3), device=P.device, generator=gen)
    P[:, 8:11] *= torch.exp(0.2 * torch.randn((sc.n, 3), device=P.device, generator=gen))
    S[:, 0:3] += 0.5 * torch.randn((sc.n, 3), device=P.device, generator=gen)
    return P, S


@pytest.mark.parametrize("config", list(CONFIGS))
def test_short_fit_reduces_the_loss(config):
    sc, fit, rays_o, rays_d, poses, targets, mean_loss = _fit_setup(config, _perturb)
    before, updates = mean_loss(), []
    for it in range(90):
        fit.step(rays_o, rays_d, poses[it % 6], targets[it % 6])
        updates.append(fit.num_update_bvh)
    after = mean_loss()
    print(f"[grt-train] {config}: mean L1 over 6 views {before:.5f} -> {after:.5f} after 90 steps, max num_update_bvh {max(updates)}")
    assert np.isfinite(after) and after < 0.6 * before
    assert fit.optimizer.steps == 90
    if config == "icosahedron_paper":
        assert max(updates) == 15 and 0 in updates[1:]  # update path up to max_consecutive_bvh_update, then a rebuild
    else:
        assert max(updates) == 0  # density clamping: a rebuild every step


def test_fit_with_gs_densification():
    import densify

    def start(sc, P, S):
        keep = torch.arange(sc.n, device=P.device) % 3 != 0  # start from two thirds of the Gaussians: the fit has to grow some back
        P2, S2 = P[keep].clone(), S[keep].clone()
        P2[:, 8:11] *= 1.3
        return P2, S2

    conf = densify.DensifyConfig(clone_grad_threshold=2e-6, split_grad_threshold=2e-6, relative_size_threshold=0.03, prune_density_threshold=0.02,
                                 densify_start=10, densify_end=200, densify_frequency=30, prune_start=10, prune_end=200, prune_frequency=45,
                                 reset_start=-1, seed=1)
    sc, fit, rays_o, rays_d, poses, targets, mean_loss = _fit_setup("instances", start, densify_conf=conf, scene_extent=3.0)
    n0, before, sizes = fit.n, mean_loss(), []
    for it in range(120):
        fit.step(rays_o, rays_d, poses[it % 6], targets[it % 6])
        sizes.append(fit.n)
    after = mean_loss()
    print(f"[grt-train+densify] N {n0} -> {fit.n} (max {max(sizes)}), mean L1 {before:.5f} -> {after:.5f}")
    assert len(set(sizes)) > 1 and max(sizes) > n0
    assert fit.exchange.n == fit.n and fit.exchange.bucket.flat.numel() == 60 * fit.n
    assert fit.optimizer.exp_avg["features_specular"].shape == (fit.n, 45)
    assert np.isfinite(after) and after < 0.95 * before


def test_fit_with_mcmc_densification():
    import densify

    def start(sc, P, S):
        P, S = _perturb(sc, P, S)
        P[::9, 3] = 0.001  # a few dead Gaussians for relocate()
        return P, S

    conf = densify.MCMCConfig(relocate_start=5, relocate_frequency=20, add_start=5, add_frequency=20, perturb_start=0, noise_lr=5e3, seed=2)
    sc, fit, rays_o, rays_d, poses, targets, mean_loss = _fit_setup("icosahedron_paper", start, densify_conf=conf, lambda_l1=0.8, lambda_ssim=0.2)
    before = mean_loss()
    for it in range(90):
        fit.step(rays_o, rays_d, poses[it % 6], targets[it % 6])
    after = mean_loss()
    print(f"[grt-train+mcmc] N {sc.n} -> {fit.n}, mean L1 {before:.5f} -> {after:.5f}")
    assert fit.n > sc.n and fit.exchange.n == fit.n and fit.optimizer.exp_avg["scale"].shape == (fit.n, 3)
    assert np.isfinite(after) and after < 0.8 * before


# ---------------------------------------------------------------------------------------------------------------------------------
# two ranks


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank_worker(rank, world, port, out_dir):
    import torch.distributed as dist

    import train_step_grt
    import view_parallel as vp

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        dev = torch.device("cuda", rank)
        sc, rays_o, rays_d, P, S, poses = _setup(dev=dev)
        targets = torch.from_numpy(np.load(os.path.join(out_dir, "targets.npy"))).to(dev)
        fit = train_step_grt.GaussianTrainStepGRT(raw_params(*_perturb(sc, P.clone(), S.clone())), LRS, selective=True)
        seen = _capture_adam(fit)
        for it in range(20):
            views = [vp.views_for_rank(it, r, world, 6)[0] for r in range(world)]
            positions = np.stack([fit.sensor_position(poses[v]) for v in views])
            fit.step(rays_o, rays_d, poses[views[rank]], targets[views[rank]], all_sensor_positions=positions)
        torch.cuda.synchronize(dev)
        np.savez(os.path.join(out_dir, f"rank{rank}.npz"), dp0=seen[0][0].cpu().numpy(), ds0=seen[0][1].cpu().numpy(),
                 **{k: v.detach().cpu().numpy() for k, v in fit.params.items()})
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_stay_bit_identical(tmp_path):
    import torch.multiprocessing as mp

    import train_step_grt
    import view_parallel as vp

    world = 2
    sc, rays_o, rays_d, P, S, poses = _setup()
    truth = train_step_grt.GaussianTrainStepGRT(raw_params(P, S), LRS)
    targets = torch.stack([truth.render(rays_o, rays_d, p)[0][0] for p in poses])
    np.save(tmp_path / "targets.npy", targets.cpu().numpy())
    mp.spawn(_rank_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [np.load(tmp_path / f"rank{r}.npz") for r in range(world)]
    for k in outs[0].files:
        if k not in ("dp0", "ds0"):
            assert np.array_equal(outs[0][k], outs[1][k]), k
    # the first step's exchanged gradient == the serial sum of the two ranks' single-view gradients (each normalised by the batch of 2)
    want_p = want_s = 0.0
    for r in range(world):
        single = train_step_grt.GaussianTrainStepGRT(raw_params(*_perturb(sc, P.clone(), S.clone())), LRS)
        seen = _capture_adam(single)
        v = vp.views_for_rank(0, r, world, 6)[0]
        single.step(rays_o, rays_d, poses[v], targets[v])
        want_p, want_s = want_p + seen[0][0].cpu().numpy() / world, want_s + seen[0][1].cpu().numpy() / world
    for r in range(world):
        ep, es = rel_l2(outs[r]["dp0"], want_p), rel_l2(outs[r]["ds0"], want_s)
        print(f"[grt-train 2 ranks] rank {r}: first-step gradient rel-L2 {ep:.2e} / {es:.2e} (bar 1e-6)")
        assert ep <= 1e-6 and es <= 1e-6

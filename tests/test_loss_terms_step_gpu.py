"""Both training steps with the rest of the reference loss: background compositing, the image mask and the opacity / scale regularisers.
One step against autograd of the reference's formulas (Tracer.render -> background.py's composite -> the mask product -> L1 + SSIM ->
+ lambda_opacity mean|sigmoid| + lambda_scale mean|exp| on the raw leaves), fits over a white background and with the MCMC loss, and
two ranks with a random background."""
import os

import numpy as np
import pytest

import scenes
from helpers import rel_l2
from test_grt_train_step_gpu import CONFIGS, LRS, _Batch, _free_port, _ImageLoss, _perturb, _raw_from, _setup

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

KINDS = ("gut", "gut_sorted", "grt_instances", "grt_icosahedron_paper")
SORTED = {"render": {"splat": {"k_buffer_size": 16}}}  # configs/paper/3dgut/sorted_*.yaml: the k-buffer of 16 hits


class _RawGaussians:
    """Raw leaf tensors with the reference's activations (model.py:102-118), in the shape the 3DGRT Tracer reads them."""

    def __init__(self, leaves, deg):
        self.positions, self.density, self.rotation, self.scale = (leaves[k] for k in ("positions", "density", "rotation", "scale"))
        self._sph = torch.cat([leaves["features_albedo"], leaves["features_specular"]], 1)
        self.n_active_features = deg
        self.rotation_activation = torch.nn.functional.normalize
        self.scale_activation = torch.exp
        self.density_activation = torch.sigmoid

    def get_rotation(self):
        return torch.nn.functional.normalize(self.rotation)

    def get_scale(self):
        return torch.exp(self.scale)

    def get_density(self):
        return torch.sigmoid(self.density)

    def get_features(self):
        return self._sph


class _Harness:
    """One scene (C1, 600 Gaussians, 96x96, 6 views) driven through either training step.  gut_sorted: the 3DGUT step with the k-buffer
    (sorted 3DGUT), whose compact backward reads final gradients from the accumulator rows."""

    def __init__(self, kind):
        self.kind = kind
        self.gut = kind.startswith("gut")
        self.sc, self.rays_o, self.rays_d, self.P, self.S, self.poses = _setup()
        self.dev = self.P.device
        self.H, self.W = self.sc.height, self.sc.width
        if self.gut:
            from threedgut_tracer.tracer import ShutterType, fromOpenCVPinholeCameraModelParameters

            sc = self.sc
            self.sensor = fromOpenCVPinholeCameraModelParameters(np.array([sc.width, sc.height]), ShutterType.GLOBAL,
                                                                 np.array([sc.cx, sc.cy], np.float32), np.array([sc.fx, sc.fy], np.float32),
                                                                 np.zeros(6, np.float32), np.zeros(2, np.float32), np.zeros(4, np.float32))
            self.views = [scenes.pose7_from_c2w(sc.camera(i, 6)) for i in range(6)]
            self.conf = SORTED if kind == "gut_sorted" else None
        else:
            self.conf = CONFIGS[kind[len("grt_"):]]

    def make(self, raw, **kw):
        if self.gut:
            import train_step

            return train_step.GaussianTrainStep(raw, LRS, conf=self.conf, **kw)
        import train_step_grt

        return train_step_grt.GaussianTrainStepGRT(raw, LRS, conf=self.conf, **kw)

    def step(self, st, v, target, mask=None):
        if self.gut:
            return st.step(self.rays_o, self.rays_d, self.sensor, self.views[v], target, mask=mask)
        return st.step(self.rays_o, self.rays_d, self.poses[v], target, mask=mask)

    def render(self, st, v):
        """(rgb [H,W,3], alpha [H,W,1]) of the step's current parameters."""
        if self.gut:
            rgba = st.render(self.rays_o, self.rays_d, self.sensor, self.views[v])[0].reshape(self.H, self.W, 4)
            return rgba[..., :3], rgba[..., 3:]
        out = st.render(self.rays_o, self.rays_d, self.poses[v])
        return out[0][0], out[1][0]

    def autograd_render(self, leaves, v):
        """Tracer.render's autograd node on the activated raw leaves: (rgb [H,W,3], alpha [H,W,1])."""
        if self.gut:
            from threedgut_tracer.tracer import SensorPose3D, SplatRaster, Tracer

            raster = SplatRaster(self.conf or {"render": {}})
            pose = self.views[v]
            rgba, _, _, _ = Tracer._Autograd.apply(raster, 0, 3, self.rays_o, self.rays_d, leaves["positions"],
                                                   torch.nn.functional.normalize(leaves["rotation"]), torch.exp(leaves["scale"]),
                                                   torch.sigmoid(leaves["density"]),
                                                   torch.cat([leaves["features_albedo"], leaves["features_specular"]], 1),
                                                   self.sensor, SensorPose3D(T_world_sensors=[pose, pose], timestamps_us=[0, 1]))
            rgba = rgba.reshape(self.H, self.W, 4)
            return rgba[..., :3], rgba[..., 3:]
        import threedgrt_tracer

        tracer = threedgrt_tracer.Tracer(self.conf)
        g = _RawGaussians(leaves, 3)
        tracer.build_acc(g, rebuild=True)
        out = tracer.render(g, _Batch(self.rays_o, self.rays_d, self.poses[v]), train=True)
        return out["pred_features"][0], out["pred_opacity"][0]


# ---------------------------------------------------------------------------------------------------------------------------------
# one step against autograd


def _step_against_autograd(hz, background, use_mask, lo, ls, weights=(0.8, 0.2)):
    """One bias-corrected step; returns ({group: rel-L2 of exp_avg / (1 - b1) against the autograd raw gradient}, step loss, autograd loss)."""
    H, W, dev = hz.H, hz.W, hz.dev
    raw = _raw_from(hz.P, hz.S)
    st = hz.make({k: v.clone() for k, v in raw.items()}, lambda_l1=weights[0], lambda_ssim=weights[1], background=background, background_seed=5,
                 lambda_opacity=lo, lambda_scale=ls)
    gen = torch.Generator(device=dev).manual_seed(3)
    target = (torch.rand((H, W, 3), device=dev, generator=gen) * 0.8).contiguous()
    mask = (torch.rand((H, W), device=dev, generator=gen) > 0.25).float() if use_mask else None
    got_loss = float(hz.step(st, 1, target, mask=None if mask is None else mask[None, :, :, None]))
    if background == "random":
        bg = st.background.image.clone()
        assert torch.equal(bg, torch.rand((H, W, 3), device=dev, generator=torch.Generator(device=dev).manual_seed(5)))  # seed + rank 0
    else:
        bg = torch.full((H, W, 3), {"white": 1.0, "black": 0.0}[background], device=dev)

    leaves = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    rgb, alpha = hz.autograd_render(leaves, 1)
    x, y = rgb, target
    if background != "black":
        x = x + bg * (1.0 - alpha)                # background.py:91 / 93
    if mask is not None:
        x, y = x * mask[..., None], y * mask[..., None]   # trainer.py:693-694
    loss = _ImageLoss.apply(torch.cat([x, torch.zeros_like(alpha)], -1), y, *weights)
    loss = loss + lo * torch.sigmoid(leaves["density"]).abs().mean() + ls * torch.exp(leaves["scale"]).abs().mean()   # trainer.py:722-736
    loss.backward()
    one_minus_b1 = float(np.float32(1) - np.float32(0.9))
    errs = {}
    for k in raw:
        want = leaves[k].grad.cpu().numpy()
        assert float(np.abs(want).max()) > 0, k
        errs[k] = rel_l2(st.optimizer.exp_avg[k].cpu().numpy() / one_minus_b1, want)
    return errs, got_loss, float(loss.detach())


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("background", ["white", "random"])
def test_one_step_matches_autograd(kind, background):
    hz = _Harness(kind)
    errs, got_loss, want_loss = _step_against_autograd(hz, background, True, 0.01, 0.02)
    assert abs(got_loss - want_loss) <= 1e-5, (got_loss, want_loss)
    floor = {}
    if kind.startswith("gut"):
        # The 3DGUT step differentiates through the compact backward, the autograd node through the full one; their rotation gradients
        # differ by ~1e-5 rel-L2 on the parent's path already (black, no mask, no regulariser), and the new terms must add nothing to it.
        floor, _, _ = _step_against_autograd(hz, "black", False, 0.0, 0.0)
    for k, err in errs.items():
        bar = max(1e-5, 2.0 * floor.get(k, 0.0))
        print(f"[loss-terms step] {kind} {background} {k}: exp_avg / (1 - b1) vs autograd rel-L2 {err:.2e} (bar {bar:.2e}"
              f"{f'; plain step {floor[k]:.2e}' if k in floor else ''})")
        assert err <= bar, k


@pytest.mark.parametrize("weights", [(1.0, 0.0), (0.8, 0.2)])
def test_sorted_gut_step_matches_autograd(weights):
    """The sorted 3DGUT step (k-buffer of 16 hits: the COMPACT, non-canonical G8 and sph_grad_from_views) with plain L1 and with L1 + SSIM,
    black background, no mask: one step's gradients against autograd through Tracer.render with the same config."""
    from threedgut_tracer.tracer import SplatRaster

    hz = _Harness("gut_sorted")
    errs, got_loss, want_loss = _step_against_autograd(hz, "black", False, 0.0, 0.0, weights=weights)
    assert abs(got_loss - want_loss) <= 1e-5, (got_loss, want_loss)
    # the compact-vs-full floor of the rotation on this frame: trace_bwd_compact against trace_bwd, same inputs
    raster = SplatRaster(SORTED)
    particles = torch.cat([hz.P[:, 0:11], torch.zeros_like(hz.P[:, :1])], 1).contiguous()
    pose = hz.views[1]
    gen = torch.Generator(device=hz.dev).manual_seed(7)
    d_rgba = torch.randn((hz.H, hz.W, 4), device=hz.dev, generator=gen)
    d_dist = torch.zeros((hz.H, hz.W, 1), device=hz.dev)
    args = (0, 3, particles, hz.S, hz.rays_o, hz.rays_d, None, hz.sensor, 0, 1, pose, pose)
    rgba, dst, _, _ = raster.trace(*args)
    dp_full, _ = raster.trace_bwd(*args, rgba, d_rgba, dst, d_dist)
    rgba, dst, _, _ = raster.trace(*args)
    dp_compact, _ = raster.trace_bwd_compact(*args, rgba, d_rgba, dst, d_dist)
    floor = rel_l2(dp_compact[:, 4:8].cpu().numpy(), dp_full[:, 4:8].cpu().numpy())
    for k, err in errs.items():
        bar = max(1e-5, 2.0 * floor) if k == "rotation" else 1e-5
        print(f"[loss-terms step] gut_sorted L1 {weights[0]} SSIM {weights[1]} {k}: exp_avg / (1 - b1) vs autograd rel-L2 {err:.2e} (bar {bar:.2e}"
              f"{f'; compact vs full rotation {floor:.2e}' if k == 'rotation' else ''})")
        assert err <= bar, k


# ---------------------------------------------------------------------------------------------------------------------------------
# fits


def _mean_composited_l1(hz, st, targets, bg=0.0):
    errs = []
    for v, t in enumerate(targets):
        rgb, alpha = hz.render(st, v)
        errs.append(float((rgb + bg * (1.0 - alpha) - t).abs().mean()))
    return float(np.mean(errs))


@pytest.mark.parametrize("kind", KINDS)
def test_fit_over_a_white_background(kind):
    hz = _Harness(kind)
    truth = hz.make(_raw_from(hz.P, hz.S))
    targets = []
    for v in range(6):
        rgb, alpha = hz.render(truth, v)
        targets.append((rgb + (1.0 - alpha)).clone())
    P2, S2 = _perturb(hz.sc, hz.P.clone(), hz.S.clone())
    fit = hz.make(_raw_from(P2, S2), background="white")
    before = _mean_composited_l1(hz, fit, targets, 1.0)
    for it in range(90):
        hz.step(fit, it % 6, targets[it % 6])
    after = _mean_composited_l1(hz, fit, targets, 1.0)
    print(f"[loss-terms fit] {kind} white: mean composited L1 over 6 views {before:.5f} -> {after:.5f} after 90 steps")
    assert np.isfinite(after) and after < 0.6 * before


@pytest.mark.parametrize("kind", KINDS)
def test_mcmc_fit_with_the_regularisers(kind):
    """The MCMC loss (base_mcmc.yaml).  A sixth of the Gaussians are floaters far below every camera, where no view constrains them, as
    in a real capture; only the regularisers act on them, so they shrink and fade, while the fit of the views is unchanged."""
    import densify

    hz = _Harness(kind)
    truth = hz.make(_raw_from(hz.P, hz.S))
    targets = [hz.render(truth, v)[0].clone() for v in range(6)]
    P2, S2 = _perturb(hz.sc, hz.P.clone(), hz.S.clone())
    gen = torch.Generator(device=hz.dev).manual_seed(9)
    k = hz.sc.n // 5
    floaters = P2[:k].clone()
    floaters[:, 0:2] = 3.0 * torch.rand((k, 2), device=hz.dev, generator=gen) - 1.5
    floaters[:, 2] = -40.0 - 5.0 * torch.rand((k,), device=hz.dev, generator=gen)   # the orbit's cameras look down at 15-35 degrees
    P2, S2 = torch.cat([P2, floaters]), torch.cat([S2, S2[:k]])
    results = {}
    for lam in (0.0, 0.01):  # base_mcmc.yaml: lambda_opacity = lambda_scale = 0.01
        conf = densify.MCMCConfig(relocate_start=5, relocate_frequency=20, add_start=5, add_frequency=20, perturb_start=0, noise_lr=5e3, seed=2)
        fit = hz.make(_raw_from(P2.clone(), S2.clone()), densify_conf=conf, lambda_opacity=lam, lambda_scale=lam)
        before = _mean_composited_l1(hz, fit, targets)
        for it in range(90):
            hz.step(fit, it % 6, targets[it % 6])
        after = _mean_composited_l1(hz, fit, targets)
        opacity = float(torch.sigmoid(fit.params["density"]).mean())
        scale = float(torch.exp(fit.params["scale"]).mean())
        results[lam] = (before, after, opacity, scale, fit.n)
        print(f"[loss-terms mcmc] {kind} lambda {lam}: N {P2.shape[0]} -> {fit.n}, mean L1 {before:.5f} -> {after:.5f}, "
              f"mean opacity {opacity:.4f}, mean scale {scale:.5f}")
    before, after, opacity, scale, _ = results[0.01]
    assert np.isfinite(after) and after < 0.6 * before
    assert opacity < results[0.0][2] and scale < results[0.0][3]


# ---------------------------------------------------------------------------------------------------------------------------------
# two ranks


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
        fit = train_step_grt.GaussianTrainStepGRT(_raw_from(*_perturb(sc, P.clone(), S.clone())), LRS, selective=True, background="random",
                                                  lambda_opacity=0.01, lambda_scale=0.01)
        first_bg = None
        for it in range(20):
            views = [vp.views_for_rank(it, r, world, 6)[0] for r in range(world)]
            positions = np.stack([fit.sensor_position(poses[v]) for v in views])
            fit.step(rays_o, rays_d, poses[views[rank]], targets[views[rank]], all_sensor_positions=positions)
            if first_bg is None:
                first_bg = fit.background.image.cpu().numpy()
        torch.cuda.synchronize(dev)
        np.savez(os.path.join(out_dir, f"rank{rank}.npz"), bg0=first_bg, **{k: v.detach().cpu().numpy() for k, v in fit.params.items()})
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_with_random_background_and_regularisers_stay_bit_identical(tmp_path):
    import torch.multiprocessing as mp

    import train_step_grt

    world = 2
    sc, rays_o, rays_d, P, S, poses = _setup()
    truth = train_step_grt.GaussianTrainStepGRT(_raw_from(P, S), LRS)
    targets = torch.stack([truth.render(rays_o, rays_d, p)[0][0] for p in poses])
    np.save(tmp_path / "targets.npy", targets.cpu().numpy())
    mp.spawn(_rank_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [np.load(tmp_path / f"rank{r}.npz") for r in range(world)]
    assert not np.array_equal(outs[0]["bg0"], outs[1]["bg0"])  # seeded background_seed + rank: the ranks draw different backgrounds
    for k in outs[0].files:
        if k != "bg0":
            assert np.array_equal(outs[0][k], outs[1][k]), k

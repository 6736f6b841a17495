"""The optimisation schedule (schedule.TrainingSchedule) inside the five training steps on the GPU: a schedule-driven run against the same
steps driven by hand from the float64 reference restatement of test_schedule.py (bit-identical parameters and Adam moments), the kernel
list of a step with and without a schedule, 90-step fits from SH degree 0 with progressive SH, and two ranks."""
import copy
import os

import numpy as np
import pytest

import scenes
from helpers import rel_l2
from test_hybrid_train_step_gpu import _setup
from test_schedule import BASE_MCMC, NHT_MCMC, _Reference, _with
from train_step import raw_params

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

KINDS = ("gut", "grt", "gut_nht", "grt_nht", "hybrid")
EXTENT = 12.5  # positions: 1.6e-4 x 12.5 = 2e-3, the rate of the other step tests
LRS_SH = dict(positions=2e-3, density=0.05, rotation=1e-3, scale=5e-3, features_albedo=1e-2, features_specular=5e-4)
LRS_NHT = dict(positions=2e-3, density=0.05, rotation=1e-3, scale=5e-3, features=2e-2, decoder=1e-3)


def _compressed(kind, max_steps=40, increase_frequency=10):
    """The reference's schedule shortened: every decay over max_steps, an SH degree more every increase_frequency steps."""
    nht = kind.endswith("nht")
    conf = copy.deepcopy(NHT_MCMC if nht else BASE_MCMC)
    for name, lr in (LRS_NHT if nht else LRS_SH).items():
        if name == "decoder":
            conf["model"]["nht_decoder"]["learning_rate"] = lr
        else:
            conf["optimizer"]["params"][name]["lr"] = lr / EXTENT if name == "positions" else lr
    conf["scheduler"]["positions"].update(lr_init=LRS_SH["positions"] / EXTENT, lr_final=LRS_SH["positions"] / EXTENT / 100, max_steps=max_steps)
    conf["scheduler"]["features"]["max_steps"] = max_steps
    conf["model"]["nht_decoder"]["scheduler"]["max_steps"] = max_steps
    return _with(conf, "model.progressive_training.increase_frequency", increase_frequency)


def _nht_step_conf():
    return {"model": {"feature_type": "nht", "nht_features": {"dim": 48, "activation": {"type": "sincos", "num_frequencies": 1},
                                                               "interpolation_type": "barycentric"}},
            "render": {"particle_feature_half": False, "pipeline_type": "referenceSlang", "backward_pipeline_type": "referenceSlangBwd"}}


class _Run:
    """C1, 600 Gaussians, 96x96, 6 views, through one of the five steps; the start is the scene with its positions, scales and colours
    perturbed, the targets are the scene rendered by a plain step at SH degree 3."""

    def __init__(self, kind, dev=None):
        self.kind = kind
        self.sc, self.rays_o, self.rays_d, self.P, self.S, self.poses, self.sensor = _setup(dev=dev)
        self.dev = self.P.device
        self.views7 = [scenes.pose7_from_c2w(self.sc.camera(i, 6)) for i in range(6)]
        rng = np.random.default_rng(5)
        self.F = torch.from_numpy(rng.uniform(-np.pi / 2, np.pi / 2, (self.sc.n, 48)).astype(np.float32)).to(self.dev)
        truth = self.make(self.raw(self.P, self.S, self.F), LRS_NHT if self.nht else LRS_SH)
        self.targets = [self.render(truth, v).clone() for v in range(6)]
        gen = torch.Generator(device=self.dev).manual_seed(0)
        self.P2, self.S2, self.F2 = self.P.clone(), self.S.clone(), self.F.clone()
        self.P2[:, 0:3] += 0.02 * torch.randn((self.sc.n, 3), device=self.dev, generator=gen)
        self.P2[:, 8:11] *= torch.exp(0.2 * torch.randn((self.sc.n, 3), device=self.dev, generator=gen))
        self.S2[:, 0:3] += 0.5 * torch.randn((self.sc.n, 3), device=self.dev, generator=gen)
        self.F2 += 0.3 * torch.randn(self.F.shape, device=self.dev, generator=gen)

    @property
    def nht(self):
        return self.kind.endswith("nht")

    def raw(self, P, S, F):
        return raw_params(P, features=F) if self.nht else raw_params(P, S)

    def start(self):
        return self.raw(self.P2, self.S2, self.F2)

    def make(self, raw, lrs, **kw):
        import train_step
        import train_step_grt
        import train_step_hybrid
        import train_step_nht

        if self.kind == "gut":
            return train_step.GaussianTrainStep(raw, lrs, **kw)
        if self.kind == "grt":
            return train_step_grt.GaussianTrainStepGRT(raw, lrs, conf={"render": {}}, **kw)
        if self.kind == "hybrid":
            return train_step_hybrid.GaussianTrainStepHybrid(raw, lrs, **kw)
        import feature_decoder as fdm

        torch.manual_seed(0)  # the same decoder weights for every step built
        decoder = fdm.FeatureDecoder(24, hidden_dim=128, num_layers=3, sh_scale=3.0).to(self.dev)
        cls = train_step_nht.GaussianTrainStepNHT if self.kind == "gut_nht" else train_step_nht.GaussianTrainStepGRTNHT
        return cls(raw, lrs, decoder, _nht_step_conf(), **kw)

    def step(self, st, v):
        t = self.targets[v]
        if self.kind in ("gut", "gut_nht"):
            return st.step(self.rays_o, self.rays_d, self.sensor, self.views7[v], t)
        if self.kind == "hybrid":
            return st.step(self.rays_o, self.rays_d, self.sensor, self.poses[v], t)
        return st.step(self.rays_o, self.rays_d, self.poses[v], t)

    def render(self, st, v):
        """rgb [H,W,3] of view v at the step's current SH degree."""
        if self.kind in ("gut", "gut_nht", "hybrid"):
            args = (self.rays_o, self.rays_d, self.sensor, self.views7[v] if self.kind != "hybrid" else self.poses[v])
        else:
            args = (self.rays_o, self.rays_d, self.poses[v])
        out = st.render(*args)[0]
        return (out[..., :3] if self.kind == "gut" else out).reshape(self.sc.height, self.sc.width, 3)


def _mcmc(**kw):
    import densify

    return densify.MCMCConfig(**{**dict(relocate_start=5, relocate_frequency=20, add_start=5, add_frequency=25, perturb_start=0,
                                        perturb_end=50, noise_lr=5e3, seed=2), **kw})


def _adam_inputs(st, args):
    """The exchanged gradients a step hands `_adam`: d_particles, d_sph / d_features and, for NHT, the decoder's."""
    tail = getattr(st.exchange, "d_tail", None)
    return [args[0], args[1]] + ([tail] if tail is not None else [])


def _state(st):
    """Parameters and both Adam moments of every group (the decoder's too)."""
    opt = st.optimizer
    out = {}
    for k in st.params:
        out[f"param.{k}"], out[f"m.{k}"], out[f"v.{k}"] = st.params[k], opt.exp_avg[k], opt.exp_avg_sq[k]
    if hasattr(opt, "decoder_exp_avg"):
        out.update({"param.decoder": opt.decoder_params, "m.decoder": opt.decoder_exp_avg, "v.decoder": opt.decoder_exp_avg_sq})
    return out


@pytest.mark.parametrize("kind", KINDS)
def test_schedule_drives_the_step_as_a_hand_loop_from_the_reference(kind):
    """Two steps run in lockstep for 60 steps under MCMC: `schedule=` against `schedule=None` with optimizer.lrs set from the reference
    restatement right after Adam (before the strategy, whose perturbation reads the position rate) and sph_degree after the step.  The
    3DGUT backward adds with float atomics, so the two backwards agree to rounding only: the hand-driven step is handed the scheduled one's
    exchanged gradients after checking they agree (which they do not if the degrees differ), so that parameters and moments stay
    bit-identical exactly when the rates, the degree and the perturbation's rate are the same."""
    import schedule

    run = _Run(kind)
    conf = _compressed(kind)
    ref = _Reference(conf, EXTENT)
    a = run.make(run.start(), None, schedule=schedule.TrainingSchedule.from_config(conf, scene_extent=EXTENT), densify_conf=_mcmc())
    b = run.make(run.start(), ref.lrs(), sph_degree=ref.n_active, densify_conf=_mcmc())
    assert a.optimizer.lrs == b.optimizer.lrs and a.sph_degree == b.sph_degree
    seen, worst = {}, [0.0]
    real_a, real_b = a._adam, b._adam

    def adam_a(*args, **kw):
        seen["grads"] = [t.clone() for t in _adam_inputs(a, args)]
        return real_a(*args, **kw)

    def adam_b(*args, **kw):
        for mine, theirs in zip(_adam_inputs(b, args), seen["grads"]):
            worst[0] = max(worst[0], rel_l2(mine.cpu(), theirs.cpu()))
            mine.copy_(theirs)
        real_b(*args, **kw)
        ref.iteration(b.frame)                 # scheduler_step(global_step), the decoder's scheduler step, progressive SH
        b.optimizer.lrs.update(ref.lrs())      # before the strategy's perturbation

    a._adam, b._adam = adam_a, adam_b
    degrees = []
    for it in range(60):
        degrees.append(a.sph_degree)
        run.step(a, it % 6)
        run.step(b, it % 6)
        b.sph_degree = ref.n_active
        assert a.n == b.n and a.optimizer.lrs == b.optimizer.lrs and a.sph_degree == b.sph_degree, it
        sa, sb = _state(a), _state(b)
        for k in sa:
            assert torch.equal(sa[k], sb[k]), f"step {it}: {k}"
    print(f"[schedule wiring {kind}] N {run.sc.n} -> {a.n}, degrees {degrees[0]}..{degrees[-1]}, worst gradient rel-L2 {worst[0]:.2e}")
    assert worst[0] <= 1e-4
    assert a.n > run.sc.n  # MCMC added Gaussians
    assert degrees == ([3] * 60 if kind.endswith("nht") else [0] * 11 + [1] * 10 + [2] * 10 + [3] * 29)
    assert a.optimizer.lrs["positions"] == pytest.approx(LRS_SH["positions"] / 100, rel=1e-12)


@pytest.mark.parametrize("kind", KINDS)
def test_a_schedule_adds_no_launch(kind):
    """torch.profiler's device activities (kernels, copies, fills) of one step with a schedule equal those of one without, in order."""
    import schedule
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    run = _Run(kind)
    mcmc = _mcmc(relocate_start=1000, add_start=1000, perturb_end=-1)  # the perturbation every step, nothing that changes N
    a = run.make(run.start(), None, schedule=schedule.TrainingSchedule.from_config(_compressed(kind), scene_extent=EXTENT), densify_conf=mcmc)
    b = run.make(run.start(), a.optimizer.lrs, sph_degree=a.sph_degree, densify_conf=mcmc)
    for it in range(2):
        run.step(a, it)
        run.step(b, it)
    b.sph_degree = a.sph_degree
    lists = []
    for st in (a, b):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run.step(st, 2)
            torch.cuda.synchronize()
        events = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA), key=lambda e: e.time_range.start)
        lists.append([e.name for e in events])
    assert len(lists[0]) > 10
    assert lists[0] == lists[1]


@pytest.mark.parametrize("kind", ["gut", "grt"])
def test_fit_from_degree_zero_with_progressive_sh(kind):
    """90 steps from SH degree 0, one degree more every 20 steps, the position rate decaying 100x over the run: the mean L1 over the six
    views (before: the start rendered at degree 3, as the targets are) falls at least as far as the constant-rate fit of
    test_train_step_gpu.py must (after < 0.6 before)."""
    import schedule

    run = _Run(kind)
    conf = _compressed(kind, max_steps=90, increase_frequency=20)
    fit = run.make(run.start(), None, schedule=schedule.TrainingSchedule.from_config(conf, scene_extent=EXTENT), lambda_l1=0.8, lambda_ssim=0.2)
    plain = run.make(run.start(), LRS_SH)

    def mean_loss(st):
        return float(np.mean([float((run.render(st, v) - run.targets[v]).abs().mean()) for v in range(6)]))

    before = mean_loss(plain)
    assert fit.sph_degree == 0
    for it in range(90):
        run.step(fit, it % 6)
    after = mean_loss(fit)
    print(f"[schedule fit {kind}] mean L1 over 6 views: {before:.5f} -> {after:.5f} after 90 steps, degree {fit.sph_degree}")
    assert fit.sph_degree == 3
    assert np.isfinite(after) and after < 0.6 * before


def _rank_worker(rank, world, port, out_dir):
    import torch.distributed as dist

    import schedule
    import view_parallel as vp

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        run = _Run("gut", dev=torch.device("cuda", rank))
        fit = run.make(run.start(), None, schedule=schedule.TrainingSchedule.from_config(_compressed("gut"), scene_extent=EXTENT),
                       densify_conf=_mcmc())
        for it in range(60):
            views = [vp.views_for_rank(it, r, world, 6)[0] for r in range(world)]
            positions = np.stack([np.asarray(run.poses[v][0, :3, 3], np.float32) for v in views])
            fit.step(run.rays_o, run.rays_d, run.sensor, run.views7[views[rank]], run.targets[views[rank]], all_sensor_positions=positions)
        torch.cuda.synchronize()
        out = {k: v.detach().cpu().numpy() for k, v in _state(fit).items()}
        np.savez(os.path.join(out_dir, f"rank{rank}.npz"), lrs=np.array([fit.optimizer.lrs[k] for k in sorted(fit.optimizer.lrs)]),
                 degree=fit.sph_degree, **out)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_with_a_schedule_and_mcmc_stay_bit_identical(tmp_path):
    import torch.multiprocessing as mp

    from test_grt_train_step_gpu import _free_port

    world = 2
    mp.spawn(_rank_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [np.load(tmp_path / f"rank{r}.npz") for r in range(world)]
    assert int(outs[0]["degree"]) == 3
    for k in outs[0].files:
        assert np.array_equal(outs[0][k], outs[1][k]), k

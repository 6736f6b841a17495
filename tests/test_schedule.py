"""The optimisation schedule (schedule.TrainingSchedule) against a float64 restatement of the reference trainer's (utils/misc.py:91-121,
model.py:819-852, trainer.py:579-596 and 1213-1262, check_step_condition) at every step of a 30,000-step run, the decoder's rates against
torch's own schedulers, progressive SH, state_dict round trips, and the schedule driving a training step's host path on a world-size-2 gloo
group (CPU stand-ins for the renderer and Adam).  No GPU."""
import copy
import json
import math
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
import torch.distributed as dist  # noqa: E402
import torch.multiprocessing as mp  # noqa: E402

from test_grt_train_exchange_gloo import _free_port  # noqa: E402

STEPS = 30000
SH = ("positions", "density", "rotation", "scale", "features_albedo", "features_specular")
NHT = ("positions", "density", "rotation", "scale", "features")

# configs/base_gs.yaml: the optimizer, scheduler, progressive-training, decoder and render keys the schedule reads
BASE_GS = {
    "n_iterations": 30000,
    "model": {"feature_type": "sh",
              "progressive_training": {"init_n_features": 0, "max_n_features": 3, "increase_frequency": 1000, "increase_step": 1},
              "nht_decoder": {"learning_rate": 0.00068, "scheduler": {"type": "cosine", "decay_final": 0.1, "max_steps": 30000}}},
    "optimizer": {"params": {"positions": {"lr": 0.00016}, "density": {"lr": 0.05}, "features_albedo": {"lr": 0.0025},
                             "features_specular": {"lr": 0.0025 / 20}, "features": {"lr": 0.015}, "rotation": {"lr": 0.001},
                             "scale": {"lr": 0.005}}},
    "scheduler": {"positions": {"type": "exp", "lr_init": 0.00016, "lr_final": 0.0000016, "max_steps": 30000},
                  "density": {"type": "skip"},
                  "features": {"type": "cosine", "decay_final": 0.1, "max_steps": 30000}},
    "render": {"particle_radiance_sph_degree": 3},
}
# configs/base_mcmc.yaml changes the initial density and scale, the loss and the strategy, none of the keys above
BASE_MCMC = copy.deepcopy(BASE_GS)
# configs/apps/colmap_3dgut_mcmc_nht.yaml (on base_mcmc, render/3dgut): model.feature_type nht
NHT_MCMC = copy.deepcopy(BASE_GS)
NHT_MCMC["model"]["feature_type"] = "nht"
CONFIGS = {"base_gs": (BASE_GS, 1.0), "base_mcmc": (BASE_MCMC, 4.25), "colmap_3dgut_mcmc_nht": (NHT_MCMC, 2.5)}


# ---- the reference, restated in float64 -----------------------------------------------------------------------------------------------

def _exponential_scheduler(lr_init, lr_final, max_steps=1000000, type=""):  # utils/misc.py:91-97
    def helper(step):
        t = np.clip(step / max_steps, 0, 1)
        return np.exp(np.log(lr_init) * (1 - t) + np.log(lr_final) * t)
    return helper


def _cosine_scheduler(lr_init, lr_final, max_steps=1000000, type=""):  # utils/misc.py:100-107
    def helper(step):
        t = np.clip(step / max_steps, 0, 1)
        return float(lr_final + 0.5 * (lr_init - lr_final) * (1 + np.cos(np.pi * t)))
    return helper


def _skip_scheduler(type="", **kwargs):  # utils/misc.py:110-114
    return lambda step: None


_SCHEDULERS = {"exp": _exponential_scheduler, "cosine": _cosine_scheduler, "skip": _skip_scheduler}


def _check_step_condition(step, start, end, freq):  # utils/misc.py:212-216
    return (start >= 0 and step > start) and (step < end or end == -1) and step % freq == 0


def _decoder_scheduler(conf, lr):
    """trainer.py:571-596 on a dummy CPU optimizer: (optimizer, torch scheduler)."""
    opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=lr)
    sc = conf["model"]["nht_decoder"]["scheduler"]
    max_steps, decay_final = int(sc.get("max_steps", conf.get("n_iterations", 30000))), float(sc.get("decay_final", 0.001))
    if sc["type"] == "exponential":
        return opt, torch.optim.lr_scheduler.ExponentialLR(opt, gamma=decay_final ** (1.0 / max_steps))
    return opt, torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=max_steps, eta_min=lr * decay_final)


class _Reference:
    """The reference's optimizer groups, schedulers, decoder scheduler and progressive SH, one `iteration(global_step)` at a time."""

    def __init__(self, conf, scene_extent):
        nht = conf["model"]["feature_type"] == "nht"
        names = NHT if nht else SH
        self.lr = {n: conf["optimizer"]["params"][n]["lr"] for n in names}
        self.lr["positions"] *= scene_extent                                   # model.py:819-820
        self.schedulers = {}
        for name, args in conf["scheduler"].items():                           # setup_scheduler, model.py:826-845
            if name not in names or args.get("type") is None:
                continue
            if name == "positions":
                self.schedulers[name] = _SCHEDULERS[args["type"]](lr_init=args["lr_init"] * scene_extent,
                                                                  lr_final=args["lr_final"] * scene_extent, max_steps=args["max_steps"])
            elif name == "features":
                lr_init = conf["optimizer"]["params"]["features"]["lr"]
                self.schedulers[name] = _SCHEDULERS[args["type"]](lr_init=lr_init, lr_final=lr_init * args.get("decay_final", 0.001),
                                                                  max_steps=args["max_steps"])
            else:
                self.schedulers[name] = _SCHEDULERS[args["type"]](**args)
        p = conf["model"]["progressive_training"]
        sh_degree = min(p["max_n_features"], conf["render"]["particle_radiance_sph_degree"])  # model.py:174-180
        self.decoder = _decoder_scheduler(conf, conf["model"]["nht_decoder"]["learning_rate"]) if nht else None
        if nht:                                                                # model.py:247-250
            self.n_active, self.progressive = sh_degree, False
        else:                                                                  # model.py:252-260
            self.n_active, self.max_n = min(p["init_n_features"], sh_degree), sh_degree
            self.progressive = self.n_active < self.max_n
            self.interval, self.increase = p["increase_frequency"], p["increase_step"]

    def lrs(self):
        out = dict(self.lr)
        if self.decoder is not None:
            out["decoder"] = self.decoder[0].param_groups[0]["lr"]
        return out

    def iteration(self, global_step):
        """What trainer.py:1213-1254 does after the optimizer step."""
        for name, sched in self.schedulers.items():                          # scheduler_step, model.py:847-852
            lr = sched(global_step)
            if lr is not None:
                self.lr[name] = lr
        if self.decoder is not None:
            self.decoder[0].step()
            self.decoder[1].step()
        if self.progressive and _check_step_condition(global_step, 0, 1e6, self.interval):
            self.n_active = min(self.max_n, self.n_active + self.increase)     # increase_num_active_features, model.py:886-887


# ---- the schedule against it ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("name", list(CONFIGS))
def test_schedule_equals_the_reference_at_every_step(name):
    import schedule

    conf, extent = CONFIGS[name]
    ref = _Reference(conf, extent)
    sched = schedule.TrainingSchedule.from_config(conf, scene_extent=extent)
    assert sched.initial_lrs() == ref.lrs() and sched.initial_sph_degree() == ref.n_active
    groups = set(NHT + ("decoder",)) if name.endswith("nht") else set(SH)
    assert set(sched.initial_lrs()) == groups
    for s in range(STEPS + 1):
        ref.iteration(s)
        lrs, degree = sched.advance(s)
        assert lrs == ref.lrs(), f"step {s}"
        assert degree == ref.n_active, f"step {s}"


def test_position_rate_reaches_the_mcmc_perturbation_decayed():
    """The rate the MCMC perturbation reads after iteration s is sched(s): at the perturbation's last step (27,500) 1 / 68 of the first."""
    import schedule

    sched = schedule.TrainingSchedule.from_config(BASE_MCMC, scene_extent=1.0)
    first = sched.initial_lrs()["positions"]
    for s in range(27501):
        lrs, _ = sched.advance(s)
    assert lrs["positions"] == pytest.approx(1.6e-4 * 100.0 ** (-27500 / 30000), rel=1e-12)
    assert 68.0 < first / lrs["positions"] < 68.2


@pytest.mark.parametrize("kind", ["cosine", "exponential"])
@pytest.mark.parametrize("decay_final,max_steps", [(0.1, 30000), (0.001, 7000)])
def test_decoder_rate_is_the_torch_scheduler(kind, decay_final, max_steps):
    """After iteration s the decoder's rate is torch's after s + 1 scheduler steps, past max_steps too (the cosine's second half-period)."""
    import schedule

    conf = copy.deepcopy(NHT_MCMC)
    conf["model"]["nht_decoder"]["scheduler"] = {"type": kind, "decay_final": decay_final, "max_steps": max_steps}
    sched = schedule.TrainingSchedule.from_config(conf)
    opt, torch_sched = _decoder_scheduler(conf, 0.00068)
    assert sched.initial_lrs()["decoder"] == opt.param_groups[0]["lr"]
    for s in range(STEPS):
        opt.step()
        torch_sched.step()
        want = opt.param_groups[0]["lr"]
        got = sched.advance(s)[0]["decoder"]
        assert got == want or abs(got - want) <= 1e-12 * abs(want), f"step {s}: {got!r} vs {want!r}"


def _degrees(conf, steps=4200):
    """The SH degree each step 0..steps-1 renders at."""
    import schedule

    sched = schedule.TrainingSchedule.from_config(conf)
    out = [sched.initial_sph_degree()]
    for s in range(steps - 1):
        out.append(sched.advance(s)[1])
    return np.array(out)


def _with(conf, path, value):
    conf = copy.deepcopy(conf)
    cur = conf
    keys = path.split(".")
    for k in keys[:-1]:
        cur = cur.setdefault(k, {})
    cur[keys[-1]] = value
    return conf


def test_sh_degree_goes_up_after_every_increase_step_and_stops_at_three():
    d = _degrees(BASE_GS)
    assert (d[:1001] == 0).all() and (d[1001:2001] == 1).all() and (d[2001:3001] == 2).all() and (d[3001:] == 3).all()


def test_sh_degree_is_clamped_to_the_rendered_degree_and_follows_the_increment():
    assert _degrees(_with(BASE_GS, "render.particle_radiance_sph_degree", 1)).max() == 1
    assert set(_degrees(_with(BASE_GS, "render.particle_radiance_sph_degree", 1))[1001:]) == {1}
    assert (_degrees(_with(BASE_GS, "model.progressive_training.init_n_features", 5)) == 3).all()   # starts at the cap: no progression
    two = _degrees(_with(BASE_GS, "model.progressive_training.increase_step", 2))
    assert (two[:1001] == 0).all() and (two[1001:2001] == 2).all() and (two[2001:] == 3).all()
    fast = _degrees(_with(BASE_GS, "model.progressive_training.increase_frequency", 10), steps=60)
    assert list(fast[[0, 10, 11, 20, 21, 30, 31, 59]]) == [0, 0, 1, 1, 2, 2, 3, 3]


def test_nht_renders_every_feature_from_the_first_step():
    d = _degrees(NHT_MCMC)
    assert (d == 3).all()
    assert (_degrees(_with(NHT_MCMC, "model.progressive_training.init_n_features", 1)) == 3).all()


def test_scene_extent_scales_the_position_rate_only():
    import schedule

    a = schedule.TrainingSchedule.from_config(NHT_MCMC, scene_extent=1.0)
    b = schedule.TrainingSchedule.from_config(NHT_MCMC, scene_extent=3.7)
    for s in [None] + list(range(0, 30001, 997)):
        la, lb = (a.initial_lrs(), b.initial_lrs()) if s is None else (a.advance(s)[0], b.advance(s)[0])
        assert lb["positions"] == pytest.approx(3.7 * la["positions"], rel=1e-12)
        assert {k: v for k, v in la.items() if k != "positions"} == {k: v for k, v in lb.items() if k != "positions"}


def test_unknown_scheduler_types_are_refused_by_key():
    import schedule

    with pytest.raises(KeyError, match="scheduler.positions.type"):
        schedule.TrainingSchedule.from_config(_with(BASE_GS, "scheduler.positions.type", "linear"))
    with pytest.raises(KeyError, match="scheduler.features.type"):
        schedule.TrainingSchedule.from_config(_with(NHT_MCMC, "scheduler.features.type", "step"))
    with pytest.raises(ValueError, match="model.nht_decoder.scheduler.type"):
        schedule.TrainingSchedule.from_config(_with(NHT_MCMC, "model.nht_decoder.scheduler.type", "exp"))
    # the reference schedules only the parameters the model has: an SH model ignores scheduler.features and the decoder
    sched = schedule.TrainingSchedule.from_config(_with(_with(BASE_GS, "scheduler.features.type", "step"),
                                                        "model.nht_decoder.scheduler.type", "step"))
    assert "features" not in sched.initial_lrs()
    # a `null` type schedules nothing (model.py:836-837)
    frozen = schedule.TrainingSchedule.from_config(_with(BASE_GS, "scheduler.positions.type", None))
    assert frozen.advance(20000)[0]["positions"] == BASE_GS["optimizer"]["params"]["positions"]["lr"]


@pytest.mark.parametrize("name", list(CONFIGS))
def test_state_dict_round_trip_continues_identically(name):
    import schedule

    conf, extent = CONFIGS[name]
    run = schedule.TrainingSchedule.from_config(conf, scene_extent=extent)
    for s in range(1500):
        run.advance(s)
    state = json.loads(json.dumps(run.state_dict()))  # plain data
    resumed = schedule.TrainingSchedule.from_config(conf, scene_extent=extent)
    resumed.load_state_dict(state)
    assert resumed.initial_lrs() == run.initial_lrs() and resumed.initial_sph_degree() == run.initial_sph_degree()
    assert state["step"] == 1500
    for s in range(1500, 6000):
        assert resumed.advance(s) == run.advance(s)
    with pytest.raises(ValueError, match="groups"):
        other = "colmap_3dgut_mcmc_nht" if name != "colmap_3dgut_mcmc_nht" else "base_gs"
        schedule.TrainingSchedule.from_config(CONFIGS[other][0]).load_state_dict(state)


# ---- the schedule in a training step's host path ----------------------------------------------------------------------------------------

N = 64
COMPRESSED = _with(_with(_with(BASE_MCMC, "scheduler.positions.max_steps", 40), "model.progressive_training.increase_frequency", 10),
                   "optimizer.params.positions.lr", 0.0016)
COMPRESSED["scheduler"]["positions"]["lr_init"] = 0.0016


class _SGD:
    """CPU stand-in for FusedGaussianAdam: p -= lr g on the exchanged gradients; records the rates of every step."""

    selective = False

    def __init__(self, params, lrs):
        self.params, self.lrs = params, {k: float(lrs[k]) for k in SH}
        self.exp_avg = {k: torch.zeros_like(v) for k, v in params.items()}
        self.exp_avg_sq = {k: torch.zeros_like(v) for k, v in params.items()}
        self.used = []

    def step(self, d_particles, d_sph, visibility=None, **reg):
        self.used.append([self.lrs[k] for k in SH])
        grads = {"positions": d_particles[:, 0:3], "density": d_particles[:, 3:4], "rotation": d_particles[:, 4:8],
                 "scale": d_particles[:, 8:11], "features_albedo": d_sph[:, 0:3], "features_specular": d_sph[:, 3:48]}
        for k, g in grads.items():
            self.params[k].sub_(self.lrs[k] * g)


def _cpu_step_class():
    import train_step
    import view_parallel

    class CPUStep(train_step.TrainStep):
        """TrainStep's host path with no renderer: the caller writes the view's gradients into exchange.out()."""

        def _init_renderer(self, conf):
            pass

        def _new_exchange(self):
            return view_parallel.FlatGradientExchange(self.n, self.device, group=self.group)

        def _new_optimizer(self, lrs, eps, selective):
            return _SGD(self.params, lrs)

    return CPUStep


def _params(seed=0):
    g = torch.Generator().manual_seed(seed)
    return {"positions": torch.randn(N, 3, generator=g), "density": torch.randn(N, 1, generator=g) - 3.0,
            "rotation": torch.randn(N, 4, generator=g), "scale": torch.randn(N, 3, generator=g) - 3.0,
            "features_albedo": torch.randn(N, 3, generator=g), "features_specular": torch.randn(N, 45, generator=g)}


def test_a_step_takes_the_schedule_and_refuses_an_explicit_degree_with_it():
    import schedule

    CPUStep = _cpu_step_class()
    sched = schedule.TrainingSchedule.from_config(BASE_GS)
    with pytest.raises(ValueError, match="sph_degree"):
        CPUStep(_params(), None, sph_degree=3, schedule=sched)
    with pytest.raises(ValueError, match="schedule"):
        CPUStep(_params(), None, schedule=schedule.TrainingSchedule.from_config(NHT_MCMC))
    with pytest.raises(ValueError, match="lrs"):
        CPUStep(_params(), None)
    step = CPUStep(_params(), {k: 1.0 for k in SH}, schedule=sched)
    assert step.optimizer.lrs == sched.initial_lrs() and step.sph_degree == 0
    plain = CPUStep(_params(), {k: 1.0 for k in SH})
    assert plain.schedule is None and plain.sph_degree == 3 and plain.optimizer.lrs == {k: 1.0 for k in SH}


STEPS_GLOO = 60


def _worker(rank, world, port, out_dir):
    import densify
    import schedule

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    CPUStep = _cpu_step_class()
    mcmc = densify.MCMCConfig(relocate_start=5, relocate_frequency=20, add_start=5, add_frequency=25, perturb_start=0, perturb_end=50,
                              noise_lr=5e3, seed=3)
    step = CPUStep(_params(), None, schedule=schedule.TrainingSchedule.from_config(COMPRESSED, scene_extent=2.0), densify_conf=mcmc)
    perturbed = []
    real_perturb = step.densifier.perturb

    def recording_perturb(positions_lr):
        perturbed.append((step.frame, positions_lr))
        return real_perturb(positions_lr)

    step.densifier.perturb = recording_perturb
    degrees = []
    g = torch.Generator().manual_seed(100 + rank)  # each rank's own view
    for _ in range(STEPS_GLOO):
        degrees.append(step.sph_degree)
        d_particles, d_sph = step.exchange.out()
        d_particles.copy_(1e-2 * torch.randn(d_particles.shape, generator=g))
        d_sph.copy_(1e-2 * torch.randn(d_sph.shape, generator=g))
        step._update(torch.zeros(()), None, None, np.zeros((world, 3), np.float32), np.zeros(3, np.float32))
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), degrees=np.array(degrees), used=np.array(step.optimizer.used),
             perturbed=np.array(perturbed), n=step.n, **{k: v.numpy() for k, v in step.params.items()})
    dist.destroy_process_group()


def test_replicas_agree_on_rates_and_degree_at_every_step(tmp_path):
    import schedule

    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [np.load(tmp_path / f"rank{r}.npz") for r in range(world)]
    for key in ("degrees", "used", "perturbed", "n") + SH:
        a, b = np.atleast_1d(outs[0][key]), np.atleast_1d(outs[1][key])
        assert a.shape == b.shape and a.tobytes() == b.tobytes(), key
    assert int(outs[0]["n"]) > N  # MCMC added Gaussians: the exchange followed
    # the rates and degree of every step are the schedule's, and the perturbation at frame s + 1 read sched(s)
    sched = schedule.TrainingSchedule.from_config(COMPRESSED, scene_extent=2.0)
    want_lrs, want_deg = [[sched.initial_lrs()[k] for k in SH]], [sched.initial_sph_degree()]
    for s in range(STEPS_GLOO - 1):
        lrs, deg = sched.advance(s)
        want_lrs.append([lrs[k] for k in SH])
        want_deg.append(deg)
    assert outs[0]["used"].tolist() == want_lrs and outs[0]["degrees"].tolist() == want_deg
    assert want_deg[:12] == [0] * 11 + [1] and want_deg[-1] == 3
    perturbed = outs[0]["perturbed"]
    assert len(perturbed) == 49  # frames 1..49 (perturb_end 50)
    for frame, lr in perturbed:
        assert lr == want_lrs[int(frame)][0]
    assert math.isclose(perturbed[-1][1], 2.0 * 0.0000016, rel_tol=1e-12)  # past max_steps 40: the final rate

"""Checkpoints (checkpoint.py, TrainStep.state_dict / load_state_dict) without a GPU: step state -> the reference's ckpt_*.pt layout ->
step state round trips bit for bit; the layout's optimizer, parameter and decoder sections load into torch's own Adam, schedulers and
nn.Parameter attributes the way the reference's loaders load them; a reference-only checkpoint (no extras) rebuilds the schedule at
global_step; refusals name their key; a TrainStep's host path (CPU stand-ins for the renderer and Adam) saves and resumes, on one rank and
on a world-size-2 gloo group with per-rank background generators."""
import copy
import io
import os

import numpy as np
import pytest

torch = pytest.importorskip("torch")
import torch.distributed as dist  # noqa: E402
import torch.multiprocessing as mp  # noqa: E402

from test_grt_train_exchange_gloo import _free_port  # noqa: E402
from test_schedule import BASE_GS, BASE_MCMC, NHT_MCMC, _with  # noqa: E402

SH = {"positions": 3, "density": 1, "rotation": 4, "scale": 3, "features_albedo": 3, "features_specular": 45}
NHT = {"positions": 3, "density": 1, "rotation": 4, "scale": 3, "features": 48}
GEOMETRY = ("positions", "density", "rotation", "scale")
DECODER_PARAMS = 300
ARCH = {"ray_feature_dim": 24, "hidden_dim": 128, "num_layers": 3, "sh_scale": 3.0, "output_activation": "Sigmoid", "unpremultiply_alpha": False}
EXTENT = 2.5


def _state(ft="sh", strategy="gs", progressive=True, frozen=False, frame=37, n=50, seed=0, conf=None):
    """A step state as TrainStep.state_dict gives it, on the CPU, with a schedule of `conf` (base_gs / the NHT config by default)."""
    import schedule

    g = torch.Generator().manual_seed(seed)
    widths = NHT if ft == "nht" else SH
    if conf is None:
        conf = NHT_MCMC if ft == "nht" else BASE_GS
        if not progressive:
            conf = _with(conf, "model.progressive_training.init_n_features", 3)
    sched = schedule.TrainingSchedule.from_config(conf, scene_extent=EXTENT).advance_to(frame)
    steps = {k: frame for k in widths}
    if frozen:  # colour refinement froze the geometry 7 steps ago
        steps.update({k: frame - 7 for k in GEOMETRY})
    settings = {"selective": False, "eps": 1e-15, "lambda_l1": 0.8, "lambda_ssim": 0.2, "lambda_opacity": 0.0, "lambda_scale": 0.0,
                "background": "random", "post_processing": None, "strategy": strategy}
    dens = None
    if strategy == "gs":
        dens = {"grad_norm_accum": torch.rand(n, 1, generator=g), "grad_norm_denom": torch.randint(0, 9, (n, 1), generator=g, dtype=torch.int32),
                "generator": torch.Generator().manual_seed(3 + seed).get_state()}
    elif strategy == "mcmc":
        dens = {"generator": torch.Generator().manual_seed(4 + seed).get_state()}
    state = {"feature_type": ft, "settings": settings, "frame": frame, "sph_degree": sched.sph_degree, "scene_extent": EXTENT,
             "lrs": dict(sched.lrs), "progression": None if sched.progression is None else list(sched.progression),
             "params": {k: torch.randn(n, w, generator=g) for k, w in widths.items()},
             "exp_avg": {k: 1e-3 * torch.randn(n, w, generator=g) for k, w in widths.items()},
             "exp_avg_sq": {k: 1e-6 * torch.rand(n, w, generator=g) for k, w in widths.items()},
             "adam_steps": steps, "densifier": dens, "background_generator": torch.Generator().manual_seed(9 + seed).get_state(),
             "schedule": sched.state_dict()}
    if ft == "nht":
        settings.update(decoder_weight_decay=0.0, color_refine_start=frame - 7 if frozen else None)
        state["adam_steps"]["decoder"] = frame
        dec = sched.decoder
        state["decoder"] = {"params": torch.randn(DECODER_PARAMS, generator=g), "exp_avg": 1e-3 * torch.randn(DECODER_PARAMS, generator=g),
                            "exp_avg_sq": 1e-6 * torch.rand(DECODER_PARAMS, generator=g), "ema": {"network.params": torch.randn(DECODER_PARAMS, generator=g)},
                            "arch": dict(ARCH), "scheduler": {"type": "cosine", "base_lr": dec.base_lr, "max_steps": dec.max_steps, "eta_min": dec.eta_min}}
    return state


def _same(a, b, path="state"):
    if isinstance(a, torch.Tensor):
        assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), path
    elif isinstance(a, dict):
        assert isinstance(b, dict) and set(a) == set(b), f"{path}: keys {sorted(a)} vs {sorted(b)}"
        for k in a:
            _same(a[k], b[k], f"{path}.{k}")
    elif isinstance(a, (list, tuple)):
        assert isinstance(b, (list, tuple)) and len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, f"{path}[{i}]")
    else:
        assert type(a) is type(b) and a == b, f"{path}: {a!r} vs {b!r}"


def _through_file(ckpt):
    buf = io.BytesIO()
    torch.save(ckpt, buf)
    buf.seek(0)
    return torch.load(buf, weights_only=True)  # plain data throughout when the config is a dict or None


CASES = [("sh", "gs", True, False), ("sh", "mcmc", False, False), ("sh", None, True, False), ("nht", "mcmc", False, False),
         ("nht", "gs", False, True), ("nht", None, False, True)]


@pytest.mark.parametrize("ft,strategy,progressive,frozen", CASES)
def test_state_round_trips_through_the_reference_layout(ft, strategy, progressive, frozen):
    import checkpoint

    state = _state(ft, strategy, progressive, frozen)
    ckpt = checkpoint.reference_layout(state, conf=None, epoch=3)
    _same(checkpoint.from_reference_layout(ckpt, feature_type=ft), state)
    _same(checkpoint.from_reference_layout(_through_file(ckpt), feature_type=ft), state)
    assert ckpt["global_step"] == 37 and ckpt["epoch"] == 3 and ckpt["feature_type"] == ft and ckpt["background"] == {}
    assert ckpt["progressive_training"] == (progressive and ft == "sh")
    if ft == "sh":
        assert ckpt["n_active_features"] == state["sph_degree"] and ckpt["max_n_features"] == 3
        assert ("feature_dim_increase_interval" in ckpt) == progressive
    else:
        assert ckpt["n_active_features"] == ckpt["max_n_features"] == ckpt["ray_feature_dim"] == 24
    assert ("densify_grad_norm_accum" in ckpt) == (strategy == "gs")
    if strategy == "gs":
        assert isinstance(ckpt["densify_grad_norm_accum"], tuple) and len(ckpt["densify_grad_norm_denom"]) == 1
    # the tensors are the state's own: nothing is copied on the way to torch.save
    assert ckpt["positions"].data_ptr() == state["params"]["positions"].data_ptr()


def _reference_adam(model_params: dict, conf, extent):
    """setup_optimizer (model.py:782-826) over nn.Parameters: groups in conf.optimizer.params order, fused Adam, positions x extent."""
    groups = [{"params": [model_params[k]], "name": k, **conf["optimizer"]["params"][k]} for k in conf["optimizer"]["params"] if k in model_params]
    opt = torch.optim.Adam(groups, lr=0.0, eps=1e-15, fused=True)
    for g in opt.param_groups:
        if g["name"] == "positions":
            g["lr"] *= extent
    return opt


@pytest.mark.parametrize("ft,frozen", [("sh", False), ("nht", True)])
def test_optimizer_section_steps_a_real_adam_with_the_exported_moments_and_count(ft, frozen):
    import checkpoint

    conf = NHT_MCMC if ft == "nht" else BASE_GS
    state = _state(ft, "mcmc", frame=12, frozen=frozen)
    ckpt = _through_file(checkpoint.reference_layout(state, conf=conf))
    names = [g["name"] for g in ckpt["optimizer"]["param_groups"]]
    assert names == [k for k in conf["optimizer"]["params"] if k in state["params"]]
    counts = {k: int(ckpt["optimizer"]["state"][i]["step"]) for i, k in enumerate(names)}
    assert counts == {k: state["adam_steps"][k] for k in names}  # frozen NHT geometry: the count it froze at (5, features 12)
    model = {k: torch.nn.Parameter(ckpt[k].detach().clone()) for k in names}
    opt = _reference_adam(model, conf, EXTENT)
    opt.load_state_dict(ckpt["optimizer"])
    assert {g["name"]: g["lr"] for g in opt.param_groups} == {k: state["lrs"][k] for k in names}
    g = torch.Generator().manual_seed(11)
    grads = {k: torch.randn(p.shape, generator=g) for k, p in model.items()}
    for k, p in model.items():
        p.grad = grads[k].clone()
    before = {k: p.detach().clone() for k, p in model.items()}
    opt.step()
    b1, b2, eps = 0.9, 0.999, 1e-15
    off_by_one = 0.0
    for k, p in model.items():
        m = b1 * state["exp_avg"][k].double() + (1 - b1) * grads[k].double()
        v = b2 * state["exp_avg_sq"][k].double() + (1 - b2) * grads[k].double() ** 2

        def adam(t):
            return before[k].double() - state["lrs"][k] * (m / (1 - b1 ** t)) / ((v / (1 - b2 ** t)).sqrt() + eps)

        err = float((p.detach().double() - adam(state["adam_steps"][k] + 1)).abs().max())
        assert err <= 1e-6, f"{k}: {err}"
        off_by_one = max(off_by_one, float((p.detach().double() - adam(state["adam_steps"][k] + 2)).abs().max()))
    assert off_by_one > 1e-5  # the comparison sees the bias-correction count


def test_parameters_assign_to_module_parameters_as_init_from_checkpoint_does():
    import checkpoint

    for ft in ("sh", "nht"):
        ckpt = checkpoint.reference_layout(_state(ft, "gs"))
        module = torch.nn.Module()
        for k in (NHT if ft == "nht" else SH):
            setattr(module, k, torch.nn.Parameter(torch.empty(0, 1)))
            setattr(module, k, ckpt[k])  # a plain tensor raises here
            assert isinstance(getattr(module, k), torch.nn.Parameter) and getattr(module, k).requires_grad
        with pytest.raises(TypeError):
            module.positions = ckpt["positions"].detach()


@pytest.mark.parametrize("kind", ["cosine", "exponential"])
def test_decoder_sections_load_into_torch_and_the_rate_is_the_schedules(kind):
    import checkpoint
    import schedule

    conf = copy.deepcopy(NHT_MCMC)
    conf["model"]["nht_decoder"]["scheduler"] = {"type": kind, "decay_final": 0.01, "max_steps": 400}
    state = _state("nht", "mcmc", conf=conf, frame=250)
    dec = schedule.TrainingSchedule.from_config(conf, scene_extent=EXTENT).decoder
    state["decoder"]["scheduler"] = ({"type": "cosine", "base_lr": dec.base_lr, "max_steps": dec.max_steps, "eta_min": dec.eta_min}
                                     if kind == "cosine" else {"type": "exponential", "base_lr": dec.base_lr, "gamma": dec.gamma})
    fd = _through_file(checkpoint.reference_layout(state, conf=conf))["feature_decoder"]
    assert set(fd) == {"module", "optimizer", "scheduler", "arch", "ema"} and fd["arch"] == ARCH
    # trainer.py:571-596, then setup_training's restore (:287-296)
    p = torch.nn.Parameter(torch.zeros(DECODER_PARAMS))
    lr = conf["model"]["nht_decoder"]["learning_rate"]
    opt = torch.optim.Adam([p], lr=lr, weight_decay=0.0)
    if kind == "cosine":
        sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=400, eta_min=lr * 0.01)
    else:
        sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=0.01 ** (1.0 / 400))
    p.data.copy_(fd["module"]["network.params"])
    opt.load_state_dict(fd["optimizer"])
    sched.load_state_dict(fd["scheduler"])
    assert sched.last_epoch == 250
    assert sched.get_last_lr() == [state["lrs"]["decoder"]] and opt.param_groups[0]["lr"] == state["lrs"]["decoder"]
    st = opt.state[p]
    assert int(st["step"]) == 250 and torch.equal(st["exp_avg"], state["decoder"]["exp_avg"])
    # the reference continues at the rate the schedule gives next
    run = schedule.TrainingSchedule.from_config(conf, scene_extent=EXTENT).advance_to(250)
    p.grad = torch.zeros_like(p)
    opt.step()
    sched.step()
    want = run.advance(250)[0]["decoder"]
    assert abs(sched.get_last_lr()[0] - want) <= 1e-12 * want


@pytest.mark.parametrize("name", ["base_gs", "base_mcmc", "colmap_3dgut_mcmc_nht"])
def test_reference_only_checkpoint_rebuilds_the_schedule_at_global_step(name):
    import checkpoint
    import schedule
    from test_schedule import CONFIGS

    conf, extent = CONFIGS[name]
    ft = "nht" if name.endswith("nht") else "sh"
    frame = 2345
    state = _state(ft, "gs" if name == "base_gs" else "mcmc", conf=conf, frame=frame)
    state["scene_extent"] = extent
    ckpt = checkpoint.reference_layout(state, conf=conf)
    del ckpt[checkpoint.EXTRAS]
    back = checkpoint.from_reference_layout(ckpt, feature_type=ft)
    stepwise = schedule.TrainingSchedule.from_config(conf, scene_extent=extent, feature_type=ft)
    for s in range(frame):
        stepwise.advance(s)
    _same(back["schedule"], stepwise.state_dict(), "schedule")
    assert back["settings"] == {} and back["background_generator"] is None
    assert back["adam_steps"] == {k: frame for k in (NHT if ft == "nht" else SH)} | ({"decoder": frame} if ft == "nht" else {})
    if name == "base_gs":
        assert back["densifier"]["generator"] is None and torch.equal(back["densifier"]["grad_norm_accum"], state["densifier"]["grad_norm_accum"])
    else:
        assert back["densifier"] is None  # MCMC writes nothing
    assert back["sph_degree"] == (state["sph_degree"] if ft == "sh" else None)
    for k in back["params"]:
        assert torch.equal(back["params"][k], state["params"][k]) and torch.equal(back["exp_avg_sq"][k], state["exp_avg_sq"][k])


def test_refusals_name_their_key():
    import checkpoint

    sh = checkpoint.reference_layout(_state("sh", "gs"))
    with pytest.raises(ValueError, match="feature_type"):
        checkpoint.from_reference_layout(sh, feature_type="nht")
    nht = checkpoint.reference_layout(_state("nht", "mcmc"))
    nht["features"] = torch.nn.Parameter(torch.zeros(50, 32))
    with pytest.raises(ValueError, match="particle_feature_dim"):
        checkpoint.from_reference_layout(nht, feature_type="nht")
    uneven = checkpoint.reference_layout(_state("sh", "gs"))
    del uneven[checkpoint.EXTRAS]
    idx = [g["name"] for g in uneven["optimizer"]["param_groups"]].index("scale")
    uneven["optimizer"]["state"][idx]["step"].fill_(12.0)
    with pytest.raises(ValueError, match="'scale'"):
        checkpoint.from_reference_layout(uneven)
    frozen = checkpoint.reference_layout(_state("nht", "mcmc", frozen=True))
    frozen[checkpoint.EXTRAS]["adam_steps"]["rotation"] = 5
    with pytest.raises(ValueError, match="'rotation'"):
        checkpoint.from_reference_layout(frozen)
    pp = checkpoint.reference_layout(_state("sh", "gs"))
    pp["post_processing"] = {"module": {}, "optimizers": [], "schedulers": []}
    with pytest.raises(NotImplementedError, match="post_processing.method"):
        checkpoint.from_reference_layout(pp)


# ---- a TrainStep's host path ------------------------------------------------------------------------------------------------------------

class _Adam:
    """CPU stand-in for FusedGaussianAdam's state (the step never runs it here)."""

    def __init__(self, params, lrs, eps, selective):
        self.params, self.lrs, self.eps, self.selective = params, {k: float(lrs[k]) for k in SH}, float(eps), bool(selective)
        self.exp_avg = {k: torch.zeros_like(v) for k, v in params.items()}
        self.exp_avg_sq = {k: torch.zeros_like(v) for k, v in params.items()}
        self.steps = 0


def _cpu_step_class():
    import train_step
    import view_parallel

    class CPUStep(train_step.TrainStep):
        def _init_renderer(self, conf):
            pass

        def _new_exchange(self):
            return view_parallel.FlatGradientExchange(self.n, self.device, group=self.group)

        def _new_optimizer(self, lrs, eps, selective):
            return _Adam(self.params, lrs, eps, selective)

    return CPUStep


def _params(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(n, w, generator=g) for k, w in SH.items()}


def _make(n=40, seed=0, **kw):
    import densify
    import schedule

    kw = {"background": "random", "background_seed": 5, "densify_conf": densify.DensifyConfig(seed=1),
          "schedule": schedule.TrainingSchedule.from_config(BASE_MCMC, scene_extent=EXTENT), "scene_extent": EXTENT, **kw}
    lrs = None if kw["schedule"] is not None else {k: 1e-3 for k in SH}
    return _cpu_step_class()(_params(n, seed), lrs, **kw)


def _advance(step, frames, seed):
    """Change every piece of state a step carries, as training would."""
    g = torch.Generator().manual_seed(seed)
    for k in SH:
        step.optimizer.exp_avg[k].copy_(torch.randn(step.optimizer.exp_avg[k].shape, generator=g))
        step.optimizer.exp_avg_sq[k].copy_(torch.rand(step.optimizer.exp_avg_sq[k].shape, generator=g))
    for s in range(frames):
        lrs, step.sph_degree = step.schedule.advance(s)
        step.optimizer.lrs.update(lrs)
        step.background.draw(4, 5)
    step.frame = frames
    step.optimizer.steps = frames
    step.densifier.grad_norm_accum += torch.rand(step.densifier.grad_norm_accum.shape, generator=g)
    step.densifier.grad_norm_denom += 2
    torch.randn(3, generator=step.densifier.generator)


def test_a_step_resumes_its_own_state_with_another_n_and_refuses_other_settings():
    a = _make(n=40)
    _advance(a, 1200, seed=1)
    b = _make(n=25, seed=7)
    b.load_state_dict(a.state_dict())
    _same(b.state_dict(), a.state_dict())
    assert b.n == 40 and b.exchange.n == 40 and b.sph_degree == 1
    assert b.params["positions"].data_ptr() != a.params["positions"].data_ptr()  # copied
    assert b.densifier.params is b.params and b.densifier.moments[0] is b.optimizer.exp_avg  # the shared dicts stay shared
    c = _make(n=25, seed=7)
    c.load_state_dict(a.state_dict(), assign=True)
    assert c.params["positions"].data_ptr() == a.params["positions"].data_ptr()  # taken as they are
    # the same draws from here on
    assert torch.equal(a.background.draw(4, 5), b.background.draw(4, 5))
    for key, value in (("selective", True), ("lambda_ssim", 0.2), ("background", "white"), ("post_processing", "linear-to-srgb")):
        other = _make(n=25, **{key: value})
        with pytest.raises(ValueError, match=key):
            other.load_state_dict(a.state_dict())
        assert other.n == 25  # refused before anything changed
    with pytest.raises(ValueError, match="feature_type"):
        _make().load_state_dict(_state("nht", "gs"))
    import densify

    with pytest.raises(ValueError, match="strategy"):
        _make(densify_conf=densify.MCMCConfig()).load_state_dict(a.state_dict())


def test_a_step_resumes_from_a_reference_only_checkpoint():
    import checkpoint

    a = _make(n=40)
    _advance(a, 1500, seed=2)
    ckpt = checkpoint.reference_layout(a.state_dict(), conf=BASE_MCMC)
    del ckpt[checkpoint.EXTRAS]
    b = _make(n=10)
    b.load_state_dict(checkpoint.from_reference_layout(ckpt, feature_type="sh"))
    fresh = _make(n=10)
    assert b.schedule.state_dict() == a.schedule.state_dict() and b.optimizer.lrs == a.optimizer.lrs and b.sph_degree == a.sph_degree
    assert torch.equal(b.background.generator.get_state(), fresh.background.generator.get_state())  # re-seeded
    assert torch.equal(b.densifier.generator.get_state(), fresh.densifier.generator.get_state())
    assert torch.equal(b.densifier.grad_norm_accum, a.densifier.grad_norm_accum) and b.optimizer.steps == 1500
    # a step given no schedule state and no config replays its own fresh schedule to the frame
    del ckpt["config"]
    c = _make(n=10)
    state = checkpoint.from_reference_layout(ckpt)
    assert state["schedule"] is None
    c.load_state_dict(state)
    assert c.schedule.state_dict() == a.schedule.state_dict()
    stale = _make(n=10)
    stale.schedule.advance_to(2000)
    with pytest.raises(ValueError, match="schedule"):
        stale.load_state_dict(state)


def test_save_and_load_files_on_one_rank(tmp_path):
    import checkpoint

    a = _make(n=40)
    _advance(a, 300, seed=3)
    path = str(tmp_path / "ckpt_300.pt")
    checkpoint.save(a, path, conf=BASE_MCMC, epoch=2)
    assert os.listdir(tmp_path) == ["ckpt_300.pt"]
    b = _make(n=12)
    ckpt = checkpoint.load(path, b, weights_only=True)
    _same(b.state_dict(), a.state_dict())
    assert ckpt["epoch"] == 2 and ckpt["config"] == BASE_MCMC and ckpt[checkpoint.EXTRAS]["background_generators"][0] is not None


def _rank_worker(rank, world, port, out_dir):
    import checkpoint

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        a = _make(n=40)
        _advance(a, 100 + 10 * rank, seed=4)  # the same parameters; each rank's background has drawn a different number of times
        a.frame, a.optimizer.steps = 100, 100
        a.schedule = None
        a.sph_degree = 3
        path = os.path.join(out_dir, "ckpt.pt")
        checkpoint.save(a, path)
        b = _make(n=12, schedule=None)
        checkpoint.load(path, b)
        np.save(os.path.join(out_dir, f"saved{rank}.npy"), a.background.generator.get_state().numpy())
        np.save(os.path.join(out_dir, f"loaded{rank}.npy"), b.background.generator.get_state().numpy())
    finally:
        dist.destroy_process_group()


def test_two_ranks_restore_their_own_background_and_reseed_on_another_world_size(tmp_path):
    import checkpoint

    world = 2
    mp.spawn(_rank_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    saved = [np.load(tmp_path / f"saved{r}.npy") for r in range(world)]
    loaded = [np.load(tmp_path / f"loaded{r}.npy") for r in range(world)]
    assert not np.array_equal(saved[0], saved[1])
    for r in range(world):
        assert np.array_equal(saved[r], loaded[r]), r
    # one rank reading the two-rank file: re-seeded (background_seed + rank)
    one = _make(n=12, schedule=None)
    checkpoint.load(str(tmp_path / "ckpt.pt"), one)
    assert torch.equal(one.background.generator.get_state(), _make(schedule=None).background.generator.get_state())
    assert len(torch.load(tmp_path / "ckpt.pt", weights_only=True)[checkpoint.EXTRAS]["background_generators"]) == 2

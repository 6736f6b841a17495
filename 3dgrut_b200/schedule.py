"""The optimisation schedule of the reference trainer as pure host logic: the learning-rate schedulers of the Gaussian groups
(`scheduler.*`, model.py:832-852, utils/misc.py:91-121), the NHT decoder's torch scheduler (`model.nht_decoder.scheduler`,
trainer.py:579-596) and progressive SH (`model.progressive_training`, model.py:174-180,245-260, trainer.py:1250-1254).

A training step takes a `TrainingSchedule` (`schedule=`) and calls `advance(step)` after its Adam launch, where the reference trainer
updates the same values.  One iteration of the reference (trainer.py:1213-1262), with global_step = s:

  1. Adam runs at the current rates;
  2. `scheduler_step(s)` sets every scheduled Gaussian group to sched(s) (a `skip` scheduler leaves its group where it is);
  3. the decoder's torch scheduler steps its own epoch counter: after iteration s its rate is the one of epoch s + 1, computed by torch's
     recursive form (this module restates `CosineAnnealingLR.get_lr` / `ExponentialLR.get_lr`, not their closed forms);
  4. the strategy's `post_optimizer_step` runs, so the MCMC perturbation scales its noise by sched(s);
  5. the SH degree goes up by `increase_step` (capped) when check_step_condition(s, 0, 1e6, increase_frequency) holds.

Index mapping: the schedule's step s is the reference's global_step, and the training step's `frame` at the start of that step (the number
of steps taken before it).  The step increments `frame` after its Adam launch, so its densifier is called with frame = s + 1; that
indexing is the densifier's own and is unchanged.  Every value is a host Python float or int: nothing here touches a device."""
from __future__ import annotations

import math

import numpy as np

from b200_native import cfg_get

SH_GROUPS = ("positions", "density", "rotation", "scale", "features_albedo", "features_specular")  # optimizers.GROUPS
NHT_GROUPS = ("positions", "density", "rotation", "scale", "features")                          # optimizers.NHT_GROUPS
# optimizer.params.*.lr of configs/base_gs.yaml (features_specular: features_albedo / 20) and model.nht_decoder.learning_rate
DEFAULT_LRS = {"positions": 0.00016, "density": 0.05, "rotation": 0.001, "scale": 0.005, "features_albedo": 0.0025, "features": 0.015}
DEFAULT_DECODER_LR = 0.00068
# model.progressive_training of configs/base_gs.yaml
DEFAULT_PROGRESSIVE = {"init_n_features": 0, "max_n_features": 3, "increase_frequency": 1000, "increase_step": 1}
GROUP_SCHEDULER_TYPES = ("exp", "cosine", "skip")        # utils/misc.py:110-114
DECODER_SCHEDULER_TYPES = ("exponential", "cosine")      # trainer.py:582-596


def check_step_condition(step: int, start: int, end: int, freq: int) -> bool:
    """utils/misc.py:212-216."""
    return bool((start >= 0 and step > start) and (step < end or end == -1) and step % freq == 0)


def exponential_lr(lr_init: float, lr_final: float, max_steps: int, step: int) -> float:
    """utils/misc.py:91-97: log-linear from lr_init to lr_final over max_steps, constant after."""
    t = np.clip(step / max_steps, 0, 1)
    return float(np.exp(np.log(lr_init) * (1 - t) + np.log(lr_final) * t))


def cosine_lr(lr_init: float, lr_final: float, max_steps: int, step: int) -> float:
    """utils/misc.py:100-107: cosine from lr_init to lr_final over max_steps, constant after."""
    t = np.clip(step / max_steps, 0, 1)
    return float(lr_final + 0.5 * (lr_init - lr_final) * (1 + np.cos(np.pi * t)))


class _GroupScheduler:
    """One Gaussian group's `scheduler.<name>` (exp or cosine; skip is never built)."""

    def __init__(self, kind: str, lr_init: float, lr_final: float, max_steps: int):
        self.fn = exponential_lr if kind == "exp" else cosine_lr
        self.lr_init, self.lr_final, self.max_steps = float(lr_init), float(lr_final), int(max_steps)

    def __call__(self, step: int) -> float:
        return self.fn(self.lr_init, self.lr_final, self.max_steps, step)


class DecoderScheduler:
    """torch.optim.lr_scheduler.CosineAnnealingLR(T_max=max_steps, eta_min=lr decay_final) or ExponentialLR(gamma=decay_final^(1/max_steps))
    on the decoder's rate, as trainer.py:579-596 builds them.  `step(lr, epoch)` is the rate torch's `get_lr` gives at `epoch` (>= 1) from
    the rate `lr` of epoch - 1: the recursive form, in torch's own operation order."""

    def __init__(self, kind: str, base_lr: float, decay_final: float, max_steps: int):
        self.kind, self.base_lr, self.max_steps = kind, float(base_lr), int(max_steps)
        self.eta_min = self.base_lr * float(decay_final)
        self.gamma = float(decay_final) ** (1.0 / self.max_steps)

    def step(self, lr: float, epoch: int) -> float:
        if self.kind == "exponential":
            return lr * self.gamma
        T, eta_min = self.max_steps, self.eta_min
        if (epoch - 1 - T) % (2 * T) == 0:
            return lr + (self.base_lr - eta_min) * (1 - math.cos(math.pi / T)) / 2
        return (1 + math.cos(math.pi * epoch / T)) / (1 + math.cos(math.pi * (epoch - 1) / T)) * (lr - eta_min) + eta_min


class TrainingSchedule:
    """The rates and the SH degree of each training step.  Build it with `from_config`; pass it to a training step as `schedule=`."""

    def __init__(self, lrs: dict, schedulers: dict, sph_degree: int, progression=None, decoder=None):
        """lrs: the rates of the first step, every group of the model (and "decoder" for NHT).  schedulers: group -> callable(step) -> rate.
        progression: None or (max degree, increase_frequency, increase_step).  decoder: None or a DecoderScheduler."""
        self.lrs = {k: float(v) for k, v in lrs.items()}
        self.schedulers = dict(schedulers)
        self.sph_degree = int(sph_degree)
        self.progression = progression
        self.decoder = decoder
        self.decoder_epoch = 0  # the decoder scheduler's last_epoch
        self.step = 0           # the next step index: one past the last one `advance` was given

    @classmethod
    def from_config(cls, conf, scene_extent: float = 1.0, feature_type: str | None = None) -> "TrainingSchedule":
        """The reference's schedule of `conf` (a dict or an attribute config).  feature_type: "sh" or "nht" (default model.feature_type).

        Reads optimizer.params.<group>.lr (positions x scene_extent, model.py:819-820), scheduler.<group> for the groups the model has
        (SH: positions, density, rotation, scale, features_albedo, features_specular; NHT: the same with features in place of the two SH
        groups), model.progressive_training (SH only: NHT renders every feature from the first step, model.py:247-250) and, for NHT,
        model.nht_decoder.learning_rate and model.nht_decoder.scheduler.  A missing optimizer rate or progressive_training key takes
        configs/base_gs.yaml's value.  A scheduler type the reference does not build raises KeyError (scheduler.<group>.type, as
        get_scheduler does) or ValueError (model.nht_decoder.scheduler.type, as trainer.py:595 does)."""
        feature_type = str(feature_type if feature_type is not None else cfg_get(conf, "model.feature_type", "sh")).lower()
        if feature_type not in ("sh", "nht"):
            raise ValueError(f"model.feature_type: unknown feature type {feature_type!r} (expected 'sh' or 'nht')")
        extent = float(scene_extent)
        groups = NHT_GROUPS if feature_type == "nht" else SH_GROUPS
        lrs = {}
        for name in groups:
            if name == "features_specular":
                default = lrs["features_albedo"] / 20  # ${div:${optimizer.params.features_albedo.lr},20}
            else:
                default = DEFAULT_LRS[name]
            lrs[name] = float(cfg_get(conf, f"optimizer.params.{name}.lr", default))
        lrs["positions"] *= extent

        schedulers = {}
        for name in groups:  # setup_scheduler (model.py:832-852): only the model's own parameters are scheduled
            args = cfg_get(conf, f"scheduler.{name}", None)
            kind = cfg_get(args, "type", None)
            if kind is None:
                continue
            if kind not in GROUP_SCHEDULER_TYPES:
                raise KeyError(f"scheduler.{name}.type: unknown scheduler {kind!r} (expected one of {', '.join(GROUP_SCHEDULER_TYPES)})")
            if kind == "skip":
                continue
            max_steps = int(cfg_get(args, "max_steps", 1000000))
            if name == "positions":
                lr_init = float(cfg_get(args, "lr_init", cfg_get(conf, "optimizer.params.positions.lr", DEFAULT_LRS["positions"]))) * extent
                lr_final = float(cfg_get(args, "lr_final", 0.0000016)) * extent
            elif name == "features":
                lr_init = lrs["features"]
                lr_final = lr_init * float(cfg_get(args, "decay_final", 0.001))
            else:
                lr_init, lr_final = float(cfg_get(args, "lr_init", lrs[name])), float(cfg_get(args, "lr_final", lrs[name]))
            schedulers[name] = _GroupScheduler(kind, lr_init, lr_final, max_steps)

        p = {k: cfg_get(conf, f"model.progressive_training.{k}", v) for k, v in DEFAULT_PROGRESSIVE.items()}
        max_degree = min(int(p["max_n_features"]), int(cfg_get(conf, "render.particle_radiance_sph_degree", 3)))  # model.py:174-180
        decoder = None
        if feature_type == "nht":
            degree, progression = max_degree, None
            lrs["decoder"] = float(cfg_get(conf, "model.nht_decoder.learning_rate", DEFAULT_DECODER_LR))
            dec = cfg_get(conf, "model.nht_decoder.scheduler", None)
            kind = cfg_get(dec, "type", None)
            if kind not in DECODER_SCHEDULER_TYPES:
                raise ValueError(f"model.nht_decoder.scheduler.type: unknown scheduler type {kind!r} "
                                 f"(expected one of {', '.join(DECODER_SCHEDULER_TYPES)})")
            max_steps = int(cfg_get(dec, "max_steps", cfg_get(conf, "n_iterations", 30000)))
            decoder = DecoderScheduler(kind, lrs["decoder"], float(cfg_get(dec, "decay_final", 0.001)), max_steps)
        else:
            degree = min(int(p["init_n_features"]), max_degree)
            progression = (max_degree, int(p["increase_frequency"]), int(p["increase_step"])) if degree < max_degree else None
        return cls(lrs, schedulers, degree, progression, decoder)

    def initial_lrs(self) -> dict:
        """The rates of the next step, in the dict shape the step's optimizer takes: the config's initial rates on a new schedule."""
        return dict(self.lrs)

    def initial_sph_degree(self) -> int:
        """The SH degree of the next step: init_n_features (clamped) on a new SH schedule; constant for NHT."""
        return self.sph_degree

    def advance(self, step: int) -> tuple[dict, int]:
        """The post-optimizer update of the reference's iteration global_step = step: returns (the rates of the next step, its SH degree)."""
        step = int(step)
        for name, sched in self.schedulers.items():
            self.lrs[name] = sched(step)
        if self.decoder is not None:
            self.decoder_epoch += 1
            self.lrs["decoder"] = self.decoder.step(self.lrs["decoder"], self.decoder_epoch)
        if self.progression is not None:
            max_degree, frequency, increment = self.progression
            if check_step_condition(step, 0, 1e6, frequency):
                self.sph_degree = min(max_degree, self.sph_degree + increment)
        self.step = step + 1
        return dict(self.lrs), self.sph_degree

    def advance_to(self, step: int) -> "TrainingSchedule":
        """Advance step by step up to (not including) `step`: a schedule fresh from `from_config` then holds what it holds after the
        reference's iteration step - 1, bit for bit (a checkpoint with no schedule state resumes so).  Returns self."""
        step = int(step)
        if step < self.step:
            raise ValueError(f"schedule: cannot go back from step {self.step} to step {step}")
        for s in range(self.step, step):
            self.advance(s)
        return self

    def state_dict(self) -> dict:
        """What a resumed run needs to continue bit for bit: the step index, the SH degree, the decoder's epoch and the current rates."""
        return {"step": self.step, "sph_degree": self.sph_degree, "decoder_epoch": self.decoder_epoch, "lrs": dict(self.lrs)}

    def load_state_dict(self, state: dict):
        if set(state["lrs"]) != set(self.lrs):
            raise ValueError(f"schedule state: groups {sorted(state['lrs'])} do not match this schedule's {sorted(self.lrs)}")
        self.step, self.sph_degree, self.decoder_epoch = int(state["step"]), int(state["sph_degree"]), int(state["decoder_epoch"])
        self.lrs = {k: float(v) for k, v in state["lrs"].items()}

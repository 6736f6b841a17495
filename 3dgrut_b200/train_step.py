"""Thin view-parallel training step for the SH Gaussian model on the 3DGUT path (SURVEY.md section 8f row 1, without densification).

Replaces the render + backward + optimizer part of Trainer.run_train_iter (threedgrut/trainer.py:1119-1263) with the pieces of this
repository wired together -- no autograd graph, no per-parameter all-reduce, no separate activation backward:

    activations (sigmoid / exp / normalize, model.py:102-118)  ->  SplatRaster.trace
    -> loss gradient on the image (L1, trainer.py:698-704 + losses.py:20-21; or L1 + SSIM, with the background composited, the
       linear-to-sRGB post-processing and the mask applied, by losses.image_loss)  ->  SplatRaster.trace_bwd_compact
    -> CompactGradientExchange (all-reduce [N,12], all-gather [N,4], rebuild [N,48])  ->  FusedGaussianAdam.step (+ the opacity and
       scale regularisers, once per step after the exchange)

Every rank holds a replica of the parameters and renders its own camera of the step's batch; the loss is normalised by the global
batch (number of ranks), so the replicas stay identical.  The trainer, datasets, densification and logging of the reference stay out
of scope; this class exists so that the path can be run -- and tested -- as the training loop uses it.

`TrainStep` holds what every training step shares: the parameters, the optimizer, the background, the densifier, the order of a step,
the loss dispatch and everything after the backward.  A renderer's step supplies its forward (a `Frame`) and its backward."""
from __future__ import annotations

from typing import NamedTuple

import numpy as np
import torch
import torch.distributed as dist

import checkpoint
import losses
import optimizers
import view_parallel
from threedgut_tracer.tracer import SplatRaster


class Frame(NamedTuple):
    """What a step reads after its renderer's forward."""
    pred: torch.Tensor    # the render the loss takes, before background and post-processing
    layout: int           # 4: pred is the 3DGUT rgba [H,W,4]; 3: pred is rgb [H,W,3] and `alpha` is separate
    rgb: torch.Tensor     # the colour channels [H,W,3]
    alpha: torch.Tensor | None  # [H,W,1] (any strides), or None where it is channel 3 of pred
    hits: torch.Tensor    # [H,W,1]
    vis: torch.Tensor     # the visibility the optimizer's selective update reads
    saved: tuple          # the renderer's own: what its `_backward` reads


class TrainStep:
    """The part of a view-parallel training step that does not depend on the renderer.  A subclass creates its renderer
    (`_init_renderer`) and its exchange (`_new_exchange`), renders a view into a `Frame` (`_forward`), writes the view's gradients into
    `exchange.out()` (`_backward`) and gives this view's sensor position (`_sensor_position`); its public `step`, `render` and
    `metrics_inputs` take the view's arguments and `_step` runs: activations -> `_forward` -> `_loss` -> `_backward` -> `_update`."""

    PHASES = ("exchange", "adam", "densify")  # the phases `phase_events` records; a subclass lists its own

    def __init__(self, params: dict, lrs: dict | None, conf=None, sph_degree: int | None = None, selective: bool = False, group=None,
                 eps: float = 1e-15, densify_conf=None, scene_extent: float = 1.0, lambda_l1: float = 1.0, lambda_ssim: float = 0.0,
                 background="black", background_seed: int = 0, lambda_opacity: float = 0.0, lambda_scale: float = 0.0, post_processing=None,
                 schedule=None):
        """params: raw leaf tensors for optimizers.GROUPS (positions, density, rotation, scale, features_albedo, features_specular).
        conf: a config with a `render:` section, read as the step's renderer reads it.
        densify_conf: a densify.DensifyConfig (GS strategy: clone / split / prune / reset) or densify.MCMCConfig (relocate / add / perturb)
        turns on the replica-consistent strategy.  background: "black", "white", "random" or (r, g, b), composited onto the render before
        the loss (model.background.color); "random" draws from a generator seeded background_seed + rank.  lambda_opacity / lambda_scale:
        the regularisers of the loss (loss.lambda_opacity / loss.lambda_scale when use_opacity / use_scale).  post_processing: None or
        "linear-to-srgb" (post_processing.method): the composited render is encoded to sRGB before the mask and the loss, for sRGB targets
        and linear radiance; "ppisp" raises NotImplementedError.  It has no parameters and adds 0 to the loss.  sph_degree: the SH degree
        rendered (default 3).  schedule: None (constant `lrs` and `sph_degree`) or a schedule.TrainingSchedule, which sets the initial rates
        (in place of `lrs`) and degree (refused together with an explicit sph_degree) and updates both after every Adam launch, as the
        reference trainer's schedulers and progressive SH do."""
        losses.post_processing_code(post_processing)  # refuse what is not built before anything is allocated
        self._buffers = {}  # name -> (resolution, buffers): see _scratch
        self.post_processing = post_processing
        self.params = {k: params[k] for k in self.GROUPS}  # ONE dict shared with the optimizer and the densifier
        self.device = self.params["positions"].device
        self.schedule = schedule
        if schedule is not None:
            if sph_degree is not None:
                raise ValueError("sph_degree and schedule: the schedule sets the SH degree (model.progressive_training); pass one of them")
            lrs, sph_degree = schedule.initial_lrs(), schedule.initial_sph_degree()
            missing = set(self.GROUPS) - set(lrs)
            if missing:
                raise ValueError(f"schedule: no learning rate for {sorted(missing)}; build it with the feature type this step trains")
        elif lrs is None:
            raise ValueError("lrs: the learning rates are required without a schedule")
        self.sph_degree = 3 if sph_degree is None else int(sph_degree)
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        self._init_renderer(conf if conf is not None else {"render": {}})
        self.optimizer = self._new_optimizer(lrs, eps, selective)
        self.exchange = self._new_exchange()
        self.frame = 0
        self.lambda_l1, self.lambda_ssim = float(lambda_l1), float(lambda_ssim)  # reference defaults: 0.8 / 0.2 (configs/base_gs.yaml:172-179)
        self.lambda_opacity, self.lambda_scale = float(lambda_opacity), float(lambda_scale)
        rank = dist.get_rank(group) if self.world > 1 else 0
        self.background = losses.Background(background, seed=int(background_seed) + rank, device=self.device)
        self.scene_extent = float(scene_extent)
        self.densifier = None
        if densify_conf is not None:
            import densify

            cls = densify.MCMCDensifier if isinstance(densify_conf, densify.MCMCConfig) else densify.GSDensifier
            self.densifier = cls(self.params, [self.optimizer.exp_avg, self.optimizer.exp_avg_sq], densify_conf, group=group)
        self.phase_events = None  # set to [] to record (phase, cuda event) pairs at the end of the phases of `step` that mark one

    GROUPS = optimizers.GROUPS  # the raw parameter tensors the step trains

    def bytes_on_wire(self) -> int:
        return self.exchange.bytes_on_wire()

    def _new_optimizer(self, lrs, eps, selective):
        return optimizers.FusedGaussianAdam(self.params, lrs, eps=eps, selective=selective)

    @property
    def n(self) -> int:
        return int(self.params["positions"].shape[0])

    @torch.no_grad()
    def activated(self):
        """[N,12] = pos3, sigmoid(density), normalize(rotation) (wxyz), exp(scale), 0 and [N,48] = cat(albedo, specular)
        (threedgut_tracer/tracer.py:176-178, threedgrt_tracer/tracer.py:61, model.py:94-118)"""
        p = self.params
        return particle_record(p), torch.cat([p["features_albedo"], p["features_specular"]], dim=1).contiguous()

    def _mark(self, phase):
        if self.phase_events is not None and phase in self.PHASES:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.phase_events.append((phase, ev))

    def _scratch(self, name, key, make):
        """The buffers `name` of resolution `key`: make() on the first step at it, and again (dropping the old ones) when it changes."""
        held = self._buffers.get(name)
        if held is None or held[0] != key:
            held = self._buffers[name] = (key, make())
        return held[1]

    def _zeros(self, H, W, channels):
        """A zero [1,H,W,channels] gradient for the renderer inputs the loss does not differentiate; never written."""
        return self._scratch(("zeros", channels), (H, W), lambda: torch.zeros((1, H, W, channels), dtype=torch.float32, device=self.device))

    def _step(self, view, target_rgb, all_sensor_positions, mask):
        """The body of every `step`.  view: the arguments of the subclass's `render`, rays_o [1,H,W,3] first."""
        H, W = int(view[0].shape[1]), int(view[0].shape[2])
        if mask is not None:
            mask = losses.mask_hw(mask, H, W)
        particles, features = self.activated()
        frame = self._forward(view, particles, features, train=True)
        loss, d_pred, d_alpha = self._loss(frame, target_rgb.reshape(H, W, 3), H, W, mask)
        self._mark("loss")
        exchange_args = self._backward(frame, d_pred, d_alpha)
        my_position = self._sensor_position(frame) if self.densifier is not None or exchange_args else None
        if exchange_args:  # the compact exchange rebuilds the SH gradient from the sensor position of every view of the step
            positions = my_position[None] if all_sensor_positions is None else all_sensor_positions
            exchange_args = (*exchange_args, np.asarray(positions, np.float32))
        return self._update(loss, particles, frame.vis, all_sensor_positions, my_position, exchange_args)

    @torch.no_grad()
    def metrics_inputs(self, *view):
        """Forward only, what the test-set metrics read (metrics.image_metrics); arguments as `render`'s.  {"pred": the render before
        background and post-processing in the loss's layout (rgba [H,W,4], or rgb [H,W,3] for the split layout), "alpha": [H,W,1], or None
        where it is channel 3 of pred, "hits": [H,W,1]}.  No BVH cadence is advanced; the NHT steps decode with the current weights."""
        f = self._forward(view, *self.activated(), train=False)
        return {"pred": f.pred, "alpha": None if f.alpha is None else f.alpha.contiguous(), "hits": f.hits}

    def _loss(self, frame, target, H, W, mask):
        """This view's loss and its gradients (d_pred in frame.pred's layout, d_alpha [H,W,1] or None where the loss gives the separate
        alpha none).  target: [H,W,3].  The gradients carry the global-batch normalisation (1 / world); the loss returned does not."""
        if self.background.black and mask is None and self.lambda_ssim == 0.0 and self.post_processing is None:
            diff = frame.rgb - target
            loss = self.lambda_l1 * diff.abs().mean()
            if frame.layout == 3:
                return loss, self._d_l1(diff), None
            d_rgba = torch.zeros_like(frame.pred)
            d_rgba[..., :3] = self._d_l1(diff)
            return loss, d_rgba, None
        # composited onto the background, post-processed and masked (then with an alpha gradient), or lambda_l1 L1 + lambda_ssim
        # (1 - SSIM): two launches (gut_loss.cu).  The L1 shortcut above does not apply in encoded space.
        target, l1, ssim = target.contiguous(), self.lambda_l1 / self.world, self.lambda_ssim / self.world
        background, post = self.background.draw(H, W), self.post_processing
        d_alpha = None
        if frame.layout == 4:  # d_rgba carries the alpha gradient when composited
            loss, _, _, d_pred = losses.image_loss(frame.pred, target, l1, ssim, background=background, mask=mask, post_processing=post)
        elif background is None and mask is None and post is None:  # black, unmasked: the rgb loss, no alpha gradient
            loss, _, _, d_pred = losses.image_loss_rgb(frame.pred, target, l1, ssim)
        else:
            loss, _, _, d_pred, d_alpha = losses.image_loss_rgb_alpha(frame.pred, frame.alpha.contiguous(), target, l1, ssim,
                                                                      background=background, mask=mask, post_processing=post)
        return loss * self.world, d_pred, d_alpha

    def _d_l1(self, diff):
        """d lambda_l1 mean|diff| / d rgb with the global-batch normalisation"""
        return self.lambda_l1 * torch.sign(diff) / (diff.numel() * self.world)

    def _update(self, loss, particles, vis, all_sensor_positions, my_position, exchange_args=()):
        """After the backward has written this view's gradients into `exchange.out()`: feed the densifier, exchange, OR-reduce the
        visibility, add the regularisers, step Adam, densify.  my_position: this view's sensor position (only the densifier reads it)."""
        if all_sensor_positions is None and self.world != 1:
            raise RuntimeError("all_sensor_positions is required when more than one rank trains")
        if self.densifier is not None:
            # this view's own position gradient, before the exchange (it is weighted by the distance to THIS view's sensor, gs.py:127-137);
            # x world undoes the global-batch normalisation so that the thresholds keep their per-view meaning
            self.densifier.update_gradient_buffer(self.exchange.d_particles[:, 0:3] * float(self.world), my_position)
        d_particles, d_sph = self.exchange.exchange(*exchange_args)
        if self.optimizer.selective and self.world > 1:
            dist.all_reduce(vis, op=dist.ReduceOp.MAX, group=self.group)  # visible in any view of the batch (SURVEY 8e)
        self._mark("exchange")
        # the regularisers belong to the step once (every rank holds the same parameters): added after the exchange, no 1 / world
        frozen = self._geometry_frozen()
        reg = {}
        if (self.lambda_opacity != 0.0 or self.lambda_scale != 0.0) and not frozen:
            loss = loss + regulariser_loss(particles, self.lambda_opacity, self.lambda_scale)
            reg = dict(lambda_opacity=self.lambda_opacity, lambda_scale=self.lambda_scale)
        self._adam(d_particles, d_sph, vis if self.optimizer.selective else None, reg)
        self._mark("adam")
        if self.schedule is not None:
            # the reference's scheduler_step(global_step = frame) and progressive SH, after Adam and before the strategy (schedule.py);
            # host scalars the next step's launches take: no launch, no copy
            lrs, self.sph_degree = self.schedule.advance(self.frame)
            self.optimizer.lrs.update(lrs)
        self.frame += 1
        if self.densifier is not None and not frozen and self.densifier.post_optimizer_step(self.frame, self.scene_extent, positions_lr=self.optimizer.lrs["positions"]):
            self._densified()
        self._mark("densify")
        return loss

    def _post_process(self, rgb):
        """render()'s rgb as the loss sees it over a black background: linear_to_srgb(rgb) under post_processing, else rgb itself."""
        return rgb if self.post_processing is None else losses.linear_to_srgb(rgb)

    def _adam(self, d_particles, d_sph, vis, reg):
        self.optimizer.step(d_particles, d_sph, visibility=vis, **reg)

    def _geometry_frozen(self) -> bool:
        """True while positions, density, rotation and scale are frozen (the NHT steps' colour refinement): the step then adds no
        regulariser and does not densify."""
        return False

    def _densified(self):
        """The number of Gaussians may have changed (identically on every rank): re-capacity the exchange buffers; the renderer's scratch
        grows by itself."""
        if self.exchange.n != self.n:
            self.exchange = self._new_exchange()

    # ---- checkpoints (checkpoint.py writes and reads these states in the reference's ckpt_*.pt layout)

    FEATURE_TYPE = "sh"  # model.feature_type of the parameters the step trains
    WIDTHS = optimizers.WIDTHS

    def _settings(self) -> dict:
        """The constructor arguments that are settings rather than state, as plain data.  A state records them, and load_state_dict
        refuses a state trained with other values."""
        bg, opt = self.background, self.optimizer
        return {"selective": bool(opt.selective), "eps": float(opt.eps), "lambda_l1": self.lambda_l1, "lambda_ssim": self.lambda_ssim,
                "lambda_opacity": self.lambda_opacity, "lambda_scale": self.lambda_scale,
                "background": "random" if bg.random else [float(c) for c in bg.color], "post_processing": self.post_processing,
                "strategy": None if self.densifier is None else self.densifier.METHOD}

    def _adam_steps(self) -> dict:
        return {k: int(self.optimizer.steps) for k in self.GROUPS}

    def _load_adam_steps(self, steps: dict):
        self.optimizer.steps = int(steps[self.GROUPS[0]])

    def state_dict(self) -> dict:
        """Everything a later `step` reads: the raw parameters, both Adam moments and the step count, frame, SH degree, scene extent and
        rates, the densifier's buffers and generator, this rank's background generator and the schedule's state, with the settings the
        step was built with.  The tensors are the step's own, not copies (as nn.Module.state_dict's); checkpoint.save writes them."""
        opt, sched = self.optimizer, self.schedule
        return {"feature_type": self.FEATURE_TYPE, "settings": self._settings(), "frame": int(self.frame), "sph_degree": int(self.sph_degree),
                "scene_extent": float(self.scene_extent), "lrs": dict(opt.lrs),
                "progression": None if sched is None or sched.progression is None else [int(v) for v in sched.progression],
                "params": dict(self.params), "exp_avg": {k: opt.exp_avg[k] for k in self.GROUPS},
                "exp_avg_sq": {k: opt.exp_avg_sq[k] for k in self.GROUPS}, "adam_steps": self._adam_steps(),
                "densifier": None if self.densifier is None else self.densifier.state_dict(),
                "background_generator": None if self.background.generator is None else self.background.generator.get_state(),
                "schedule": None if sched is None else sched.state_dict()}

    def _check_state(self, state: dict):
        """Refuse (ValueError naming the key) a state this step cannot continue, before anything is changed."""
        if state.get("feature_type", "sh") != self.FEATURE_TYPE:
            raise ValueError(f"feature_type: the state holds {state.get('feature_type')!r} parameters, this step trains {self.FEATURE_TYPE!r}")
        mine = self._settings()
        for key, theirs in (state.get("settings") or {}).items():
            if key in mine and _plain(theirs) != _plain(mine[key]):
                raise ValueError(f"{key}: the state was trained with {theirs!r}, this step is built with {mine[key]!r} (a constructor "
                                 f"setting, not state: build the step as the run was built)")
        n = int(state["params"]["positions"].shape[0])
        for k, w in zip(self.GROUPS, self.WIDTHS):
            for what in ("params", "exp_avg", "exp_avg_sq"):
                if tuple(state[what][k].shape) != (n, w):
                    raise ValueError(f"{what}.{k}: expected shape {(n, w)}, got {tuple(state[what][k].shape)}")
        checkpoint.check_step_counts(self.FEATURE_TYPE, state["adam_steps"])
        missing = set(self.optimizer.lrs) - set(state["lrs"])
        if missing:
            raise ValueError(f"lrs: the state has no rate for {sorted(missing)}")
        if self.schedule is not None and state.get("schedule") is None and self.schedule.step > int(state["frame"]):
            raise ValueError(f"schedule: the state has no schedule and this step's is past its frame {int(state['frame'])}")

    def _load_extra(self, state: dict, take):
        """What a subclass holds beyond TrainStep's state; called after the parameters are in place."""

    @torch.no_grad()
    def load_state_dict(self, state: dict, assign: bool = False):
        """Continue from `state` (state_dict()'s, or checkpoint.from_reference_layout's), which may hold a different N: the tensors inside
        the shared parameter and moment dicts are replaced, as densification replaces them, and the exchange is re-capacitied.
        assign=False copies the state's tensors; assign=True takes them as the step's own where they already are float32 on the step's
        device (as nn.Module.load_state_dict(assign=True)), so a state read onto the device is not copied again.  A state without generator
        states re-seeds them as the constructor does; without a schedule state, the step's schedule (fresh from from_config) is replayed to
        the state's frame."""
        self._check_state(state)

        def take(t):
            out = t.detach().to(device=self.device, dtype=torch.float32)
            if not assign and out.data_ptr() == t.data_ptr():
                out = out.clone()
            return out.contiguous()

        opt = self.optimizer
        for k in self.GROUPS:  # the same dict objects: the optimizer and the densifier see the new tensors
            self.params[k], opt.exp_avg[k], opt.exp_avg_sq[k] = take(state["params"][k]), take(state["exp_avg"][k]), take(state["exp_avg_sq"][k])
        self._load_adam_steps(state["adam_steps"])
        opt.lrs.update({k: float(state["lrs"][k]) for k in opt.lrs})
        self.frame, self.scene_extent = int(state["frame"]), float(state["scene_extent"])
        if self.densifier is not None:
            self.densifier.load_state_dict(state.get("densifier"))
        if self.background.generator is not None:
            import densify

            densify.load_generator(self.background.generator, state.get("background_generator"), self.background.seed)
        if self.schedule is not None:
            if state.get("schedule") is not None:
                self.schedule.load_state_dict(state["schedule"])
            else:
                self.schedule.advance_to(self.frame)
        if state.get("sph_degree") is not None:
            self.sph_degree = int(state["sph_degree"])
        elif self.schedule is not None:
            self.sph_degree = self.schedule.sph_degree
        self._load_extra(state, take)
        self._densified()


def _plain(v):
    """Settings as compared: tuples as lists."""
    if isinstance(v, (list, tuple)):
        return [_plain(x) for x in v]
    if isinstance(v, dict):
        return {k: _plain(x) for k, x in v.items()}
    return v


class GaussianTrainStep(TrainStep):
    def _init_renderer(self, conf):
        self.raster = SplatRaster(conf)

    def _new_exchange(self):
        return view_parallel.CompactGradientExchange(self.raster, self.n, self.device, group=self.group)

    def _forward(self, view, particles, sph, train):
        rays_o, rays_d, sensor, pose = view
        rgba, dst, hits, vis = self.raster.trace(self.frame, self.sph_degree, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose)
        return Frame(rgba, 4, rgba[..., :3], None, hits, vis, (view, particles, sph, dst))

    def _backward(self, frame, d_rgba, d_alpha):
        (rays_o, rays_d, sensor, pose), particles, sph, dst = frame.saved
        d_dist = torch.zeros_like(dst)
        self.raster.trace_bwd_compact(self.frame, self.sph_degree, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose, frame.pred,
                                      d_rgba, dst, d_dist, out=self.exchange.out())
        return self.sph_degree, particles

    def _sensor_position(self, frame):
        _, _, sensor, pose = frame.saved[0]
        return self.raster.sensor_position(sensor, pose, pose, frame.rgb.shape[1], frame.rgb.shape[0])

    @torch.no_grad()
    def render(self, rays_o, rays_d, sensor, pose):
        """Forward only: (rgba [H,W,4], dist, hits, visibility); under post_processing the rgb channels are encoded, alpha is not."""
        f = self._forward((rays_o, rays_d, sensor, pose), *self.activated(), train=False)
        rgba = f.pred if self.post_processing is None else torch.cat([self._post_process(f.rgb), f.pred[..., 3:]], -1)
        return rgba, f.saved[3], f.hits, f.vis

    @torch.no_grad()
    def step(self, rays_o, rays_d, sensor, pose, target_rgb, all_sensor_positions=None, mask=None):
        """One optimisation step on this rank's view.  target_rgb: [H,W,3].  all_sensor_positions: [world,3] sensor positions of every
        rank's view of this step in rank order (omit on a single GPU).  mask: optional [H,W] ([H,W,1], [1,H,W,1]) float CUDA tensor that
        multiplies prediction and target before the loss.  Returns this view's loss (a device scalar), the regularisers included."""
        return self._step((rays_o, rays_d, sensor, pose), target_rgb, all_sensor_positions, mask)


def particle_record(p: dict) -> torch.Tensor:
    """The activated [N,12] record of the raw parameter dict p: pos3, sigmoid(density), normalize(rotation) (wxyz), exp(scale), 0."""
    return torch.cat([p["positions"], torch.sigmoid(p["density"]), torch.nn.functional.normalize(p["rotation"]), torch.exp(p["scale"]),
                      torch.zeros_like(p["density"])], dim=1).contiguous()


def raw_params(particles: torch.Tensor, sph: torch.Tensor | None = None, features: torch.Tensor | None = None) -> dict:
    """The raw parameter dict of the activated [N,12] record: the inverse of particle_record, with the density clamped to
    [1e-4, 1 - 1e-4] before its logit.  Exactly one of sph ([N,48] SH: features_albedo, features_specular) and features ([N,F] NHT)."""
    if (sph is None) == (features is None):
        raise ValueError("raw_params takes exactly one of sph and features")
    d = particles[:, 3:4].clamp(1e-4, 1 - 1e-4)
    raw = {"positions": particles[:, 0:3].clone(), "density": torch.log(d / (1 - d)), "rotation": particles[:, 4:8].clone(),
           "scale": torch.log(particles[:, 8:11])}
    if sph is not None:
        raw.update(features_albedo=sph[:, 0:3].clone(), features_specular=sph[:, 3:48].clone())
    else:
        raw["features"] = features.clone()
    return raw


def regulariser_loss(particles, lambda_opacity: float, lambda_scale: float):
    """lambda_opacity mean|density| + lambda_scale mean|scale| on the activated [N,12] record (trainer.py:722-736); 0 when both are 0."""
    reg = 0.0
    if lambda_opacity != 0.0:
        reg = reg + lambda_opacity * particles[:, 3].abs().mean()
    if lambda_scale != 0.0:
        reg = reg + lambda_scale * particles[:, 8:11].abs().mean()
    return reg

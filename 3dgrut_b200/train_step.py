"""Thin view-parallel training step for the SH Gaussian model on the 3DGUT path (SURVEY.md section 8f row 1, without densification).

Replaces the render + backward + optimizer part of Trainer.run_train_iter (threedgrut/trainer.py:1119-1263) with the pieces of this
repository wired together -- no autograd graph, no per-parameter all-reduce, no separate activation backward:

    activations (sigmoid / exp / normalize, model.py:102-118)  ->  SplatRaster.trace
    -> loss gradient on the image (L1, trainer.py:698-704 + losses.py:20-21; or L1 + SSIM, with the background composited and the mask
       applied, by losses.image_loss)  ->  SplatRaster.trace_bwd_compact
    -> CompactGradientExchange (all-reduce [N,12], all-gather [N,4], rebuild [N,48])  ->  FusedGaussianAdam.step (+ the opacity and
       scale regularisers, once per step after the exchange)

Every rank holds a replica of the parameters and renders its own camera of the step's batch; the loss is normalised by the global
batch (number of ranks), so the replicas stay identical.  The trainer, datasets, densification and logging of the reference stay out
of scope; this class exists so that the path can be run -- and tested -- as the training loop uses it.

`TrainStep` holds what this step and the 3DGRT one (train_step_grt.GaussianTrainStepGRT) share: the parameters, the optimizer, the
background, the densifier, the loss dispatch and everything after the backward."""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist

import losses
import optimizers
import view_parallel
from threedgut_tracer.tracer import SplatRaster


class TrainStep:
    """The part of a view-parallel training step that does not depend on the renderer.  A subclass creates its renderer
    (`_init_renderer`) and its exchange (`_new_exchange`), gives the loss gradient its renderer's layout (`_image_loss`, `_l1_grads`),
    and writes `step` as: activations -> trace -> `_loss` -> backward into `exchange.out()` -> `_update`."""

    def __init__(self, params: dict, lrs: dict, conf=None, sph_degree: int = 3, selective: bool = False, group=None, eps: float = 1e-15,
                 densify_conf=None, scene_extent: float = 1.0, lambda_l1: float = 1.0, lambda_ssim: float = 0.0, background="black",
                 background_seed: int = 0, lambda_opacity: float = 0.0, lambda_scale: float = 0.0):
        """params: raw leaf tensors for optimizers.GROUPS (positions, density, rotation, scale, features_albedo, features_specular).
        conf: a config with a `render:` section, read as the step's renderer reads it.
        densify_conf: a densify.DensifyConfig (GS strategy: clone / split / prune / reset) or densify.MCMCConfig (relocate / add / perturb)
        turns on the replica-consistent strategy.  background: "black", "white", "random" or (r, g, b), composited onto the render before
        the loss (model.background.color); "random" draws from a generator seeded background_seed + rank.  lambda_opacity / lambda_scale:
        the regularisers of the loss (loss.lambda_opacity / loss.lambda_scale when use_opacity / use_scale)."""
        self.params = {k: params[k] for k in self.GROUPS}  # ONE dict shared with the optimizer and the densifier
        self.device = self.params["positions"].device
        self.sph_degree = int(sph_degree)
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
        if self.phase_events is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.phase_events.append((phase, ev))

    def _loss(self, pred, rgb, target, H, W, mask):
        """This view's loss and its gradient in the renderer's layout.  pred: the render as `_image_loss` / `_l1_grads` take it; rgb: its
        colour channels [H,W,3]; target: [H,W,3].  The gradient carries the global-batch normalisation (1 / world); the loss returned
        does not."""
        if not self.background.black or mask is not None or self.lambda_ssim != 0.0:
            # composited onto the background and masked (then with an alpha gradient), or lambda_l1 L1 + lambda_ssim (1 - SSIM): two
            # launches (gut_loss.cu)
            loss, grads = self._image_loss(pred, target.contiguous(), self.lambda_l1 / self.world, self.lambda_ssim / self.world,
                                           self.background.draw(H, W), mask)
            return loss * self.world, grads
        diff = rgb - target
        return self.lambda_l1 * diff.abs().mean(), self._l1_grads(pred, diff)

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
        self.frame += 1
        if self.densifier is not None and not frozen and self.densifier.post_optimizer_step(self.frame, self.scene_extent, positions_lr=self.optimizer.lrs["positions"]):
            self._densified()
        self._mark("densify")
        return loss

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


class GaussianTrainStep(TrainStep):
    def _init_renderer(self, conf):
        self.raster = SplatRaster(conf)

    def _new_exchange(self):
        return view_parallel.CompactGradientExchange(self.raster, self.n, self.device, group=self.group)

    def _image_loss(self, rgba, target, lambda_l1, lambda_ssim, background, mask):
        loss, _, _, d_rgba = losses.image_loss(rgba, target, lambda_l1, lambda_ssim, background=background, mask=mask)
        return loss, d_rgba  # d_rgba carries the alpha gradient when composited (gut_loss.cu)

    def _l1_grads(self, rgba, diff):
        d_rgba = torch.zeros_like(rgba)
        d_rgba[..., :3] = self._d_l1(diff)
        return d_rgba

    @torch.no_grad()
    def render(self, rays_o, rays_d, sensor, pose):
        particles, sph = self.activated()
        rgba, dist_, hits, vis = self.raster.trace(self.frame, self.sph_degree, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose)
        return rgba, dist_, hits, vis

    @torch.no_grad()
    def step(self, rays_o, rays_d, sensor, pose, target_rgb, all_sensor_positions=None, mask=None):
        """One optimisation step on this rank's view.  target_rgb: [H,W,3].  all_sensor_positions: [world,3] sensor positions of every
        rank's view of this step in rank order (omit on a single GPU).  mask: optional [H,W] ([H,W,1], [1,H,W,1]) float CUDA tensor that
        multiplies prediction and target before the loss.  Returns this view's loss (a device scalar), the regularisers included."""
        H, W = int(rays_o.shape[1]), int(rays_o.shape[2])
        if mask is not None:
            mask = losses.mask_hw(mask, H, W)
        particles, sph = self.activated()
        rgba, dst, hits, vis = self.raster.trace(self.frame, self.sph_degree, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose)
        loss, d_rgba = self._loss(rgba, rgba[..., :3], target_rgb, H, W, mask)
        d_dist = torch.zeros_like(dst)
        self.raster.trace_bwd_compact(self.frame, self.sph_degree, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose, rgba, d_rgba,
                                      dst, d_dist, out=self.exchange.out())
        my_position = self.raster.sensor_position(sensor, pose, pose, W, H)
        positions = my_position[None] if all_sensor_positions is None else all_sensor_positions
        return self._update(loss, particles, vis, all_sensor_positions, my_position,
                            (self.sph_degree, particles, np.asarray(positions, np.float32)))


def particle_record(p: dict) -> torch.Tensor:
    """The activated [N,12] record of the raw parameter dict p: pos3, sigmoid(density), normalize(rotation) (wxyz), exp(scale), 0."""
    return torch.cat([p["positions"], torch.sigmoid(p["density"]), torch.nn.functional.normalize(p["rotation"]), torch.exp(p["scale"]),
                      torch.zeros_like(p["density"])], dim=1).contiguous()


def regulariser_loss(particles, lambda_opacity: float, lambda_scale: float):
    """lambda_opacity mean|density| + lambda_scale mean|scale| on the activated [N,12] record (trainer.py:722-736); 0 when both are 0."""
    reg = 0.0
    if lambda_opacity != 0.0:
        reg = reg + lambda_opacity * particles[:, 3].abs().mean()
    if lambda_scale != 0.0:
        reg = reg + lambda_scale * particles[:, 8:11].abs().mean()
    return reg

"""View-parallel training step for the SH Gaussian model on the 3DGRT path: the ray-traced twin of train_step.GaussianTrainStep.

Replaces Tracer.render + loss + autograd + per-parameter Adam of the reference trainer (threedgrut/trainer.py:1119-1263 with the 3DGRT
renderer) by the pieces of this repository wired together, with no autograd graph:

    activations (model.py:102-118)  ->  LBVH build from the [N,12] record (cadence of Tracer.build_acc, threedgrt_tracer/tracer.py:198-216)
    -> OptixTracer.trace (hit lists recorded)  ->  image loss gradient (L1, or L1 + SSIM with losses.image_loss_rgb; with a background
       or a mask, losses.image_loss_rgb_alpha, which also gives the alpha gradient)
    -> OptixTracer.trace_bwd (hit-list replay) into the exchange buffer  ->  FlatGradientExchange (one all-reduce of 240 B x N)
    -> FusedGaussianAdam.step (+ the opacity and scale regularisers, once per step)  ->  GS / MCMC densification (replica-consistent)

Every rank holds a replica of the parameters and traces its own camera of the step's batch; the loss is normalised by the global batch
(number of ranks), so the replicas stay identical.  Rays are given as the 3DGRT tracer takes them: rays_o / rays_d [1,H,W,3] in ray space
and T_to_world [1,4,4] (a host tensor or array avoids a device read-back per trace)."""
from __future__ import annotations

import numpy as np
import torch
import torch.distributed as dist

import losses
import optimizers
import view_parallel
from threedgrt_tracer.tracer import Tracer
from train_step import regulariser_loss

PHASES = ("build", "trace", "loss", "backward", "exchange", "adam", "densify")


class GaussianTrainStepGRT:
    def __init__(self, params: dict, lrs: dict, conf=None, sph_degree: int = 3, selective: bool = False, group=None, eps: float = 1e-15,
                 densify_conf=None, scene_extent: float = 1.0, lambda_l1: float = 1.0, lambda_ssim: float = 0.0, background="black",
                 background_seed: int = 0, lambda_opacity: float = 0.0, lambda_scale: float = 0.0):
        """params: raw leaf tensors for optimizers.GROUPS.  conf: a config with a `render:` section read as threedgrt_tracer.Tracer reads
        it (primitive_type, particle_kernel_degree, particle_kernel_density_clamping, max_consecutive_bvh_update, min_transmittance,
        particle_kernel_max_alpha, ...).  densify_conf: densify.DensifyConfig (GS) or densify.MCMCConfig turns densification on.
        background / background_seed / lambda_opacity / lambda_scale: as in train_step.GaussianTrainStep."""
        self.params = {k: params[k] for k in optimizers.GROUPS}  # ONE dict shared with the optimizer and the densifier
        self.device = self.params["positions"].device
        self.sph_degree = int(sph_degree)
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        with torch.cuda.device(self.device):
            self.tracer = Tracer(conf if conf is not None else {"render": {}})
        self.tracer.tracer_wrapper.set_replay(True, self.device)
        self.min_transmittance = self.tracer._min_transmittance
        self.optimizer = optimizers.FusedGaussianAdam(self.params, lrs, eps=eps, selective=selective)
        self.exchange = view_parallel.FlatGradientExchange(self.n, self.device, group=group)
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
        self._rebuild = True   # the first build, and the first after densification, is a rebuild (build_acc(rebuild=True))
        self._zeros = {}       # zero d_alpha / d_dist / d_normals per resolution: the loss has no depth term, and no alpha term on black
        self.phase_events = None  # set to [] to record (phase, cuda event) pairs at the end of each phase of `step`

    @property
    def n(self) -> int:
        return int(self.params["positions"].shape[0])

    @property
    def num_update_bvh(self) -> int:
        return self.tracer.num_update_bvh

    @torch.no_grad()
    def activated(self):
        """[N,12] = pos3, sigmoid(density), normalize(rotation) (wxyz), exp(scale), 0 and [N,48] = cat(albedo, specular)
        (threedgrt_tracer/tracer.py:61, model.py:94-118)"""
        p = self.params
        particles = torch.cat([p["positions"], torch.sigmoid(p["density"]), torch.nn.functional.normalize(p["rotation"]), torch.exp(p["scale"]),
                               torch.zeros_like(p["density"])], dim=1).contiguous()
        sph = torch.cat([p["features_albedo"], p["features_specular"]], dim=1).contiguous()
        return particles, sph

    def _build(self, particles):
        """Tracer.build_acc's cadence: with density clamping every build is a rebuild, otherwise the update path is taken until
        max_consecutive_bvh_update.  The native build is a full rebuild either way; num_update_bvh counts what the reference would do."""
        t = self.tracer
        rebuild = self._rebuild or t._clamping or t.num_update_bvh >= t._max_updates
        t.tracer_wrapper.build_bvh_packed(particles)
        t.num_update_bvh = 0 if rebuild else t.num_update_bvh + 1
        self._rebuild = False

    def _zero_grads(self, H, W):
        key = (H, W)
        if key not in self._zeros:
            self._zeros = {key: (torch.zeros((1, H, W, 1), dtype=torch.float32, device=self.device),
                                 torch.zeros((1, H, W, 3), dtype=torch.float32, device=self.device))}
        return self._zeros[key]

    def _mark(self, phase):
        if self.phase_events is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.phase_events.append((phase, ev))

    @torch.no_grad()
    def render(self, rays_o, rays_d, T_to_world):
        """Forward only: (rgb [1,H,W,3], alpha [1,H,W,1], dist [1,H,W,2], hits [1,H,W,1], visibility [N,1]).  The build it needs does not
        advance the step's BVH cadence."""
        particles, sph = self.activated()
        self.tracer.tracer_wrapper.build_bvh_packed(particles)
        rgb, alpha, dst, _, hits, vis = self.tracer.tracer_wrapper.trace(self.frame, T_to_world, rays_o, rays_d, particles, sph, 0,
                                                                          self.sph_degree, self.min_transmittance)
        return rgb, alpha, dst, hits, vis

    @staticmethod
    def sensor_position(T_to_world) -> np.ndarray:
        """World position of the view's sensor: the translation of T_to_world (float32 [3])."""
        t = T_to_world.detach().cpu().numpy() if torch.is_tensor(T_to_world) else np.asarray(T_to_world)
        return np.ascontiguousarray(t.reshape(-1, 4, 4)[0, :3, 3], dtype=np.float32)

    @torch.no_grad()
    def step(self, rays_o, rays_d, T_to_world, target_rgb, all_sensor_positions=None, mask=None):
        """One optimisation step on this rank's view.  target_rgb: [H,W,3].  all_sensor_positions: [world,3] sensor positions of every
        rank's view of this step in rank order (omit on a single GPU; only the densifier reads this rank's own).  mask: optional [H,W]
        ([H,W,1], [1,H,W,1]) float CUDA tensor that multiplies prediction and target before the loss.  Returns this view's loss (a device
        scalar), the regularisers included."""
        H, W = int(rays_o.shape[1]), int(rays_o.shape[2])
        if mask is not None:
            mask = losses.mask_hw(mask, H, W)
        ot = self.tracer.tracer_wrapper
        particles, sph = self.activated()
        self._build(particles)
        self._mark("build")
        rgb, alpha, dst, nrm, hits, vis = ot.trace(self.frame, T_to_world, rays_o, rays_d, particles, sph, 0, self.sph_degree,
                                                   self.min_transmittance)
        self._mark("trace")
        target = target_rgb.reshape(H, W, 3)
        zero1, zero3 = self._zero_grads(H, W)
        d_alpha = zero1
        if not self.background.black or mask is not None:
            # composited onto the background, masked: rgb and alpha gradients (gut_loss.cu); global-batch normalisation
            loss, _, _, d_rgb, d_alpha = losses.image_loss_rgb_alpha(rgb, alpha, target.contiguous(), self.lambda_l1 / self.world,
                                                                     self.lambda_ssim / self.world, background=self.background.draw(H, W),
                                                                     mask=mask)
            loss = loss * self.world
        elif self.lambda_ssim != 0.0:
            # lambda_l1 L1 + lambda_ssim (1 - SSIM) and its rgb gradient in two launches (gut_loss.cu); global-batch normalisation
            loss, _, _, d_rgb = losses.image_loss_rgb(rgb, target.contiguous(), self.lambda_l1 / self.world, self.lambda_ssim / self.world)
            loss = loss * self.world
        else:
            diff = rgb[0] - target
            loss = self.lambda_l1 * diff.abs().mean()
            d_rgb = self.lambda_l1 * torch.sign(diff) / (diff.numel() * self.world)  # d mean|.| / d rgb, global-batch normalisation
        self._mark("loss")
        ot.trace_bwd(self.frame, T_to_world, rays_o, rays_d, rgb, alpha, dst, nrm, particles, sph, d_rgb, d_alpha, zero1, zero3, 0,
                     self.sph_degree, self.min_transmittance, out=self.exchange.out())
        self._mark("backward")
        if all_sensor_positions is None and self.world != 1:
            raise RuntimeError("all_sensor_positions is required when more than one rank trains")
        if self.densifier is not None:
            # this view's own position gradient, before the exchange (weighted by the distance to THIS view's sensor, gs.py:127-137);
            # x world undoes the global-batch normalisation so that the thresholds keep their per-view meaning
            self.densifier.update_gradient_buffer(self.exchange.d_particles[:, 0:3] * float(self.world), self.sensor_position(T_to_world))
        d_particles, d_sph = self.exchange.exchange()
        if self.optimizer.selective and self.world > 1:
            dist.all_reduce(vis, op=dist.ReduceOp.MAX, group=self.group)  # visible in any view of the batch (SURVEY 8e)
        self._mark("exchange")
        # the regularisers belong to the step once (every rank holds the same parameters): added after the exchange, no 1 / world
        reg = {}
        if self.lambda_opacity != 0.0 or self.lambda_scale != 0.0:
            loss = loss + regulariser_loss(particles, self.lambda_opacity, self.lambda_scale)
            reg = dict(lambda_opacity=self.lambda_opacity, lambda_scale=self.lambda_scale)
        self.optimizer.step(d_particles, d_sph, visibility=vis if self.optimizer.selective else None, **reg)
        self._mark("adam")
        self.frame += 1
        if self.densifier is not None and self.densifier.post_optimizer_step(self.frame, self.scene_extent, positions_lr=self.optimizer.lrs["positions"]):
            # the Gaussians changed (identically on every rank): re-capacity the exchange buffer, rebuild the BVH from scratch next step
            self._rebuild = True
            if self.exchange.n != self.n:
                self.exchange = view_parallel.FlatGradientExchange(self.n, self.device, group=self.group)
        self._mark("densify")
        return loss

    def bytes_on_wire(self) -> int:
        return self.exchange.bytes_on_wire()

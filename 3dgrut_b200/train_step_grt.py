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

import losses
import view_parallel
from threedgrt_tracer.tracer import Tracer
from train_step import TrainStep

PHASES = ("build", "trace", "loss", "backward", "exchange", "adam", "densify")


class GaussianTrainStepGRT(TrainStep):
    """Constructor as train_step.TrainStep's; conf is read as threedgrt_tracer.Tracer reads it (primitive_type, particle_kernel_degree,
    particle_kernel_density_clamping, max_consecutive_bvh_update, min_transmittance, particle_kernel_max_alpha, ...).  `phase_events`
    records every phase of PHASES."""

    def _init_renderer(self, conf):
        with torch.cuda.device(self.device):
            self.tracer = Tracer(conf)
        self.tracer.tracer_wrapper.set_replay(True, self.device)
        self.min_transmittance = self.tracer._min_transmittance
        self._rebuild = True   # the first build, and the first after densification, is a rebuild (build_acc(rebuild=True))
        self._zeros = {}       # zero d_alpha / d_dist / d_normals per resolution: the loss has no depth term, and no alpha term on black

    def _new_exchange(self):
        return view_parallel.FlatGradientExchange(self.n, self.device, group=self.group)

    def _image_loss(self, pred, target, lambda_l1, lambda_ssim, background, mask):
        rgb, alpha, zero1 = pred
        if background is None and mask is None:  # black, unmasked: the rgb loss, no alpha gradient
            loss, _, _, d_rgb = losses.image_loss_rgb(rgb, target, lambda_l1, lambda_ssim)
            return loss, (d_rgb, zero1)
        # composited onto the background, masked: rgb and alpha gradients (gut_loss.cu)
        loss, _, _, d_rgb, d_alpha = losses.image_loss_rgb_alpha(rgb, alpha, target, lambda_l1, lambda_ssim, background=background, mask=mask)
        return loss, (d_rgb, d_alpha)

    def _l1_grads(self, pred, diff):
        return self._d_l1(diff), pred[2]

    def _densified(self):
        self._rebuild = True  # the Gaussians changed: rebuild the BVH from scratch next step
        super()._densified()

    @property
    def num_update_bvh(self) -> int:
        return self.tracer.num_update_bvh

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
        zero1, zero3 = self._zero_grads(H, W)
        loss, (d_rgb, d_alpha) = self._loss((rgb, alpha, zero1), rgb[0], target_rgb.reshape(H, W, 3), H, W, mask)
        self._mark("loss")
        ot.trace_bwd(self.frame, T_to_world, rays_o, rays_d, rgb, alpha, dst, nrm, particles, sph, d_rgb, d_alpha, zero1, zero3, 0,
                     self.sph_degree, self.min_transmittance, out=self.exchange.out())
        self._mark("backward")
        my_position = self.sensor_position(T_to_world) if self.densifier is not None else None
        return self._update(loss, particles, vis, all_sensor_positions, my_position)

    def bytes_on_wire(self) -> int:
        return self.exchange.bytes_on_wire()

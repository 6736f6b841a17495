"""View-parallel training step for the SH Gaussian model on the 3DGRT path: the ray-traced twin of train_step.GaussianTrainStep.

Replaces Tracer.render + loss + autograd + per-parameter Adam of the reference trainer (threedgrut/trainer.py:1119-1263 with the 3DGRT
renderer) by the pieces of this repository wired together, with no autograd graph:

    activations (model.py:102-118)  ->  LBVH build from the [N,12] record (cadence of Tracer.build_acc, threedgrt_tracer/tracer.py:198-216)
    -> OptixTracer.trace (hit lists recorded)  ->  image loss gradient (L1, or L1 + SSIM with losses.image_loss_rgb; with a background,
       a mask or the linear-to-sRGB post-processing, losses.image_loss_rgb_alpha, which also gives the alpha gradient)
    -> OptixTracer.trace_bwd (hit-list replay) into the exchange buffer  ->  FlatGradientExchange (one all-reduce of 240 B x N)
    -> FusedGaussianAdam.step (+ the opacity and scale regularisers, once per step)  ->  GS / MCMC densification (replica-consistent)

Every rank holds a replica of the parameters and traces its own camera of the step's batch; the loss is normalised by the global batch
(number of ranks), so the replicas stay identical.  Rays are given as the 3DGRT tracer takes them: rays_o / rays_d [1,H,W,3] in ray space
and T_to_world [1,4,4] (a host tensor or array avoids a device read-back per trace)."""
from __future__ import annotations

import numpy as np
import torch

import view_parallel
from threedgrt_tracer.tracer import Tracer
from train_step import Frame, TrainStep

PHASES = ("build", "trace", "loss", "backward", "exchange", "adam", "densify")


class GaussianTrainStepGRT(TrainStep):
    """Constructor as train_step.TrainStep's; conf is read as threedgrt_tracer.Tracer reads it (primitive_type, particle_kernel_degree,
    particle_kernel_density_clamping, max_consecutive_bvh_update, min_transmittance, particle_kernel_max_alpha, ...).  `phase_events`
    records every phase of PHASES."""

    PHASES = PHASES

    def _init_renderer(self, conf):
        with torch.cuda.device(self.device):
            self.tracer = Tracer(conf)
        self.tracer.tracer_wrapper.set_replay(True, self.device)
        self.min_transmittance = self.tracer._min_transmittance
        self._rebuild = True   # the first build, and the first after densification, is a rebuild (build_acc(rebuild=True))

    def _new_exchange(self):
        return view_parallel.FlatGradientExchange(self.n, self.device, group=self.group)

    def _densified(self):
        self._rebuild = True  # the Gaussians changed: rebuild the BVH from scratch next step
        super()._densified()

    @property
    def num_update_bvh(self) -> int:
        return self.tracer.num_update_bvh

    def state_dict(self) -> dict:
        return {**super().state_dict(), "num_update_bvh": int(self.tracer.num_update_bvh)}

    def _load_extra(self, state: dict, take):
        """The BVH cadence counter; the next build is a rebuild (_densified sets _rebuild), as after the reference's build_acc on resume."""
        super()._load_extra(state, take)
        self.tracer.num_update_bvh = int(state.get("num_update_bvh") or 0)

    def _build(self, particles, train):
        """The packed BVH of `particles`.  train: Tracer.build_acc's cadence -- with density clamping every build is a rebuild, otherwise
        the update path is taken until max_consecutive_bvh_update; the native build is a full rebuild either way, num_update_bvh counts what
        the reference would do.  Otherwise (render, metrics_inputs) the build does not advance the cadence."""
        t = self.tracer
        t.tracer_wrapper.build_bvh_packed(particles)
        if train:
            rebuild = self._rebuild or t._clamping or t.num_update_bvh >= t._max_updates
            t.num_update_bvh = 0 if rebuild else t.num_update_bvh + 1
            self._rebuild = False
        self._mark("build")

    def _forward(self, view, particles, sph, train):
        rays_o, rays_d, T_to_world = view
        self._build(particles, train)
        rgb, alpha, dst, nrm, hits, vis = self.tracer.tracer_wrapper.trace(self.frame, T_to_world, rays_o, rays_d, particles, sph, 0, self.sph_degree,
                                                                          self.min_transmittance, normals=False)  # the loss reads no normals
        self._mark("trace")
        return Frame(rgb[0], 3, rgb[0], alpha[0], hits[0], vis, (view, particles, sph, rgb, alpha, dst, nrm))

    def _backward(self, frame, d_rgb, d_alpha):
        """The loss has no depth or normal term, and no alpha term on black: those gradients are zero."""
        (rays_o, rays_d, T_to_world), particles, sph, rgb, alpha, dst, nrm = frame.saved
        H, W = frame.rgb.shape[:2]
        zero1, zero3 = self._zeros(H, W, 1), self._zeros(H, W, 3)
        self.tracer.tracer_wrapper.trace_bwd(self.frame, T_to_world, rays_o, rays_d, rgb, alpha, dst, nrm, particles, sph, d_rgb,
                                             zero1 if d_alpha is None else d_alpha, zero1, zero3, 0, self.sph_degree, self.min_transmittance,
                                             out=self.exchange.out())
        self._mark("backward")
        return ()

    def _sensor_position(self, frame):
        return self.sensor_position(frame.saved[0][2])

    @torch.no_grad()
    def render(self, rays_o, rays_d, T_to_world):
        """Forward only: (rgb [1,H,W,3], alpha [1,H,W,1], dist [1,H,W,2], hits [1,H,W,1], visibility [N,1]); rgb encoded under
        post_processing.  The build it needs does not advance the step's BVH cadence."""
        f = self._forward((rays_o, rays_d, T_to_world), *self.activated(), train=False)
        _, _, _, rgb, alpha, dst, _ = f.saved
        return self._post_process(rgb), alpha, dst, f.hits[None], f.vis

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
        return self._step((rays_o, rays_d, T_to_world), target_rgb, all_sensor_positions, mask)

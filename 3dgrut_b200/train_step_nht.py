"""View-parallel training steps for the Neural Harmonic Texture (NHT) model (model.feature_type: nht) on both renderers:
GaussianTrainStepNHT (3DGUT) and GaussianTrainStepGRTNHT (3DGRT), on the TrainStep core of train_step.py.

Replaces Tracer.render -> apply_feature_decoder -> apply_background -> loss -> autograd -> two torch.optim.Adam of the reference trainer
(threedgrut/trainer.py:1119-1263, utils/render.py:54-92) with no autograd graph:

    activations  ->  render the [N,48] features (3DGUT: [H,W,25] = 24 features + alpha; 3DGRT: packed BVH build, then [1,H,W,24] + alpha)
    -> FeatureDecoder forward on the world ray directions normalize(R_c2w rays_d)  ->  image loss on the decoded rgb (L1, L1 + SSIM, or
       composited onto the background / masked, which gives the render's alpha its gradient)
    -> decoder backward: d_features into a per-resolution buffer, d_params straight into the tail of the exchange buffer
    -> render backward into the exchange buffer  ->  FlatGradientExchange ([N,12] + [N,48] + decoder params in ONE all-reduce)
    -> FusedNHTAdam (the Gaussians and the decoder in one launch)  ->  FeatureDecoder.ema_update  ->  GS / MCMC densification

The exchange is flat on both renderers: a Gaussian's feature gradient in one view depends on where each ray hits it, so it has no low-rank
per-view summary like the SH gradient's on the 3DGUT path.  Colour refinement (model.nht_decoder.color_refine_steps, trainer.py:153-195)
freezes positions, density, rotation and scale, drops the opacity and scale regularisers and suspends the densifier for the last steps."""
from __future__ import annotations

import numpy as np
import torch

import feature_decoder as fd
import losses
import optimizers
import view_parallel
from b200_native import NHT_FEATURE_DIM, cfg_get, nht_feature_config
from threedgut_tracer.tracer import SplatRaster
from train_step import TrainStep, particle_record
from train_step_grt import GaussianTrainStepGRT

PHASES = ("render", "decode", "loss", "decode_backward", "render_backward", "exchange", "adam", "densify")
PHASES_GRT = ("build",) + PHASES
GEOMETRY = ("positions", "density", "rotation", "scale")  # trainer.py:95, frozen during colour refinement
RAY_FEATURES = NHT_FEATURE_DIM // 2  # features per ray the renderers composite


def color_refine_start_step(conf) -> int:
    """Trainer._get_color_refine_start_step (trainer.py:153-163): the first step of the colour-only refinement, n_iterations when there is
    none."""
    n_iterations = int(cfg_get(conf, "n_iterations", 0))
    if str(cfg_get(conf, "model.feature_type", "sh")).lower() != "nht":
        return n_iterations
    steps = int(cfg_get(conf, "model.nht_decoder.color_refine_steps", 0) or 0)
    if steps <= 0:
        return n_iterations
    return max(0, n_iterations - steps)


def nht_step_settings(conf, decoder=None) -> dict:
    """What the NHT steps read from the config: {"weight_decay": model.nht_decoder.reg_weight, "color_refine_start": first frozen step or
    None}.  Settings the steps do not build raise NotImplementedError naming the key (none of them is used by the shipped NHT apps).
    Pure config logic: needs no GPU."""
    if nht_feature_config(conf, "NHT training step") is None:
        raise ValueError("model.feature_type: the NHT training steps train model.feature_type 'nht'")
    if not bool(cfg_get(conf, "model.nht_decoder.enabled", True)):
        raise NotImplementedError("model.nht_decoder.enabled=False: the NHT training steps decode through the feature decoder")
    if bool(cfg_get(conf, "model.nht_decoder.unpremultiply_alpha", False)) or bool(getattr(decoder, "unpremultiply_alpha", False)):
        raise NotImplementedError("model.nht_decoder.unpremultiply_alpha=True is not built in the NHT training steps")
    if bool(cfg_get(conf, "model.nht_decoder.center_ray_encoding", False)):
        raise NotImplementedError("model.nht_decoder.center_ray_encoding=True is not built in the NHT training steps")
    start = color_refine_start_step(conf)
    refine = start < int(cfg_get(conf, "n_iterations", 0))  # Trainer._is_color_refine_active
    return {"weight_decay": float(cfg_get(conf, "model.nht_decoder.reg_weight", 0.0)), "color_refine_start": start if refine else None}


def c2w_rotation_from_pose7(pose) -> np.ndarray:
    """R_c2w [3,3] (float64) of a 3DGUT sensor pose [t.xyz, q.xyzw] of the world -> sensor transform: the transpose of q's rotation."""
    p = np.asarray(pose.detach().cpu().numpy() if torch.is_tensor(pose) else pose, dtype=np.float64).reshape(-1)
    x, y, z, w = p[3:7] / np.linalg.norm(p[3:7])
    r_w2s = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                      [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                      [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    return r_w2s.T


def c2w_rotation_from_T(T_to_world) -> np.ndarray:
    """R_c2w [3,3] (float64) of a 3DGRT T_to_world [1,4,4] (or [4,4])."""
    t = T_to_world.detach().cpu().numpy() if torch.is_tensor(T_to_world) else np.asarray(T_to_world)
    return np.asarray(t, dtype=np.float64).reshape(-1, 4, 4)[0, :3, :3]


def world_ray_directions(R_c2w, rays_d: torch.Tensor) -> torch.Tensor:
    """[H*W,3] = normalize(R_c2w rays_d) as apply_feature_decoder computes the decoder's directions (utils/render.py:75-83)."""
    R = torch.as_tensor(np.asarray(R_c2w, np.float32), device=rays_d.device)
    return torch.nn.functional.normalize(rays_d.reshape(-1, 3).float() @ R.T, dim=-1).contiguous()


class _NHTStep:
    """What both NHT steps add to their renderer's step: the decoder, the NHT optimizer and exchange, the loss on the decoded rgb, the
    decoder backward and colour refinement.  Mixed in ahead of the renderer's step class."""

    GROUPS = optimizers.NHT_GROUPS

    def __init__(self, params: dict, lrs: dict, decoder: fd.FeatureDecoder, conf, **kw):
        """params: raw leaf tensors for optimizers.NHT_GROUPS (features [N,48] raw).  lrs: learning rates of NHT_GROUPS and "decoder".
        decoder: the FeatureDecoder on the Gaussians' device; its `network.params` are trained in place (Adam with eps 1e-8 and
        weight_decay model.nht_decoder.reg_weight, trainer.py:573-577) and its EMA is updated every step.  conf: the renderer's config with
        model.feature_type: nht; n_iterations and model.nht_decoder.color_refine_steps set colour refinement.  Other arguments as
        TrainStep's (sph_degree is not used)."""
        settings = nht_step_settings(conf, decoder)
        self.decoder = decoder
        self.decoder_weight_decay = settings["weight_decay"]
        self.color_refine_start = settings["color_refine_start"]
        self._buffers = {}  # per resolution: the decoder's backward workspace and the [H*W,24] feature gradient
        super().__init__(params, lrs, conf=conf, **kw)

    def _new_optimizer(self, lrs, eps, selective):
        return optimizers.FusedNHTAdam(self.params, self.decoder.network.params, lrs, eps=eps, selective=selective,
                                       decoder_weight_decay=self.decoder_weight_decay)

    def _new_exchange(self):
        return view_parallel.FlatGradientExchange(self.n, self.device, group=self.group, tail=self.decoder.network.params.numel())

    _image_loss = GaussianTrainStepGRT._image_loss  # the decoded rgb and the render's alpha are split as on the 3DGRT layout
    _l1_grads = GaussianTrainStepGRT._l1_grads

    @torch.no_grad()
    def activated(self):
        """[N,12] activated record and the raw [N,48] features."""
        return particle_record(self.params), self.params["features"].contiguous()

    def _geometry_frozen(self) -> bool:
        return self.color_refine_start is not None and self.frame >= self.color_refine_start

    def _adam(self, d_particles, d_features, vis, reg):
        self.optimizer.step(d_particles, d_features, self.exchange.d_tail, visibility=vis, frozen=GEOMETRY if self._geometry_frozen() else (),
                            **reg)
        self.decoder.ema_update(self.frame)

    def _decode(self, features, dirs):
        """rgb [H*W,3] of the [H*W,24] composited features."""
        return fd.decode(features, dirs, self.decoder.network.params.data, self.decoder.config)

    def _decode_backward(self, features, dirs, d_rgb):
        """d_features [H*W,24]; the decoder's parameter gradient goes to the exchange buffer's tail."""
        rows = int(features.shape[0])
        if rows not in self._buffers:
            self._buffers = {rows: (fd.backward_workspace(self.decoder.config, rows, self.device),
                                    torch.empty((rows, RAY_FEATURES), dtype=torch.float32, device=self.device))}
        ws, d_features = self._buffers[rows]
        fd.decode_backward(features, dirs, self.decoder.network.params.data, self.decoder.config, d_rgb.reshape(rows, 3), d_features,
                           self.exchange.d_tail, ws)
        return d_features


class GaussianTrainStepNHT(_NHTStep, TrainStep):
    """NHT step on the 3DGUT path.  Constructor: (params, lrs, decoder, conf, **TrainStep options); `phase_events` records PHASES."""

    def _init_renderer(self, conf):
        self.raster = SplatRaster(conf)
        self._zeros = {}

    def _zero(self, H, W):
        if (H, W) not in self._zeros:
            self._zeros = {(H, W): torch.zeros((H, W, 1), dtype=torch.float32, device=self.device)}
        return self._zeros[(H, W)]

    def _forward(self, rays_o, rays_d, sensor, pose):
        particles, feats = self.activated()
        feats = self.raster._nht_features(feats)  # rounded once (fp16 under render.particle_feature_half) for the forward and the backward
        H, W = int(rays_o.shape[1]), int(rays_o.shape[2])
        out, dst, hits, vis = self.raster.trace(self.frame, 0, particles, feats, rays_o, rays_d, None, sensor, 0, 1, pose, pose)
        self._mark("render")
        features = out[..., :RAY_FEATURES].reshape(H * W, RAY_FEATURES).contiguous()
        alpha = out[..., RAY_FEATURES:].contiguous()
        dirs = world_ray_directions(c2w_rotation_from_pose7(pose), rays_d)
        rgb = self._decode(features, dirs).view(H, W, 3)
        self._mark("decode")
        return particles, feats, out, dst, vis, features, alpha, dirs, rgb

    @torch.no_grad()
    def render(self, rays_o, rays_d, sensor, pose):
        """Forward only: (decoded rgb [H,W,3], alpha [H,W,1])."""
        out = self._forward(rays_o, rays_d, sensor, pose)
        return out[8], out[6]

    @torch.no_grad()
    def step(self, rays_o, rays_d, sensor, pose, target_rgb, all_sensor_positions=None, mask=None):
        """One optimisation step on this rank's view; arguments as GaussianTrainStep.step.  Returns this view's loss (a device scalar), the
        regularisers included while they apply."""
        H, W = int(rays_o.shape[1]), int(rays_o.shape[2])
        if mask is not None:
            mask = losses.mask_hw(mask, H, W)
        particles, feats, out, dst, vis, features, alpha, dirs, rgb = self._forward(rays_o, rays_d, sensor, pose)
        zero1 = self._zero(H, W)
        loss, (d_rgb, d_alpha) = self._loss((rgb, alpha, zero1), rgb, target_rgb.reshape(H, W, 3), H, W, mask)
        self._mark("loss")
        d_features = self._decode_backward(features, dirs, d_rgb)
        self._mark("decode_backward")
        d_out = torch.cat([d_features.view(H, W, RAY_FEATURES), d_alpha.reshape(H, W, 1)], -1)
        self.raster.trace_bwd(self.frame, 0, particles, feats, rays_o, rays_d, None, sensor, 0, 1, pose, pose, out, d_out, dst, zero1,
                              out=self.exchange.out())
        self._mark("render_backward")
        my_position = self.raster.sensor_position(sensor, pose, pose, W, H) if self.densifier is not None else None
        return self._update(loss, particles, vis, all_sensor_positions, my_position)

    def bytes_on_wire(self) -> int:
        return self.exchange.bytes_on_wire()


class GaussianTrainStepGRTNHT(_NHTStep, GaussianTrainStepGRT):
    """NHT step on the 3DGRT path.  Constructor: (params, lrs, decoder, conf, **TrainStep options), conf read as threedgrt_tracer.Tracer
    reads it; `phase_events` records PHASES_GRT."""

    def _forward(self, rays_o, rays_d, T_to_world, particles, feats):
        """After the build from `particles`."""
        ot = self.tracer.tracer_wrapper
        H, W = int(rays_o.shape[1]), int(rays_o.shape[2])
        feat, alpha, dst, nrm, hits, vis = ot.trace(self.frame, T_to_world, rays_o, rays_d, particles, feats, 0, 0, self.min_transmittance)
        self._mark("render")
        features = feat.view(H * W, RAY_FEATURES)
        dirs = world_ray_directions(c2w_rotation_from_T(T_to_world), rays_d)
        rgb = self._decode(features, dirs).view(H, W, 3)
        self._mark("decode")
        return particles, feats, feat, alpha, dst, nrm, vis, dirs, rgb

    @torch.no_grad()
    def render(self, rays_o, rays_d, T_to_world):
        """Forward only: (decoded rgb [H,W,3], alpha [H,W,1]).  The build it needs does not advance the step's BVH cadence."""
        particles, feats = self.activated()
        self.tracer.tracer_wrapper.build_bvh_packed(particles)
        out = self._forward(rays_o, rays_d, T_to_world, particles, feats)
        return out[8], out[3][0]

    @torch.no_grad()
    def step(self, rays_o, rays_d, T_to_world, target_rgb, all_sensor_positions=None, mask=None):
        """One optimisation step on this rank's view; arguments as GaussianTrainStepGRT.step."""
        H, W = int(rays_o.shape[1]), int(rays_o.shape[2])
        if mask is not None:
            mask = losses.mask_hw(mask, H, W)
        particles, feats = self.activated()
        self._build(particles)
        self._mark("build")
        _, _, feat, alpha, dst, nrm, vis, dirs, rgb = self._forward(rays_o, rays_d, T_to_world, particles, feats)
        zero1, zero3 = self._zero_grads(H, W)
        loss, (d_rgb, d_alpha) = self._loss((rgb, alpha, zero1), rgb, target_rgb.reshape(H, W, 3), H, W, mask)
        self._mark("loss")
        d_features = self._decode_backward(feat.view(H * W, RAY_FEATURES), dirs, d_rgb)
        self._mark("decode_backward")
        self.tracer.tracer_wrapper.trace_bwd(self.frame, T_to_world, rays_o, rays_d, feat, alpha, dst, nrm, particles, feats,
                                             d_features.view(1, H, W, RAY_FEATURES), d_alpha, zero1, zero3, 0, 0, self.min_transmittance,
                                             out=self.exchange.out())
        self._mark("render_backward")
        my_position = self.sensor_position(T_to_world) if self.densifier is not None else None
        return self._update(loss, particles, vis, all_sensor_positions, my_position)

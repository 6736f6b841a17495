"""View-parallel training step for the 3DGRUT hybrid (BASELINE.json config 5): primary camera rays rasterised through 3DGUT, their mirror
reflections off a plane ray-traced through 3DGRT, both on the same Gaussians, with the two gradients summed in one exchange buffer.

hybrid.render_hybrid is the autograd composition of the two tracers; this step replaces it, the loss, autograd and the per-parameter Adam by
the pieces of this repository wired together, with no autograd graph:

    activations  ->  hybrid_rays (the world-space mirror rays and their hit mask, csrc/hybrid.cu)  ->  SplatRaster.trace (primary)
    -> packed LBVH build  ->  OptixTracer.trace of the [1,H,W,3] secondary rays (identity ray-to-world)
    -> hybrid_composite: rgb = primary_rgb + reflectivity (1 - primary alpha) hit secondary_rgb
    -> image loss (L1; L1 + SSIM; or composited onto the background with the PRIMARY alpha and masked, which gives that alpha a gradient)
    -> hybrid_composite_bwd -> SplatRaster.trace_bwd into the exchange buffer -> OptixTracer.trace_bwd(accumulate=True) into the same rows
    -> FlatGradientExchange (one all-reduce of 240 B x N)  ->  FusedGaussianAdam  ->  GS / MCMC densification (BVH rebuilt after it)

Rays that miss the mirror are traced too, with weight 0, as render_hybrid traces them.  Both tracers read one `render:` section; keys it
does not set take the values of the reference's configs/render/3dgut.yaml, so both passes render the same kernel."""
from __future__ import annotations

import copy

import numpy as np
import torch

import b200_native as native
import losses
from b200_native import cfg_get, ptr
from threedgut_tracer.tracer import ShutterType, SplatRaster, Tracer as GutTracer
from train_step_grt import GaussianTrainStepGRT

PHASES = ("rays", "primary", "build", "secondary", "loss", "backward_primary", "backward_secondary", "exchange", "adam", "densify")
MIRROR_DEFAULTS = dict(plane_point=(0.0, 0.0, -1.2), plane_normal=(0.0, 0.0, 1.0), reflectivity=0.3)  # render_hybrid's
# configs/render/3dgut.yaml (which composes configs/render/3dgrt.yaml): the render keys either tracer reads, as the hybrid fills them in
RENDER_DEFAULTS = {
    "particle_kernel_degree": 2, "particle_kernel_min_response": 0.0113, "particle_kernel_min_alpha": 1.0 / 255.0,
    "particle_kernel_max_alpha": 0.99, "particle_kernel_density_clamping": True, "particle_radiance_sph_degree": 3,
    "primitive_type": "instances", "min_transmittance": 0.0001, "max_consecutive_bvh_update": 15,
}


def hybrid_render_conf(conf) -> dict:
    """A copy of conf whose `render:` section has every key of RENDER_DEFAULTS (the user's values kept), read by both tracers.
    model.feature_type nht raises NotImplementedError.  Pure config logic: needs no GPU."""
    if str(cfg_get(conf, "model.feature_type", "sh")).lower() != "sh":
        raise NotImplementedError("model.feature_type: the hybrid step trains SH radiance only (NHT features are not built for it)")
    out = copy.deepcopy(conf) if isinstance(conf, dict) else {"render": copy.deepcopy(dict(cfg_get(conf, "render", {})))}
    render = dict(out.get("render") or {})
    for key, value in RENDER_DEFAULTS.items():
        if render.get(key) is None:
            render[key] = value
    if abs(float(render["particle_kernel_min_alpha"]) - 1.0 / 255.0) > 1e-12:
        # the 3DGRT tracer's threshold is fixed (grtb200_default_config): another value would give the two passes different kernels
        raise NotImplementedError(f"render.particle_kernel_min_alpha={render['particle_kernel_min_alpha']}: the hybrid step is built for 1/255")
    out["render"] = render
    return out


def mirror_settings(mirror=None) -> dict:
    """The mirror of the step: {"plane_point": float32 [3], "plane_normal": unit float32 [3], "reflectivity": float}.  A zero normal or a
    reflectivity outside [0, 1] raises NotImplementedError naming the key.  Pure config logic: needs no GPU."""
    m = dict(MIRROR_DEFAULTS)
    if mirror is not None:
        unknown = set(mirror) - set(MIRROR_DEFAULTS)
        if unknown:
            raise ValueError(f"mirror: unknown keys {sorted(unknown)} (expected {sorted(MIRROR_DEFAULTS)})")
        m.update(mirror)
    p0 = np.asarray(m["plane_point"], np.float32).reshape(3)
    n = np.asarray(m["plane_normal"], np.float32).reshape(3)
    norm = np.float32(np.sqrt(np.sum(n * n, dtype=np.float32)))
    if not np.isfinite(norm) or norm == 0:
        raise NotImplementedError(f"mirror.plane_normal={tuple(m['plane_normal'])}: the plane needs a non-zero normal")
    r = float(m["reflectivity"])
    if not 0.0 <= r <= 1.0:
        raise NotImplementedError(f"mirror.reflectivity={r}: the hybrid composite is built for a reflectivity in [0, 1]")
    return {"plane_point": p0, "plane_normal": (n / norm).astype(np.float32), "reflectivity": r}


def check_sensor(sensor):
    """Refuse a rolling-shutter sensor (NotImplementedError naming shutter_type): the secondary rays are spawned with one pose."""
    shutter = ShutterType(getattr(sensor, "shutter_type", ShutterType.GLOBAL))
    if shutter != ShutterType.GLOBAL:
        raise NotImplementedError(f"shutter_type={shutter.name}: the hybrid step reflects the rays of a global-shutter sensor only")


def _c2w_rows(T_to_world) -> np.ndarray:
    """The 12 floats of the camera-to-world [R | t] (row-major 3x4, host float32) of T_to_world [1,4,4] / [4,4]."""
    t = T_to_world.detach().cpu().numpy() if torch.is_tensor(T_to_world) else np.asarray(T_to_world)
    return np.ascontiguousarray(np.asarray(t, np.float32).reshape(-1, 4, 4)[0, :3, :4])


def _check(rc: int, what: str):
    if rc != 0:
        raise RuntimeError(f"{what} failed ({rc})")


def _stream(dev) -> int:
    return torch.cuda.current_stream(dev).cuda_stream


def hybrid_rays(rays_o, rays_d, T_to_world, plane_point, plane_normal, out=None):
    """World-space mirror rays of camera rays (hybrid.mirror_rays per pixel, gutb200_hybrid_rays).  rays_o / rays_d: [1,H,W,3] float32 CUDA
    tensors in camera space; T_to_world: [1,4,4] or [4,4] camera-to-world (host tensor or array: no read-back); plane_normal: unit.
    Returns (origins [1,H,W,3], directions [1,H,W,3], hit [H*W] float 0 / 1); `out` = that triple to write into."""
    rays_o, rays_d = rays_o.contiguous(), rays_d.contiguous()
    pixels = rays_o.numel() // 3
    dev = rays_o.device
    if out is None:
        out = (torch.empty((1,) + tuple(rays_o.shape[-3:]), dtype=torch.float32, device=dev),
               torch.empty((1,) + tuple(rays_o.shape[-3:]), dtype=torch.float32, device=dev), torch.empty(pixels, dtype=torch.float32, device=dev))
    r = _c2w_rows(T_to_world)
    p0, n = np.ascontiguousarray(plane_point, np.float32), np.ascontiguousarray(plane_normal, np.float32)
    _check(native.load().gutb200_hybrid_rays(_stream(dev), pixels, ptr(rays_o), ptr(rays_d), r.ctypes.data, p0.ctypes.data, n.ctypes.data,
                                             ptr(out[0]), ptr(out[1]), ptr(out[2])), "gutb200_hybrid_rays")
    return out


def hybrid_composite(primary_rgba, secondary_rgb, hit, reflectivity: float, out=None):
    """[H,W,3] = primary rgb + reflectivity (1 - primary alpha) hit secondary_rgb (render_hybrid's pred_features_hybrid,
    gutb200_hybrid_composite).  primary_rgba: the 3DGUT [H,W,4]; secondary_rgb: the 3DGRT [1,H,W,3] (or [H*W,3]); hit: [H*W]."""
    H, W = int(primary_rgba.shape[0]), int(primary_rgba.shape[1])
    primary_rgba, secondary_rgb, hit = primary_rgba.contiguous(), secondary_rgb.contiguous(), hit.contiguous()
    if out is None:
        out = torch.empty((H, W, 3), dtype=torch.float32, device=primary_rgba.device)
    _check(native.load().gutb200_hybrid_composite(_stream(primary_rgba.device), H * W, ptr(primary_rgba), ptr(secondary_rgb), ptr(hit),
                                                  float(reflectivity), ptr(out)), "gutb200_hybrid_composite")
    return out


def hybrid_composite_bwd(primary_rgba, secondary_rgb, hit, reflectivity: float, d_rgb, d_alpha=None, out=None):
    """Adjoint of hybrid_composite (gutb200_hybrid_composite_bwd): d_rgb [H,W,3] and the loss's gradient on the primary alpha d_alpha
    ([H,W] / [H,W,1] or None = 0) -> (d_rgba [H,W,4], the 3DGUT backward's input; d_secondary [1,H,W,3], the 3DGRT backward's).  Every
    element is written."""
    H, W = int(primary_rgba.shape[0]), int(primary_rgba.shape[1])
    dev = primary_rgba.device
    primary_rgba, secondary_rgb, hit, d_rgb = primary_rgba.contiguous(), secondary_rgb.contiguous(), hit.contiguous(), d_rgb.contiguous()
    if d_alpha is not None:
        d_alpha = d_alpha.contiguous()
    if out is None:
        out = (torch.empty((H, W, 4), dtype=torch.float32, device=dev), torch.empty((1, H, W, 3), dtype=torch.float32, device=dev))
    _check(native.load().gutb200_hybrid_composite_bwd(_stream(dev), H * W, ptr(primary_rgba), ptr(secondary_rgb), ptr(hit), float(reflectivity),
                                                      ptr(d_rgb), None if d_alpha is None else ptr(d_alpha), ptr(out[0]), ptr(out[1])),
           "gutb200_hybrid_composite_bwd")
    return out


class GaussianTrainStepHybrid(GaussianTrainStepGRT):
    """Constructor as train_step.TrainStep's plus `mirror` (dict of MIRROR_DEFAULTS keys).  conf's `render:` section is read by both
    tracers after hybrid_render_conf; the 3DGRT-only keys (primitive_type, particle_kernel_density_clamping, max_consecutive_bvh_update) as
    the 3DGRT step reads them.  Rays are given as the 3DGUT step takes them (camera space, [1,H,W,3], with its sensor) together with the
    camera-to-world T_to_world [1,4,4] (a host tensor or array), from which the 3DGUT pose is derived as threedgut_tracer.Tracer does.
    `phase_events` records PHASES."""

    def __init__(self, params: dict, lrs: dict, conf=None, mirror=None, **kw):
        m = mirror_settings(mirror)
        self.plane_point, self.plane_normal, self.reflectivity = m["plane_point"], m["plane_normal"], m["reflectivity"]
        super().__init__(params, lrs, conf=hybrid_render_conf(conf if conf is not None else {"render": {}}), **kw)

    def _init_renderer(self, conf):
        super()._init_renderer(conf)  # the 3DGRT tracer of the secondary rays
        self.raster = SplatRaster(conf)
        self._identity = torch.eye(4, dtype=torch.float32)[None]  # the secondary rays are in world space (host: no read-back per trace)
        self._buffers = {}

    def _scratch(self, H, W):
        """Per-resolution buffers: the secondary rays and hit mask, the composite and its gradients."""
        key = (H, W)
        if key not in self._buffers:
            e = lambda *s: torch.empty(s, dtype=torch.float32, device=self.device)  # noqa: E731
            self._buffers = {key: dict(rays=(e(1, H, W, 3), e(1, H, W, 3), e(H * W)), rgb=e(H, W, 3), grads=(e(H, W, 4), e(1, H, W, 3)),
                                       zero_dist=torch.zeros((H, W, 1), dtype=torch.float32, device=self.device))}
        return self._buffers[key]

    @staticmethod
    def pose_from_c2w(T_to_world) -> np.ndarray:
        """The 3DGUT world->sensor pose [t, q.xyzw] of T_to_world, exactly as threedgut_tracer.Tracer derives it."""
        t = T_to_world.detach().cpu() if torch.is_tensor(T_to_world) else np.asarray(T_to_world)
        return GutTracer._pose_from_c2w(t.reshape(-1, 4, 4)[0])

    def _forward(self, rays_o, rays_d, sensor, T_to_world, particles, sph, train):
        """Rays, primary trace, build, secondary trace, composite.  train: the step's BVH cadence and buffers (True), or a plain rebuild
        and new tensors (render)."""
        check_sensor(sensor)
        H, W = int(rays_o.shape[1]), int(rays_o.shape[2])
        buf = self._scratch(H, W) if train else {"rays": None, "rgb": None}
        sec_o, sec_d, hit = hybrid_rays(rays_o, rays_d, T_to_world, self.plane_point, self.plane_normal, out=buf["rays"])
        self._mark("rays")
        pose = self.pose_from_c2w(T_to_world)
        rgba, dst, _, vis_p = self.raster.trace(self.frame, self.sph_degree, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose)
        self._mark("primary")
        if train:
            self._build(particles)
        else:
            self.tracer.tracer_wrapper.build_bvh_packed(particles)
        self._mark("build")
        sec = self.tracer.tracer_wrapper.trace(self.frame, self._identity, sec_o, sec_d, particles, sph, 0, self.sph_degree, self.min_transmittance)
        self._mark("secondary")
        rgb = hybrid_composite(rgba, sec[0], hit, self.reflectivity, out=buf["rgb"])
        return pose, rgba, dst, vis_p, sec, (sec_o, sec_d, hit), rgb

    @torch.no_grad()
    def render(self, rays_o, rays_d, sensor, T_to_world):
        """Forward only: (hybrid rgb [H,W,3], primary rgba [H,W,4], secondary rgb [1,H,W,3], hit [H*W]).  The build it needs does not
        advance the step's BVH cadence."""
        particles, sph = self.activated()
        _, rgba, _, _, sec, (_, _, hit), rgb = self._forward(rays_o, rays_d, sensor, T_to_world, particles, sph, train=False)
        return rgb, rgba, sec[0], hit

    def _image_loss(self, pred, target, lambda_l1, lambda_ssim, background, mask):
        rgb, rgba, zero1 = pred
        alpha = rgba[..., 3:].contiguous() if (background is not None or mask is not None) else None
        return GaussianTrainStepGRT._image_loss(self, (rgb, alpha, zero1), target, lambda_l1, lambda_ssim, background, mask)

    @torch.no_grad()
    def step(self, rays_o, rays_d, sensor, T_to_world, target_rgb, all_sensor_positions=None, mask=None):
        """One optimisation step on this rank's view.  rays_o / rays_d: [1,H,W,3] camera space; sensor: the 3DGUT camera model;
        T_to_world: [1,4,4] camera-to-world (host); target_rgb: [H,W,3].  all_sensor_positions: [world,3] sensor positions of every rank's
        view of this step in rank order (omit on a single GPU; only the densifier reads this rank's own).  mask: optional [H,W] ([H,W,1],
        [1,H,W,1]) float CUDA tensor that multiplies prediction and target before the loss.  Returns this view's loss (a device scalar), the
        regularisers included."""
        H, W = int(rays_o.shape[1]), int(rays_o.shape[2])
        if mask is not None:
            mask = losses.mask_hw(mask, H, W)
        particles, sph = self.activated()
        pose, rgba, dst, vis_p, (srgb, salpha, sdst, snrm, _, vis_s), (sec_o, sec_d, hit), rgb = self._forward(
            rays_o, rays_d, sensor, T_to_world, particles, sph, train=True)
        buf = self._scratch(H, W)
        zero1, zero3 = self._zero_grads(H, W)
        loss, (d_rgb, d_alpha) = self._loss((rgb, rgba, zero1), rgb, target_rgb.reshape(H, W, 3), H, W, mask)
        self._mark("loss")
        d_rgba, d_sec = hybrid_composite_bwd(rgba, srgb, hit, self.reflectivity, d_rgb, None if d_alpha is zero1 else d_alpha, out=buf["grads"])
        self.raster.trace_bwd(self.frame, self.sph_degree, particles, sph, rays_o, rays_d, None, sensor, 0, 1, pose, pose, rgba, d_rgba, dst,
                              buf["zero_dist"], out=self.exchange.out())
        self._mark("backward_primary")
        self.tracer.tracer_wrapper.trace_bwd(self.frame, self._identity, sec_o, sec_d, srgb, salpha, sdst, snrm, particles, sph, d_sec, zero1,
                                             zero1, zero3, 0, self.sph_degree, self.min_transmittance, out=self.exchange.out(), accumulate=True)
        self._mark("backward_secondary")
        vis = torch.maximum(vis_p, vis_s) if self.optimizer.selective else vis_p
        my_position = self.raster.sensor_position(sensor, pose, pose, W, H) if self.densifier is not None else None
        return self._update(loss, particles, vis, all_sensor_positions, my_position)

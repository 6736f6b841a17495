"""Host-side mirror of the reference's 3DGRT tracer surface, backed by our LBVH ray tracer (csrc/grt.cu).

Same names, argument meaning and tensor contracts as the reference:
  Tracer / Tracer._Autograd / build_acc / render        threedgrt_tracer/tracer.py:50-255
  OptixTracer{trace, trace_bwd, build_bvh}              threedgrt_tracer/bindings.cpp:32-38, include/3dgrt/optixTracer.h:128-177
The class keeps the name OptixTracer for drop-in compatibility; there is no OptiX here (the traversal runs on the SMs).
"""
from __future__ import annotations

from enum import IntEnum

import numpy as np
import torch

import b200_native as native
from b200_native import NHT_FEATURE_DIM, cfg_get, ptr

# render.pipeline_type / backward_pipeline_type of each feature kind: the reference's CUDA programs trace SH radiance
# (referenceOptix.cu / referenceBwdOptix.cu), its Slang programs NHT features (referenceSlangOptix.cu / referenceSlangBwdOptix.cu)
SH_PIPELINES = ("reference", "referenceBwd")
NHT_PIPELINES = ("referenceSlang", "referenceSlangBwd")


def _check_pipelines(pipeline, backward_pipeline, nht: bool, enable_normals: bool):
    """Refuse, with NotImplementedError naming the key, every pairing this tracer does not build: SH radiance goes with the reference /
    referenceBwd pipelines, NHT features with referenceSlang / referenceSlangBwd; normals with SH radiance only.  Needs no GPU."""
    want, kind = (NHT_PIPELINES, "NHT features (model.feature_type: nht)") if nht else (SH_PIPELINES, "SH radiance (model.feature_type: sh)")
    if str(pipeline) != want[0]:
        raise NotImplementedError(f"render.pipeline_type={pipeline!r}: {kind} are traced through {want[0]!r} only")
    if str(backward_pipeline) != want[1]:
        raise NotImplementedError(f"render.backward_pipeline_type={backward_pipeline!r}: {kind} are differentiated through {want[1]!r} only")
    if enable_normals and nht:
        raise NotImplementedError("render.enable_normals=True: normals are built for SH radiance (reference pipeline) only")


def _nht_config(conf):
    """model.feature_type -> None (SH radiance) or {"half": render.particle_feature_half} for NHT features, after refusing the pairings
    and NHT settings that are not built (b200_native.nht_feature_config, shared with the 3DGUT tracer).  Pure config logic: needs no GPU."""
    nht = native.nht_feature_config(conf, "3DGRT")
    _check_pipelines(cfg_get(conf, "render.pipeline_type", "reference"), cfg_get(conf, "render.backward_pipeline_type", "referenceBwd"),
                     nht is not None, bool(cfg_get(conf, "render.enable_normals", False)))
    return nht


class OptixTracer:
    """Python twin of lib3dgrt_cc.OptixTracer (bindings.cpp:32-38); constructor arguments as optixTracer.h:128-141."""

    def __init__(self, path=None, cuda_path=None, pipeline="reference", backward_pipeline="referenceBwd", primitive="instances",
                 particle_kernel_degree=4, particle_kernel_min_response=0.0113, particle_kernel_max_alpha=0.99,
                 particle_kernel_density_clamping=True, particle_radiance_sph_degree=3, enable_normals=False, enable_hitcounts=True, nht=None):
        """nht (ours): None for SH radiance, or the NHT settings of _nht_config ({"half": ...}) to trace NHT features."""
        if not torch.cuda.is_available():
            raise RuntimeError("threedgrt_tracer: CUDA device required; there is no CPU path")
        _check_pipelines(pipeline, backward_pipeline, nht is not None, enable_normals)
        if primitive not in native.GRT_PRIMITIVES:
            raise NotImplementedError(f"primitive_type {primitive!r} is not built; built proxies: {', '.join(native.GRT_PRIMITIVES)}")
        if nht is None and int(particle_radiance_sph_degree) != 3:
            raise NotImplementedError("this build stores 16 SH coefficients per particle")
        self._nht = nht
        self._normals = bool(enable_normals)
        # kind-dependent parts of trace / trace_bwd, resolved once: ray-feature channels, how the per-particle features are handed to the
        # kernels, and the native forward / backward with the arguments that select the kind (SH degree, or the NHT row layout)
        if nht is None:
            self._out_channels, self._features = 3, torch.Tensor.contiguous
            self._native_trace = native.GrtContext.trace
            self._native_trace_bwd = lambda ctx, *args, accumulate: ctx.trace_bwd(*args, accumulate=accumulate)
            self._kind_args = lambda sph_degree: (int(sph_degree),)
        else:
            self._out_channels, self._features = NHT_FEATURE_DIM // 2, self._nht_features
            self._native_trace = native.GrtContext.trace_nht
            self._native_trace_bwd = lambda ctx, *args, accumulate: ctx.trace_bwd_nht(*args)  # accumulate=True is refused for NHT
            self._kind_args = lambda sph_degree: (NHT_FEATURE_DIM, int(nht["half"]))
        cfg = native.grt_default_config()
        cfg.kernel_degree = int(particle_kernel_degree)
        cfg.min_response = float(particle_kernel_min_response)
        cfg.max_alpha = float(particle_kernel_max_alpha)
        cfg.density_clamping = int(bool(particle_kernel_density_clamping))
        cfg.primitive = native.GRT_PRIMITIVES[primitive]
        self._cfg = cfg
        self._ctx = {}

    def _context(self, device) -> native.GrtContext:
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if idx not in self._ctx:
            self._ctx[idx] = native.GrtContext(self._cfg, idx)
        return self._ctx[idx]

    def build_bvh(self, mog_pos, mog_rot, mog_scl, mog_dns, rebuild=True, allow_update=False):
        """optixTracer.cpp:616-890"""
        dev = mog_pos.device
        pos, rot, scl, dns = (t.detach().contiguous().float() for t in (mog_pos, mog_rot, mog_scl, mog_dns))
        self._keep = (pos, rot, scl, dns)  # keep alive until the stream has consumed them
        stream = torch.cuda.current_stream(dev).cuda_stream
        self._context(dev).build_bvh(stream, int(pos.shape[0]), ptr(pos), ptr(rot), ptr(scl), ptr(dns), rebuild, allow_update)

    def build_bvh_packed(self, particles):
        """The same build from the [N,12] particle record that `trace` reads (grtb200_build_bvh_packed; no reference twin): bit-identical
        to build_bvh on the record's columns, without copying them out.  Every call is a full rebuild."""
        particles = particles.detach()
        if not (particles.is_cuda and particles.dtype == torch.float32 and particles.is_contiguous() and particles.dim() == 2
                and particles.shape[1] == 12):
            raise RuntimeError("particles: expected a contiguous float32 CUDA tensor [N,12]")
        self._keep = (particles,)  # keep alive until the stream has consumed it
        dev = particles.device
        self._context(dev).build_bvh_packed(torch.cuda.current_stream(dev).cuda_stream, int(particles.shape[0]), ptr(particles))

    @staticmethod
    def _r2w(ray_to_world) -> np.ndarray:
        m = ray_to_world.detach().cpu().numpy().reshape(-1, 4, 4)[0][:3, :4]  # first pose, 3 rows (optixTracer.cpp:931)
        return np.ascontiguousarray(m, dtype=np.float32)

    def _nht_features(self, features: torch.Tensor) -> torch.Tensor:
        """[N,48] features as the kernels read them: rounded to fp16 under render.particle_feature_half (optixTracer.cpp's
        particleFeatures of TParticleFeatureElem)"""
        if features.shape[-1] != NHT_FEATURE_DIM or not features.is_cuda:
            raise RuntimeError(f"trace: NHT features must be a [N,{NHT_FEATURE_DIM}] CUDA tensor, got {tuple(features.shape)}")
        return features.detach().to(torch.float16 if self._nht["half"] else torch.float32).contiguous()

    def trace(self, frame_id, ray_to_world, ray_ori, ray_dir, particle_density, particle_features, render_opts, sph_degree, min_transmittance,
              normals=None):
        """optixTracer.cpp:893-960 -> (feat [B,H,W,3], alpha [B,H,W,1], hit [B,H,W,2], normals [B,H,W,3], hits [B,H,W,1], vis [N,1]);
        with NHT features feat is [B,H,W,24] and particle_features the [N,48] features.  normals (ours): None follows enable_normals;
        False skips them for one call (a training step whose loss never reads them).  With normals the [B,H,W,3] tensor holds each ray's
        unnormalised normal sum (grtb200_trace_normals), otherwise zeros; every other output is the same either way."""
        dev = ray_ori.device
        b, h, w = (int(v) for v in ray_ori.shape[:3])
        n = int(particle_density.shape[0])
        particle_density, particle_features = particle_density.contiguous(), self._features(particle_features)
        ray_ori, ray_dir = ray_ori.contiguous(), ray_dir.contiguous()
        opts = dict(dtype=torch.float32, device=dev)
        feat, alpha = torch.empty((b, h, w, self._out_channels), **opts), torch.empty((b, h, w, 1), **opts)
        hit, hits = torch.empty((b, h, w, 2), **opts), torch.empty((b, h, w, 1), **opts)
        with_normals = self._normals if normals is None else bool(normals) and self._normals
        nrm = (torch.empty if with_normals else torch.zeros)((b, h, w, 3), **opts)  # the normals forward writes every ray
        vis = torch.empty((max(n, 1), 1), **opts)
        r2w = self._r2w(ray_to_world)
        stream = torch.cuda.current_stream(dev).cuda_stream
        args = (self._context(dev), stream, n, ptr(particle_density), ptr(particle_features), *self._kind_args(sph_degree), float(min_transmittance),
                b, h, w, ptr(ray_ori), ptr(ray_dir), r2w.ctypes.data, ptr(feat), ptr(alpha), ptr(hit), ptr(hits), ptr(vis))
        if with_normals:
            native.GrtContext.trace_normals(*args, ptr(nrm))
        else:
            self._native_trace(*args)
        return feat, alpha, hit, nrm, hits, vis[:n]

    def set_replay(self, enable, device):
        """Measurement-free switch (no reference twin): record the forward's hit lists for the backward (grtb200_set_replay)."""
        if getattr(self, "_replay", None) != bool(enable):
            self._context(device).set_replay(bool(enable))
            self._replay = bool(enable)

    def trace_counters(self, ray_to_world, ray_ori, ray_dir, particle_density, particle_features, sph_degree, min_transmittance):
        """Measurement helper (no reference twin): work counters of one forward trace -- rays, k-nearest queries, node visits, box / proxy
        tests, candidate and accepted hits (grtb200_debug_trace_counters); writes no image."""
        dev = ray_ori.device
        b, h, w = (int(v) for v in ray_ori.shape[:3])
        n = int(particle_density.shape[0])
        particle_density, particle_features = particle_density.contiguous(), particle_features.contiguous()
        ray_ori, ray_dir = ray_ori.contiguous(), ray_dir.contiguous()
        vis = torch.empty((max(n, 1), 1), dtype=torch.float32, device=dev)
        r2w = self._r2w(ray_to_world)
        stream = torch.cuda.current_stream(dev).cuda_stream
        return self._context(dev).trace_counters(stream, n, ptr(particle_density), ptr(particle_features), int(sph_degree), float(min_transmittance),
                                                 b, h, w, ptr(ray_ori), ptr(ray_dir), r2w.ctypes.data, ptr(vis))

    def trace_bwd(self, frame_id, ray_to_world, ray_ori, ray_dir, ray_features, ray_density, ray_hit_distance, ray_normals, particle_density,
                  particle_features, ray_features_grd, ray_density_grd, ray_hit_distance_grd, ray_normals_grd, render_opts, sph_degree,
                  min_transmittance, out=None, accumulate=False):
        """optixTracer.cpp:962-1031 -> (dDensity [N,12], dFeatures [N,48]).  out=(d_particles [N,12], d_sph [N,48]): contiguous float32
        tensors to write the gradients into (e.g. views of a flat exchange buffer); they are zeroed first and returned.  accumulate=True
        (SH radiance, with `out`): this trace's gradients are added to what `out` holds instead (grtb200_trace_bwd_accumulate), so that
        two passes can write one buffer.  With NHT features dFeatures is the fp32 [N,48] feature gradient, and `out` is taken the same way.
        The reference's Slang backward reads the forward's features rounded to fp16 under render.feature_output_half; this one reads
        them as the forward wrote them, in fp32 (feature_output_half is not applied, DESIGN.md section 13).  ray_normals and
        ray_normals_grd are accepted and ignored: the normals get no gradient, as in the reference, whose backward (referenceBwdOptix.cu)
        never reads them (DESIGN.md section 17); a forward with normals is replayed as one without."""
        if accumulate and (out is None or self._nht is not None):
            raise NotImplementedError("trace_bwd(accumulate=True) adds SH radiance gradients into a given `out` pair")
        dev = ray_ori.device
        b, h, w = (int(v) for v in ray_ori.shape[:3])
        n = int(particle_density.shape[0])
        particle_density, particle_features = particle_density.contiguous(), self._features(particle_features)
        ray_ori, ray_dir = ray_ori.contiguous(), ray_dir.contiguous()
        rf, rd_, rh = ray_features.contiguous(), ray_density.contiguous(), ray_hit_distance.contiguous()
        g_f, g_a = ray_features_grd.contiguous().float(), ray_density_grd.contiguous().float()
        g_d = ray_hit_distance_grd.contiguous().float()
        if g_d.shape[-1] != 1:
            g_d = g_d[..., 0:1].contiguous()
        d_density, d_features = self._grad_out(out, n, dev)
        r2w = self._r2w(ray_to_world)
        stream = torch.cuda.current_stream(dev).cuda_stream
        self._native_trace_bwd(self._context(dev), stream, n, ptr(particle_density), ptr(particle_features), *self._kind_args(sph_degree),
                               float(min_transmittance), b, h, w, ptr(ray_ori), ptr(ray_dir), r2w.ctypes.data, ptr(rf), ptr(rd_), ptr(rh),
                               ptr(g_f), ptr(g_a), ptr(g_d), ptr(d_density), ptr(d_features), accumulate=accumulate)
        return d_density[:n], d_features[:n]

    @staticmethod
    def _grad_out(out, n: int, dev):
        """The (d_particles [N,12], d_features [N,48]) pair trace_bwd writes: `out` checked, or two new tensors."""
        if out is None:
            return (torch.empty((max(n, 1), 12), dtype=torch.float32, device=dev),
                    torch.empty((max(n, 1), NHT_FEATURE_DIM), dtype=torch.float32, device=dev))
        d_density, d_features = out
        for t, name, k in ((d_density, "d_particles", 12), (d_features, "d_sph", NHT_FEATURE_DIM)):
            if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == (n, k)):
                raise RuntimeError(f"out: {name} must be a contiguous float32 CUDA tensor [{n},{k}]")
        return d_density, d_features

    def native_context(self, device=None) -> native.GrtContext:
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        return self._context(dev)


class Tracer:
    class _Autograd(torch.autograd.Function):
        """threedgrt_tracer/tracer.py:51-164"""

        @staticmethod
        def forward(ctx, tracer_wrapper, frame_id, ray_to_world, ray_ori, ray_dir, mog_pos, mog_rot, mog_scl, mog_dns, mog_sph, render_opts,
                    sph_degree, min_transmittance):
            particle_density = torch.concat([mog_pos, mog_dns, mog_rot, mog_scl, torch.zeros_like(mog_dns)], dim=1)
            ray_features, ray_density, ray_hit_distance, ray_normals, hits_count, mog_visibility = tracer_wrapper.trace(
                frame_id, ray_to_world, ray_ori, ray_dir, particle_density, mog_sph, render_opts, sph_degree, min_transmittance)
            ctx.save_for_backward(ray_to_world, ray_ori, ray_dir, ray_features, ray_density, ray_hit_distance, ray_normals, particle_density, mog_sph)
            ctx.frame_id, ctx.render_opts, ctx.sph_degree = frame_id, render_opts, sph_degree
            ctx.min_transmittance, ctx.tracer_wrapper = min_transmittance, tracer_wrapper
            return ray_features, ray_density, ray_hit_distance[:, :, :, 0:1], ray_normals, hits_count, mog_visibility

        @staticmethod
        def backward(ctx, ray_features_grd, ray_density_grd, ray_hit_distance_grd, ray_normals_grd, ray_hits_count_grd_UNUSED,
                     mog_visibility_grd_UNUSED):
            (ray_to_world, ray_ori, ray_dir, ray_features, ray_density, ray_hit_distance, ray_normals, particle_density, mog_sph) = ctx.saved_tensors
            particle_density_grd, mog_sph_grd = ctx.tracer_wrapper.trace_bwd(
                ctx.frame_id, ray_to_world, ray_ori, ray_dir, ray_features, ray_density, ray_hit_distance, ray_normals, particle_density, mog_sph,
                ray_features_grd, ray_density_grd, ray_hit_distance_grd, ray_normals_grd, ctx.render_opts, ctx.sph_degree, ctx.min_transmittance)
            mog_pos_grd, mog_dns_grd, mog_rot_grd, mog_scl_grd, _ = torch.split(particle_density_grd, [3, 1, 4, 3, 1], dim=1)
            return (None, None, None, None, None, mog_pos_grd, mog_rot_grd, mog_scl_grd, mog_dns_grd, mog_sph_grd, None, None, None)

    class RenderOpts(IntEnum):
        NONE = 0
        DEFAULT = NONE

    def __init__(self, conf):
        self.device = "cuda"
        self.conf = conf
        self.num_update_bvh = 0
        torch.zeros(1, device=self.device)
        g = lambda k, d: cfg_get(conf, "render." + k, d)  # noqa: E731
        nht = _nht_config(conf)  # None: SH radiance
        self.tracer_wrapper = OptixTracer(
            None, None, g("pipeline_type", "reference"), g("backward_pipeline_type", "referenceBwd"), g("primitive_type", "instances"),
            g("particle_kernel_degree", 4), g("particle_kernel_min_response", 0.0113), g("particle_kernel_max_alpha", 0.99),
            g("particle_kernel_density_clamping", True), g("particle_radiance_sph_degree", 3), g("enable_normals", False),
            g("enable_hitcounts", True), nht=nht)
        self._min_transmittance = float(g("min_transmittance", 0.001))
        self._clamping = bool(g("particle_kernel_density_clamping", True))
        self._max_updates = int(g("max_consecutive_bvh_update", 1))
        self._timings_on = bool(g("enable_kernel_timings", False))
        self.timings = {}

    def build_acc(self, gaussians, rebuild=True):
        """tracer.py:198-216"""
        allow_bvh_update = (self._max_updates > 1) and not self._clamping
        rebuild_bvh = rebuild or self._clamping or self.num_update_bvh >= self._max_updates
        self.tracer_wrapper.build_bvh(
            gaussians.positions.view(-1, 3).contiguous(), gaussians.rotation_activation(gaussians.rotation).view(-1, 4).contiguous(),
            gaussians.scale_activation(gaussians.scale).view(-1, 3).contiguous(),
            gaussians.density_activation(gaussians.density).view(-1, 1).contiguous(), rebuild_bvh, allow_bvh_update)
        self.num_update_bvh = 0 if rebuild_bvh else self.num_update_bvh + 1

    def render(self, gaussians, gpu_batch, train=False, frame_id=0):
        """tracer.py:218-255; with NHT features (model.feature_type: nht) pred_features is [B,H,W,24] and gaussians.get_features() the
        [N,48] features, which receive fp32 gradients."""
        start = end = None
        if self._timings_on:
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
        # hit lists for the backward's replay are only worth recording when a backward can follow
        self.tracer_wrapper.set_replay(bool(train) or torch.is_grad_enabled(), gpu_batch.rays_ori.device)
        pred_features, pred_opacity, pred_dist, pred_normals, hits_count, mog_visibility = Tracer._Autograd.apply(
            self.tracer_wrapper, frame_id, gpu_batch.T_to_world.contiguous(), gpu_batch.rays_ori.contiguous(), gpu_batch.rays_dir.contiguous(),
            gaussians.positions.contiguous(), gaussians.get_rotation().contiguous(), gaussians.get_scale().contiguous(),
            gaussians.get_density().contiguous(), gaussians.get_features().contiguous(), Tracer.RenderOpts.DEFAULT,
            gaussians.n_active_features, self._min_transmittance)
        frame_ms = 0.0
        if self._timings_on:
            end.record()
            end.synchronize()
            frame_ms = start.elapsed_time(end)
            self.timings["forward_render"] = frame_ms
        return {
            "pred_features": pred_features,
            "pred_opacity": pred_opacity,
            "pred_dist": pred_dist,
            "pred_normals": torch.nn.functional.normalize(pred_normals, dim=3),
            "hits_count": hits_count,
            "frame_time_ms": frame_ms,
            "mog_visibility": mog_visibility,
        }

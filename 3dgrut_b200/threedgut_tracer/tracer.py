"""Host-side mirror of the reference's 3DGUT tracer surface, backed by libgut_b200.so.

Same names, argument meaning and tensor contracts as the reference:
  Tracer / Tracer._Autograd            threedgut_tracer/tracer.py:158-349
  SplatRaster{trace,trace_bwd,collect_times}   threedgut_tracer/bindings.cpp:103-109, src/splatRaster.cpp:184-382
  fromOpenCVPinholeCameraModelParameters, fromOpenCVFisheyeCameraModelParameters, ShutterType   threedgut_tracer/bindings.cpp:34-101
PyTorch is used for device memory, streams and autograd only; every kernel is ours (csrc/*.cu).
"""
from __future__ import annotations

import enum
import math
import os
from dataclasses import dataclass

import numpy as np
import torch

import b200_native as native
from b200_native import NHT_FEATURE_DIM, cfg_get, ptr


class ShutterType(enum.IntEnum):  # bindings.cpp:36-42
    ROLLING_TOP_TO_BOTTOM = 0
    ROLLING_LEFT_TO_RIGHT = 1
    ROLLING_BOTTOM_TO_TOP = 2
    ROLLING_RIGHT_TO_LEFT = 3
    GLOBAL = 4


@dataclass
class CameraModelParameters:
    resolution: np.ndarray
    shutter_type: ShutterType
    principal_point: np.ndarray
    focal_length: np.ndarray
    radial_coeffs: np.ndarray
    tangential_coeffs: np.ndarray
    thin_prism_coeffs: np.ndarray
    model: int = 0          # CameraModelParameters::ModelType: 0 OpenCVPinholeModel, 1 OpenCVFisheyeModel, 2 FThetaModel
    max_angle: float = 0.0  # fisheye / f-theta
    ftheta: dict | None = None  # f-theta: reference_poly (0 / 1), bw [6], fw [6], cde [3]


class PolynomialType(enum.IntEnum):  # bindings.cpp:44-48
    PIXELDIST_TO_ANGLE = 0
    ANGLE_TO_PIXELDIST = 1


def fromFThetaCameraModelParameters(resolution, shutter_type, principal_point, reference_poly, pixeldist_to_angle_poly, angle_to_pixeldist_poly,
                                    max_angle, linear_cde) -> CameraModelParameters:
    """bindings.cpp:86-101: f-theta camera (polynomials of 6 coefficients, linear term [c d; e 1])"""
    f32 = lambda a, n: np.asarray(a, dtype=np.float32).reshape(n)  # noqa: E731
    ft = dict(reference_poly=int(PolynomialType(reference_poly)), bw=f32(pixeldist_to_angle_poly, 6), fw=f32(angle_to_pixeldist_poly, 6),
              cde=f32(linear_cde, 3))
    return CameraModelParameters(np.asarray(resolution, dtype=np.int64).reshape(2), ShutterType(shutter_type), f32(principal_point, 2),
                                 np.ones(2, np.float32), np.zeros(6, np.float32), np.zeros(2, np.float32), np.zeros(4, np.float32), model=2,
                                 max_angle=float(max_angle), ftheta=ft)


def fromOpenCVFisheyeCameraModelParameters(resolution, shutter_type, principal_point, focal_length, radial_coeffs, max_angle) -> CameraModelParameters:
    """bindings.cpp:68-84: OpenCV fisheye (equidistant + 4 radial coefficients, valid cone max_angle)"""
    f32 = lambda a, n: np.asarray(a, dtype=np.float32).reshape(n)  # noqa: E731
    radial6 = np.zeros(6, np.float32)
    radial6[:4] = f32(radial_coeffs, 4)
    return CameraModelParameters(np.asarray(resolution, dtype=np.int64).reshape(2), ShutterType(shutter_type), f32(principal_point, 2),
                                 f32(focal_length, 2), radial6, np.zeros(2, np.float32), np.zeros(4, np.float32), model=1,
                                 max_angle=float(max_angle))


def fromOpenCVPinholeCameraModelParameters(resolution, shutter_type, principal_point, focal_length, radial_coeffs,
                                            tangential_coeffs, thin_prism_coeffs) -> CameraModelParameters:
    """bindings.cpp:50-66"""
    f32 = lambda a, n: np.asarray(a, dtype=np.float32).reshape(n)  # noqa: E731
    return CameraModelParameters(np.asarray(resolution, dtype=np.int64).reshape(2), ShutterType(shutter_type), f32(principal_point, 2),
                                 f32(focal_length, 2), f32(radial_coeffs, 6), f32(tangential_coeffs, 2), f32(thin_prism_coeffs, 4))


@dataclass
class SensorPose3D:  # tracer.py:55-58
    T_world_sensors: list  # two [t.xyz, q.xyzw] world->sensor poses (shutter open / close)
    timestamps_us: list


def _so3_matrix_to_quat_xyzw(R: np.ndarray) -> np.ndarray:
    """tracer.py:88-136, evaluated in float32 like the reference's torch code (it receives a float32 matrix)."""
    R = np.asarray(R, dtype=np.float32)
    f = np.float32
    d = np.array([R[0, 0], R[1, 1], R[2, 2], f(f(R[0, 0] + R[1, 1]) + R[2, 2])], dtype=np.float32)
    c = int(np.argmax(d))
    q = np.zeros(4, dtype=np.float32)
    if c != 3:
        i, j, k = c, (c + 1) % 3, (c + 2) % 3
        q[i] = f(f(f(1) - d[3]) + f(f(2) * R[i, i]))
        q[j] = R[j, i] + R[i, j]
        q[k] = R[k, i] + R[i, k]
        q[3] = R[k, j] - R[j, k]
    else:
        q[0] = R[2, 1] - R[1, 2]
        q[1] = R[0, 2] - R[2, 0]
        q[2] = R[1, 0] - R[0, 1]
        q[3] = f(1) + d[3]
    return (q / np.sqrt(np.sum(q * q, dtype=np.float32), dtype=np.float32)).astype(np.float32)


def _native_config(conf) -> native.Config:
    """Config -> what the reference bakes in as -D constants (setup_3dgut.py:64-95)."""
    cfg = native.default_config()
    cfg.kernel_degree = int(cfg_get(conf, "render.particle_kernel_degree", 2))
    cfg.min_kernel_density = float(cfg_get(conf, "render.particle_kernel_min_response", 0.0113))
    cfg.min_alpha = float(cfg_get(conf, "render.particle_kernel_min_alpha", 1.0 / 255.0))
    cfg.max_alpha = float(cfg_get(conf, "render.particle_kernel_max_alpha", 0.99))
    cfg.min_transmittance = float(cfg_get(conf, "render.min_transmittance", 0.0001))
    a = float(cfg_get(conf, "render.splat.ut_alpha", 1.0))
    k = float(cfg_get(conf, "render.splat.ut_kappa", 0.0))
    cfg.ut_alpha, cfg.ut_beta, cfg.ut_kappa = a, float(cfg_get(conf, "render.splat.ut_beta", 2.0)), k
    cfg.ut_delta = math.sqrt(a * a * (3 + k))
    cfg.ut_margin = float(cfg_get(conf, "render.splat.ut_in_image_margin_factor", 0.1))
    cfg.rect_bounding = int(bool(cfg_get(conf, "render.splat.rect_bounding", True)))
    cfg.tight_opacity_bounding = int(bool(cfg_get(conf, "render.splat.tight_opacity_bounding", True)))
    cfg.tile_culling = int(bool(cfg_get(conf, "render.splat.tile_based_culling", True)))
    cfg.global_z_order = int(bool(cfg_get(conf, "render.splat.global_z_order", True)))
    cfg.enable_timings = int(bool(cfg_get(conf, "render.enable_kernel_timings", False)))
    cfg.n_rolling_shutter_iterations = int(cfg_get(conf, "render.splat.n_rolling_shutter_iterations", 5))
    cfg.k_buffer_size = int(cfg_get(conf, "render.splat.k_buffer_size", 0))
    if not (0 <= cfg.k_buffer_size <= 16):
        raise NotImplementedError("k_buffer_size must be within 0..16 (configs/paper/3dgut/sorted_*.yaml use 16)")
    if int(cfg_get(conf, "render.particle_radiance_sph_degree", 3)) != 3:
        raise NotImplementedError("this build stores 16 SH coefficients per particle (particle_radiance_sph_degree=3)")
    return cfg


def _nht_config(conf):
    """model.feature_type -> None (SH radiance) or the NHT settings the kernels take: {"half": render.particle_feature_half}.
    The shipped NHT configuration only (b200_native.nht_feature_config, shared with the 3DGRT tracer), and not with the k-buffer;
    anything else raises NotImplementedError naming the key.  Pure config logic: needs no GPU."""
    nht = native.nht_feature_config(conf, "3DGUT")
    if nht is not None and int(cfg_get(conf, "render.splat.k_buffer_size", 0)) > 0:
        raise NotImplementedError("render.splat.k_buffer_size > 0: NHT features are not built with the k-buffer")
    return nht


def _c(t: torch.Tensor) -> torch.Tensor:
    """.contiguous() without the dispatcher round trip when the tensor already is (the host side of a 0.9 ms frame is on the critical path)"""
    return t if t.is_contiguous() else t.contiguous()


def _raw_stream(dev: torch.device) -> int:
    """cudaStream_t of torch's current stream on `dev` (what torch.cuda.current_stream(dev).cuda_stream returns, minus ~10 us of Python)"""
    return torch._C._cuda_getCurrentRawStream(dev.index if dev.index is not None else torch.cuda.current_device())


class SplatRaster:
    """Python twin of the pybind class lib3dgut_cc.SplatRaster (bindings.cpp:103-109)."""

    def __init__(self, conf):
        if not torch.cuda.is_available():
            raise RuntimeError("threedgut_tracer: CUDA device required; there is no CPU path")
        self._cfg = _native_config(conf)
        self._nht = _nht_config(conf)  # None: SH radiance
        # kind-dependent parts of trace / trace_bwd, resolved once: ray-feature channels (rgb | 24 NHT features, then alpha) and how the
        # per-particle radiance is handed to the kernels
        if self._nht is None:
            self._out_channels, self._radiance = 4, _c
        else:
            self._out_channels, self._radiance = NHT_FEATURE_DIM // 2 + 1, self._nht_features
        self._ctx = {}  # one native context per device, like one SplatRaster per process/GPU in the reference
        self._last_camera = None  # (sensor, pose_start, pose_end, w, h, native.Camera) of the latest call: trace_bwd re-uses trace's struct

    def _context(self, device: torch.device) -> native.Context:
        idx = device.index if device.index is not None else torch.cuda.current_device()
        if idx not in self._ctx:
            self._ctx[idx] = native.Context(self._cfg, idx)
        return self._ctx[idx]

    def _camera_cached(self, sensor, pose_start, pose_end, width: int, height: int) -> native.Camera:
        """_camera, re-used when the very same sensor / pose OBJECTS come back with the same values (trace -> trace_bwd of one frame); the
        tuple keeps them alive, so an `is` match cannot be a recycled id, and the value snapshot catches a pose array mutated in place in
        between.  (The C side rejects a backward whose camera differs from the forward's either way.)"""
        def snap(pose):  # host copy of a pose given as ndarray / sequence / tensor (the reference takes tensors and calls .cpu())
            return pose.detach().cpu().numpy().copy() if isinstance(pose, torch.Tensor) else np.array(pose, copy=True)
        ps, pe = snap(pose_start), snap(pose_end)
        last = self._last_camera
        if (last is not None and last[0] is sensor and last[1] is pose_start and last[2] is pose_end and last[3] == width and last[4] == height
                and np.array_equal(last[6], ps) and np.array_equal(last[7], pe)):
            return last[5]
        cam = self._camera(sensor, ps, pe, width, height)
        self._last_camera = (sensor, pose_start, pose_end, width, height, cam, ps, pe)
        return cam

    @staticmethod
    def _camera(sensor: CameraModelParameters, pose_start, pose_end, width: int, height: int) -> native.Camera:
        cam = native.Camera()
        cam.width, cam.height = int(width), int(height)
        cam.principal[:] = [float(v) for v in sensor.principal_point]
        cam.focal[:] = [float(v) for v in sensor.focal_length]
        cam.radial[:] = [float(v) for v in sensor.radial_coeffs]
        cam.tangential[:] = [float(v) for v in sensor.tangential_coeffs]
        cam.thin_prism[:] = [float(v) for v in sensor.thin_prism_coeffs]
        cam.pose_start[:] = [float(v) for v in pose_start]  # .cpu() as in toSensorState (splatRaster.cpp:108-116)
        cam.pose_end[:] = [float(v) for v in pose_end]
        shutter = ShutterType(getattr(sensor, "shutter_type", ShutterType.GLOBAL))
        cam.rolling_shutter = 0 if shutter == ShutterType.GLOBAL else int(shutter) + 1  # gutb200_camera.rolling_shutter
        cam.model = int(getattr(sensor, "model", 0))
        cam.max_angle = float(getattr(sensor, "max_angle", 0.0))
        ft = getattr(sensor, "ftheta", None)
        if ft is not None:
            cam.ftheta_reference_poly = int(ft["reference_poly"])
            cam.ftheta_bw[:] = [float(v) for v in ft["bw"]]
            cam.ftheta_fw[:] = [float(v) for v in ft["fw"]]
            cam.ftheta_cde[:] = [float(v) for v in ft["cde"]]
        return cam

    def trace(self, frame_id, n_active_features, particle_density, particle_radiance, ray_ori, ray_dir, ray_time, sensor_params,
              timestamp_start, timestamp_end, pose_start, pose_end):
        """splatRaster.cpp:184-262 -> (feat+alpha [H,W,4], dist [H,W,1], hits [H,W,1], visibility [N,1]); with NHT features
        (model.feature_type: nht) feat+alpha is [H,W,25] and particle_radiance the [N,48] features."""
        nht = self._nht
        dev = ray_ori.device
        h, w = int(ray_ori.shape[1]), int(ray_ori.shape[2])
        n = int(particle_density.shape[0])
        particle_density, particle_radiance = _c(particle_density), self._radiance(particle_radiance)
        ray_ori, ray_dir = _c(ray_ori), _c(ray_dir)
        # NHT features are checked (and rounded) by _nht_features; they may be fp16 here
        for t in ((particle_density, particle_radiance, ray_ori, ray_dir) if nht is None else (particle_density, ray_ori, ray_dir)):
            if t.dtype != torch.float32 or not t.is_cuda:
                raise RuntimeError("trace: tensors must be float32 CUDA tensors")
        out = torch.empty((h, w, self._out_channels), dtype=torch.float32, device=dev)
        dist = torch.empty((h, w, 1), dtype=torch.float32, device=dev)
        hits = torch.empty((h, w, 1), dtype=torch.float32, device=dev)
        vis = torch.empty((n, 1), dtype=torch.float32, device=dev)
        cam = self._camera_cached(sensor_params, pose_start, pose_end, w, h)
        stream, ctx = _raw_stream(dev), self._context(dev)
        if nht is None:
            ctx.forward(stream, cam, n, ptr(particle_density), ptr(particle_radiance), int(n_active_features), ptr(ray_ori), ptr(ray_dir),
                        ptr(out), ptr(dist), ptr(hits), ptr(vis))
        else:
            ctx.forward_nht(stream, cam, n, ptr(particle_density), ptr(particle_radiance), NHT_FEATURE_DIM, int(nht["half"]), ptr(ray_ori),
                            ptr(ray_dir), ptr(out), ptr(dist), ptr(hits), ptr(vis))
        return out, dist, hits, vis

    def trace_bwd(self, frame_id, n_active_features, particle_density, particle_radiance, ray_ori, ray_dir, ray_time, sensor_params,
                  timestamp_start, timestamp_end, pose_start, pose_end, ray_radiance_density, ray_radiance_density_grd,
                  ray_hit_distance, ray_hit_distance_grd, out=None):
        """splatRaster.cpp:264-350 -> (dDensity [N,12], dRadiance [N,48]).  `out` (extension): a pair of preallocated
        tensors to write into, e.g. two views of one flat buffer so that a single all-reduce covers both.  With NHT features dRadiance
        is the fp32 [N,48] feature gradient (and `out` the [N,12] and [N,48] pair)."""
        return self._backward("backward", n_active_features, particle_density, particle_radiance, ray_ori, ray_dir, sensor_params, pose_start,
                              pose_end, ray_radiance_density, ray_radiance_density_grd, ray_hit_distance, ray_hit_distance_grd, out)

    def _nht_features(self, features: torch.Tensor) -> torch.Tensor:
        """[N,48] features as the kernels read them: rounded to fp16 under render.particle_feature_half (splatRaster.cpp:90-98)"""
        if features.shape[-1] != NHT_FEATURE_DIM or not features.is_cuda:
            raise RuntimeError(f"trace: NHT features must be a [N,{NHT_FEATURE_DIM}] CUDA tensor, got {tuple(features.shape)}")
        return _c(features.to(torch.float16 if self._nht["half"] else torch.float32))

    def _backward(self, sh_call, n_active_features, particle_density, particle_radiance, ray_ori, ray_dir, sensor_params, pose_start, pose_end,
                  rgba, d_rgba, dist, d_dist, out):
        """trace_bwd (sh_call "backward") and trace_bwd_compact ("backward_compact", the SH compact backward whatever the feature type):
        the second output is the [N,48] SH or NHT feature gradient, or, compact, the [N,4] masked radiance gradient."""
        compact = sh_call == "backward_compact"
        nht = None if compact else self._nht
        dev = ray_ori.device
        h, w = int(ray_ori.shape[1]), int(ray_ori.shape[2])
        n = int(particle_density.shape[0])
        particle_density, ray_ori, ray_dir = _c(particle_density), _c(ray_ori), _c(ray_dir)
        particle_radiance = _c(particle_radiance) if nht is None else self._nht_features(particle_radiance)
        rgba, d_rgba = _c(rgba), _c(d_rgba).float()
        dist, d_dist = _c(dist), _c(d_dist).float()
        width = 4 if compact else 48
        if out is not None:
            d_density, d_radiance = out
            assert d_density.shape == (n, 12) and d_radiance.shape == (n, width) and d_density.is_contiguous() and d_radiance.is_contiguous()
        else:
            d_density = torch.empty((n, 12), dtype=torch.float32, device=dev)
            d_radiance = torch.empty((n, width), dtype=torch.float32, device=dev)
        cam = self._camera_cached(sensor_params, pose_start, pose_end, w, h)
        stream, ctx = _raw_stream(dev), self._context(dev)
        if nht is None:
            getattr(ctx, sh_call)(stream, cam, n, ptr(particle_density), ptr(particle_radiance), int(n_active_features), ptr(ray_ori),
                                  ptr(ray_dir), ptr(rgba), ptr(d_rgba), ptr(dist), ptr(d_dist), ptr(d_density), ptr(d_radiance))
        else:
            ctx.backward_nht(stream, cam, n, ptr(particle_density), ptr(particle_radiance), NHT_FEATURE_DIM, int(nht["half"]), ptr(ray_ori),
                             ptr(ray_dir), ptr(rgba), ptr(d_rgba), ptr(dist), ptr(d_dist), ptr(d_density), ptr(d_radiance))
        return d_density, d_radiance

    # ---- view-parallel extensions (no reference twin: the reference trains on one GPU) -----------------------------------------

    def trace_bwd_compact(self, frame_id, n_active_features, particle_density, particle_radiance, ray_ori, ray_dir, ray_time, sensor_params,
                          timestamp_start, timestamp_end, pose_start, pose_end, ray_radiance_density, ray_radiance_density_grd,
                          ray_hit_distance, ray_hit_distance_grd, out=None):
        """trace_bwd that returns (dDensity [N,12], g [N,4]): g is the masked dL/d(radiance) of each particle in this view, from
        which sph_grad_from_views rebuilds the [N,48] SH gradient of any set of views (16 instead of 192 bytes per particle to exchange)."""
        return self._backward("backward_compact", n_active_features, particle_density, particle_radiance, ray_ori, ray_dir, sensor_params, pose_start,
                              pose_end, ray_radiance_density, ray_radiance_density_grd, ray_hit_distance, ray_hit_distance_grd, out)

    def sensor_position(self, sensor_params, pose_start, pose_end, width, height):
        """World-space sensor position of a view exactly as the kernels compute it: float32 numpy [3]."""
        return native.camera_position(self._camera(sensor_params, pose_start, pose_end, int(width), int(height)))

    def sph_grad_from_views(self, n_active_features, particle_density, view_positions, g_all, out=None):
        """Sum over views of basis16(direction particle <- sensor_v) x g_v: the all-reduced [N,48] SH gradient.
        view_positions: [views,3] (numpy / sequence, host); g_all: [views,N,4] device tensor (e.g. the result of an all-gather)."""
        dev = particle_density.device
        n = int(particle_density.shape[0])
        particle_density = _c(particle_density)
        g_all = _c(g_all)
        assert g_all.dim() == 3 and g_all.shape[1] == n and g_all.shape[2] == 4
        d_radiance = out if out is not None else torch.empty((n, 48), dtype=torch.float32, device=dev)
        assert d_radiance.shape == (n, 48) and d_radiance.is_contiguous()
        stream = _raw_stream(dev)
        self._context(dev).sph_grad_from_views(stream, n, ptr(particle_density), int(n_active_features),
                                               np.asarray(view_positions, np.float32).reshape(-1, 3), ptr(g_all), ptr(d_radiance))
        return d_radiance

    def collect_times(self):
        """splatRaster.cpp:352-382: mean ms of the timers recorded since the last call"""
        out = {}
        for ctx in self._ctx.values():
            f, b = ctx.collect_times()
            if f > 0:
                out["forward_render"] = f
            if b > 0:
                out["backward_render"] = b
        return out

    def native_context(self, device=None) -> native.Context:
        dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        return self._context(dev)


class Tracer:
    class _Autograd(torch.autograd.Function):
        """tracer.py:159-286 (argument list and returned tensors are identical)"""

        @staticmethod
        def forward(ctx, tracer_wrapper, frame_id, n_active_features, ray_ori, ray_dir, mog_pos, mog_rot, mog_scl, mog_dns, mog_sph,
                    sensor_params, sensor_poses):
            particle_density = _c(torch.concat([mog_pos, mog_dns, mog_rot, mog_scl, torch.zeros_like(mog_dns)], dim=1))
            particle_features = _c(mog_sph)
            ray_features_density, ray_hit_distance, ray_hit_count, mog_visibility = tracer_wrapper.trace(
                frame_id, n_active_features, particle_density, particle_features, _c(ray_ori), _c(ray_dir), None,
                sensor_params, sensor_poses.timestamps_us[0], sensor_poses.timestamps_us[1], sensor_poses.T_world_sensors[0],
                sensor_poses.T_world_sensors[1])
            ctx.save_for_backward(ray_ori, ray_dir, ray_features_density, ray_hit_distance, particle_density, particle_features)
            ctx.frame_id = frame_id
            ctx.n_active_features = n_active_features
            ctx.sensor_params = sensor_params
            ctx.sensor_poses = sensor_poses
            ctx.tracer_wrapper = tracer_wrapper
            return ray_features_density, ray_hit_distance, ray_hit_count, mog_visibility

        @staticmethod
        def backward(ctx, ray_features_density_grd, ray_hit_distance_grd, ray_hit_count_grd_UNUSED, mog_visibility_grd_UNUSED):
            ray_ori, ray_dir, ray_features_density, ray_hit_distance, particle_density, particle_features = ctx.saved_tensors
            sensor_poses = ctx.sensor_poses
            particle_density_grd, particle_features_grd = ctx.tracer_wrapper.trace_bwd(
                ctx.frame_id, ctx.n_active_features, particle_density, particle_features, ray_ori, ray_dir, None, ctx.sensor_params,
                sensor_poses.timestamps_us[0], sensor_poses.timestamps_us[1], sensor_poses.T_world_sensors[0],
                sensor_poses.T_world_sensors[1], ray_features_density, ray_features_density_grd, ray_hit_distance, ray_hit_distance_grd)
            mog_pos_grd, mog_dns_grd, mog_rot_grd, mog_scl_grd, _ = torch.split(particle_density_grd, [3, 1, 4, 3, 1], dim=1)
            return (None, None, None, None, None, mog_pos_grd.contiguous(), mog_rot_grd.contiguous(), mog_scl_grd.contiguous(),
                    mog_dns_grd.contiguous(), particle_features_grd.contiguous(), None, None)

    def __init__(self, conf):
        self.device = "cuda"
        self.conf = conf
        torch.zeros(1, device=self.device)  # force the CUDA context, as the reference does (tracer.py:292)
        self.tracer_wrapper = SplatRaster(conf)

    @property
    def timings(self):
        return self.tracer_wrapper.collect_times()

    def build_acc(self, gaussians, rebuild=True):
        pass  # no-op for 3DGUT (tracer.py:301)

    def _constant_normals(self, like: torch.Tensor) -> torch.Tensor:
        """normalize(ones_like(pred_features), dim=3) (tracer.py:304-349 returns this constant as "pred_normals"): a function of shape /
        dtype / device only, so it is built once per shape instead of with four kernels per frame."""
        key = (tuple(like.shape), like.dtype, like.device)
        cached = getattr(self, "_normals_cache", None)
        if cached is None or cached[0] != key:
            cached = (key, torch.nn.functional.normalize(torch.ones_like(like), dim=3))
            self._normals_cache = cached
        return cached[1]

    def render(self, gaussians, gpu_batch, train=False, frame_id=0):
        """tracer.py:304-349"""
        rays_o, rays_d = gpu_batch.rays_ori, gpu_batch.rays_dir
        sensor, poses = Tracer._create_camera_parameters(gpu_batch)
        pred_features_alpha, pred_dist, hits_count, mog_visibility = Tracer._Autograd.apply(
            self.tracer_wrapper, frame_id, gaussians.n_active_features, _c(rays_o), _c(rays_d),
            _c(gaussians.positions), _c(gaussians.get_rotation()), _c(gaussians.get_scale()),
            _c(gaussians.get_density()), _c(gaussians.get_features()), sensor, poses)
        ray_feature_dim = getattr(gaussians, "ray_feature_dim", 3 if self.tracer_wrapper._nht is None else NHT_FEATURE_DIM // 2)
        pred_features = pred_features_alpha[..., :ray_feature_dim].unsqueeze(0).contiguous()
        pred_opacity = pred_features_alpha[..., ray_feature_dim:].unsqueeze(0).contiguous()
        timings = self.tracer_wrapper.collect_times()
        return {
            "pred_features": pred_features,
            "pred_opacity": pred_opacity,
            "pred_dist": _c(pred_dist.unsqueeze(0)),
            "pred_normals": self._constant_normals(pred_features),
            "hits_count": _c(hits_count.unsqueeze(0)),
            "frame_time_ms": timings["forward_render"] if "forward_render" in timings else 0.0,
            "mog_visibility": mog_visibility,
        }

    @staticmethod
    def _pose_from_c2w(pose) -> np.ndarray:
        """tracer.py:404-423 + 360-380: C2W -> world->sensor [t, q.xyzw]"""
        p = pose.detach().cpu().numpy() if isinstance(pose, torch.Tensor) else np.asarray(pose)
        C2W = np.concatenate((p[:3, :4].astype(np.float64), np.zeros((1, 4))))
        C2W[3, 3] = 1.0
        W2C = np.linalg.inv(C2W)
        return np.concatenate([W2C[:3, 3].astype(np.float32), _so3_matrix_to_quat_xyzw(np.float32(W2C[:3, :3]))]).astype(np.float32)

    @staticmethod
    def _create_camera_parameters(gpu_batch):
        """tracer.py:383-488 (pinhole branches; fisheye / f-theta are a later row of SURVEY 8f)"""
        if getattr(gpu_batch, "rays_in_world_space", False):
            pose_start = pose_end = np.array([0, 0, 0, 0, 0, 0, 1], dtype=np.float32)
        else:
            start = gpu_batch.T_to_world.squeeze()
            assert start.ndim == 2
            end_raw = getattr(gpu_batch, "T_to_world_end", None)
            pose_start = Tracer._pose_from_c2w(start)
            pose_end = pose_start.copy() if end_raw is None else Tracer._pose_from_c2w(end_raw.squeeze())
        poses = SensorPose3D(T_world_sensors=[pose_start, pose_end], timestamps_us=[0, 1])
        K = getattr(gpu_batch, "intrinsics", None)
        if K is not None:
            focalx, focaly, cx, cy = float(K[0]), float(K[1]), float(K[2]), float(K[3])
            orig_w, orig_h = int(2 * cx), int(2 * cy)
            fovx, fovy = 2 * math.atan(orig_w / (2 * focalx)), 2 * math.atan(orig_h / (2 * focaly))
            sensor = fromOpenCVPinholeCameraModelParameters(
                resolution=np.array([orig_w, orig_h], dtype=np.uint32), shutter_type=ShutterType.GLOBAL,
                principal_point=np.array([orig_w, orig_h], dtype=np.float32) / 2,
                focal_length=np.array([orig_w / (2.0 * math.tan(fovx * 0.5)), orig_h / (2.0 * math.tan(fovy * 0.5))], dtype=np.float32),
                radial_coeffs=np.zeros((6,), dtype=np.float32), tangential_coeffs=np.zeros((2,), dtype=np.float32),
                thin_prism_coeffs=np.zeros((4,), dtype=np.float32))
            return sensor, poses
        K = getattr(gpu_batch, "intrinsics_OpenCVPinholeCameraModelParameters", None)
        if K is not None:
            shutter = K["shutter_type"]
            shutter = ShutterType[shutter] if isinstance(shutter, str) else ShutterType(shutter)
            sensor = fromOpenCVPinholeCameraModelParameters(
                resolution=K["resolution"], shutter_type=shutter, principal_point=K["principal_point"], focal_length=K["focal_length"],
                radial_coeffs=K["radial_coeffs"], tangential_coeffs=K["tangential_coeffs"],
                thin_prism_coeffs=K.get("thin_prism_coeffs", np.zeros((4,), dtype=np.float32)))
            return sensor, poses
        K = getattr(gpu_batch, "intrinsics_OpenCVFisheyeCameraModelParameters", None)
        if K is not None:  # tracer.py:458-467
            shutter = K["shutter_type"]
            shutter = ShutterType[shutter] if isinstance(shutter, str) else ShutterType(shutter)
            sensor = fromOpenCVFisheyeCameraModelParameters(
                resolution=K["resolution"], shutter_type=shutter, principal_point=K["principal_point"], focal_length=K["focal_length"],
                radial_coeffs=K["radial_coeffs"], max_angle=K["max_angle"])
            return sensor, poses
        K = getattr(gpu_batch, "intrinsics_FThetaCameraModelParameters", None)
        if K is not None:  # tracer.py:469-485
            shutter = K["shutter_type"]
            shutter = ShutterType[shutter] if isinstance(shutter, str) else ShutterType(shutter)
            ref_poly = K["reference_poly"]
            ref_poly = PolynomialType[ref_poly] if isinstance(ref_poly, str) else PolynomialType(ref_poly)
            sensor = fromFThetaCameraModelParameters(
                resolution=K["resolution"], shutter_type=shutter, principal_point=K["principal_point"], reference_poly=ref_poly,
                pixeldist_to_angle_poly=K["pixeldist_to_angle_poly"], angle_to_pixeldist_poly=K["angle_to_pixeldist_poly"],
                max_angle=K["max_angle"], linear_cde=K["linear_cde"])
            return sensor, poses
        raise ValueError("Camera intrinsics unavailable or unsupported (OpenCV pinhole, OpenCV fisheye and f-theta models)")

"""ctypes binding of include/gut_b200.h, grt_b200.h and nht_b200.h (one shared library, libgut_b200.so).  There is NO CPU or PyTorch
fallback: if the CUDA extension cannot be built/loaded, or no GPU is present when a context is created, this raises."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libgut_b200.so")
_LIB = None


class Camera(C.Structure):
    """gutb200_camera"""

    _fields_ = [
        ("width", C.c_int32), ("height", C.c_int32),
        ("principal", C.c_float * 2), ("focal", C.c_float * 2),
        ("radial", C.c_float * 6), ("tangential", C.c_float * 2), ("thin_prism", C.c_float * 4),
        ("pose_start", C.c_float * 7), ("pose_end", C.c_float * 7),
        ("model", C.c_int32), ("max_angle", C.c_float),
        ("ftheta_reference_poly", C.c_int32), ("ftheta_bw", C.c_float * 6), ("ftheta_fw", C.c_float * 6), ("ftheta_cde", C.c_float * 3),
        ("rolling_shutter", C.c_int32),
    ]


class Config(C.Structure):
    """gutb200_config"""

    _fields_ = [
        ("kernel_degree", C.c_int32), ("min_kernel_density", C.c_float), ("min_alpha", C.c_float),
        ("max_alpha", C.c_float), ("min_transmittance", C.c_float),
        ("ut_alpha", C.c_float), ("ut_beta", C.c_float), ("ut_kappa", C.c_float), ("ut_delta", C.c_float),
        ("ut_margin", C.c_float),
        ("rect_bounding", C.c_int32), ("tight_opacity_bounding", C.c_int32), ("tile_culling", C.c_int32),
        ("global_z_order", C.c_int32), ("enable_timings", C.c_int32), ("n_rolling_shutter_iterations", C.c_int32),
        ("k_buffer_size", C.c_int32), ("subtile_culling", C.c_int32),
    ]


class GrtConfig(C.Structure):
    """grtb200_config"""

    _fields_ = [("kernel_degree", C.c_int32), ("min_response", C.c_float), ("min_alpha", C.c_float), ("max_alpha", C.c_float),
                ("density_clamping", C.c_int32), ("primitive", C.c_int32)]


# grtb200_config.primitive (render.primitive_type)
GRT_PRIMITIVES = {"instances": 0, "icosahedron": 1}


class NhtConfig(C.Structure):
    """nhtb200_config"""

    _fields_ = [("n_features", C.c_int32), ("sh_degree", C.c_int32), ("n_hidden_layers", C.c_int32), ("width", C.c_int32),
                ("output_activation", C.c_int32), ("sh_scale", C.c_float)]


# nhtb200_config.output_activation (FeatureDecoder output_activation)
NHT_ACTIVATIONS = {"None": 0, "ReLU": 1, "Sigmoid": 2}
NHT_UNSUPPORTED = 1

_vp, _i32, _i64, _f32, _int, _sz, _str = C.c_void_p, C.c_int32, C.c_int64, C.c_float, C.c_int, C.c_size_t, C.c_char_p
_cam, _vpp, _i64p, _f32p = C.POINTER(Camera), C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.POINTER(C.c_float)
_adam = [_vp, _i64, _vpp, _vpp, _vpp, _f32p, _f32, _f32, _f32, _i64, _i32, _vp, _vp, _vp]
_grt_trace = [_vp, _vp, _i64, _vp, _vp, _i32, _f32, _i32, _i32, _i32, _vp, _vp, _vp]  # ctx ... ray_to_world_host
_grt_trace_nht = [_vp, _vp, _i64, _vp, _vp, _i32, _i32, _f32, _i32, _i32, _i32, _vp, _vp, _vp]  # ctx ... ray_to_world_host (NHT features)
_nht = C.POINTER(NhtConfig)

# C function -> (restype, argtypes) for every function the three headers declare; load() applies it once.  None = void.
# tests/test_cabi_bindings.py checks each entry against its prototype, type for type.
SIGNATURES = {
    # include/gut_b200.h
    "gutb200_default_config": (None, [C.POINTER(Config)]),
    "gutb200_create": (_int, [C.POINTER(Config), _int, _vpp]),
    "gutb200_destroy": (None, [_vp]),
    "gutb200_last_error": (_str, [_vp]),
    "gutb200_version": (_str, []),
    "gutb200_forward": (_int, [_vp, _vp, _cam, _i64, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gutb200_backward": (_int, [_vp, _vp, _cam, _i64, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gutb200_forward_nht": (_int, [_vp, _vp, _cam, _i64, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gutb200_backward_nht": (_int, [_vp, _vp, _cam, _i64, _vp, _vp, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gutb200_backward_compact": (_int, [_vp, _vp, _cam, _i64, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gutb200_sph_grad_from_views": (_int, [_vp, _vp, _i64, _vp, _i32, _i32, _vp, _vp, _vp]),
    "gutb200_camera_position": (_int, [_cam, _vp]),
    "gutb200_selective_adam_update": (_int, [_vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _f32, _f32, _i64, _i64]),
    "gutb200_gaussian_adam_step": (_int, _adam),
    "gutb200_gaussian_adam_step_reg": (_int, _adam + [_f32, _f32]),
    "gutb200_nht_adam_step": (_int, [_vp, _i64, _i64, _vpp, _vpp, _vpp, _f32p, _i64p, _f32, _f32, _f32, _i32, _f32, _f32, _f32, _f32, _i32,
                                     _vp, _vp, _vp, _vp, _f32, _f32]),
    "gutb200_image_loss_scratch_bytes": (_sz, [_i32, _i32]),
    "gutb200_image_loss": (_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _vp, _vp, _vp, _vp, _i32]),
    "gutb200_image_metrics_scratch_bytes": (_sz, [_i32, _i32]),
    "gutb200_image_metrics": (_int, [_vp, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp]),
    "gutb200_hybrid_rays": (_int, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gutb200_hybrid_composite": (_int, [_vp, _i64, _vp, _vp, _vp, _f32, _vp]),
    "gutb200_hybrid_composite_bwd": (_int, [_vp, _i64, _vp, _vp, _vp, _f32, _vp, _vp, _vp, _vp]),
    "gutb200_knn_workspace_bytes": (_sz, [_i64]),
    "gutb200_knn": (_int, [_vp, _i64, _vp, _i64, _vp, _i32, _vp, _sz, _vp, _vp]),
    "gutb200_forward_host": (_int, [_vp, _cam, _i64, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gutb200_backward_host": (_int, [_vp, _cam, _i64, _vp, _vp, _i32, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "gutb200_last_stats": (_int, [_vp, _i64p, _i64p, _i64p, _i64p]),
    "gutb200_debug_copy": (_int, [_vp, _int, _vp, _sz]),
    "gutb200_collect_times": (_int, [_vp, _f32p, _f32p]),
    "gutb200_set_timings": (_int, [_vp, _int]),
    "gutb200_collect_stage_times": (_int, [_vp, _f32p]),
    "gutb200_debug_work_counters": (_int, [_vp, _vp, _vp, _vp, _vp]),
    "gutb200_debug_fma_peak": (_int, [_vp, _int, _f32p]),
    "gutb200_launch_count": (_i64, [_vp]),
    # include/grt_b200.h (3DGRT: LBVH build + ordered ray tracing)
    "grtb200_default_config": (None, [C.POINTER(GrtConfig)]),
    "grtb200_create": (_int, [C.POINTER(GrtConfig), _int, _vpp]),
    "grtb200_destroy": (None, [_vp]),
    "grtb200_last_error": (_str, [_vp]),
    "grtb200_build_bvh": (_int, [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _i32, _i32]),
    "grtb200_build_bvh_packed": (_int, [_vp, _vp, _i64, _vp]),
    "grtb200_trace": (_int, _grt_trace + [_vp, _vp, _vp, _vp, _vp]),
    "grtb200_trace_normals": (_int, _grt_trace + [_vp, _vp, _vp, _vp, _vp, _vp]),
    "grtb200_trace_bwd": (_int, _grt_trace + [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "grtb200_trace_bwd_accumulate": (_int, _grt_trace + [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "grtb200_trace_nht": (_int, _grt_trace_nht + [_vp, _vp, _vp, _vp, _vp]),
    "grtb200_trace_bwd_nht": (_int, _grt_trace_nht + [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "grtb200_scene_aabb": (_int, [_vp, _vp]),
    "grtb200_launch_count": (_i64, [_vp]),
    "grtb200_set_replay": (_int, [_vp, _i32]),
    "grtb200_debug_trace_counters": (_int, _grt_trace + [_vp, _vp]),
    "grtb200_mesh_create": (_int, [_int, _vpp]),
    "grtb200_mesh_destroy": (None, [_vp]),
    "grtb200_mesh_last_error": (_str, [_vp]),
    "grtb200_build_mesh_bvh": (_int, [_vp, _vp, _i64, _vp, _vp, _i64, _vp, _vp, _i32, _vp]),
    "grtb200_mesh_closest_hit": (_int, [_vp, _vp, _i64, _vp, _vp, _vp, _vp]),
    "grtb200_trace_playground": (_int, [_vp, _vp, _vp, _i64, _vp, _vp, _i32, _f32, _i32, _i32, _i32, _vp, _vp, _vp, _vp, _vp, _i32, _vp, _vp,
                                        _vp]),
    # include/nht_b200.h (NHT feature decoder: fused tensor-core MLP)
    "nhtb200_last_error": (_str, []),
    "nhtb200_n_params": (_i64, [_nht]),
    "nhtb200_backward_workspace_bytes": (_sz, [_nht, _i64]),
    "nhtb200_forward": (_int, [_nht, _vp, _i64, _vp, _vp, _vp, _vp]),
    "nhtb200_backward": (_int, [_nht, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
}
EXPORTS = [k for k in SIGNATURES if k.startswith("gutb200_")]
GRT_EXPORTS = [k for k in SIGNATURES if k.startswith("grtb200_")]
NHT_EXPORTS = [k for k in SIGNATURES if k.startswith("nhtb200_")]


def camera_position(cam):
    """Sensor position in world space as the kernels compute it (gutb200_camera_position): numpy float32 [3]."""
    import numpy as np

    out = np.zeros(3, np.float32)
    if load().gutb200_camera_position(C.byref(cam), out.ctypes.data) != 0:
        raise RuntimeError("gutb200_camera_position failed")
    return out


DBG_TILES_COUNT, DBG_SORTED_KEYS, DBG_SORTED_VALUES, DBG_TILE_RANGES, DBG_DEPTH, DBG_RGB, DBG_PROJ = range(7)


def lib_path() -> str:
    return _SO


def load():
    """Load (building in-tree if sources are newer) the sm_90a shared library, with every function of SIGNATURES bound."""
    global _LIB
    if _LIB is not None:
        return _LIB
    import build as _build  # 3dgrut_b200/build.py

    if _build.needs_build():
        _build.build()
    if not os.path.exists(_SO):
        raise RuntimeError(f"{_SO} is missing: the CUDA extension was not built (no fallback path exists)")
    lib = C.CDLL(_SO)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    _LIB = lib
    return lib


def cfg_get(conf, path, default):
    """conf's value at the dotted `path` (dict keys or attributes), `default` where it is missing or None."""
    cur = conf
    for key in path.split("."):
        if cur is None:
            return default
        cur = cur.get(key, None) if isinstance(cur, dict) else getattr(cur, key, None)
    return default if cur is None else cur


def ptr(t) -> int:
    return t.data_ptr()


def default_config() -> Config:
    cfg = Config()
    load().gutb200_default_config(C.byref(cfg))
    return cfg


class _Handle:
    """Owning wrapper of a `<PREFIX>_ctx*`: created by `<PREFIX>_create`, released by `close` (or garbage collection); `_check` raises
    with `<PREFIX>_last_error` for a non-zero return code."""

    PREFIX = ""

    def __init__(self, cfg, device: int = 0):
        self._lib = load()
        self._h = C.c_void_p()
        rc = getattr(self._lib, self.PREFIX + "_create")(C.byref(cfg), int(device), C.byref(self._h))
        self._check_create(rc, cfg)
        self.cfg = cfg

    def _check_create(self, rc: int, cfg):
        if rc != 0 or not self._h:
            raise RuntimeError(f"{self.PREFIX}_create failed (rc={rc}): a CUDA device is required, there is no CPU path")

    def close(self):
        if getattr(self, "_h", None):
            getattr(self._lib, self.PREFIX + "_destroy")(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int, what: str):
        if rc != 0:
            raise RuntimeError(f"{what} failed: {getattr(self._lib, self.PREFIX + '_last_error')(self._h).decode()}")


class Context(_Handle):
    """Owning wrapper of a gutb200_ctx*."""

    PREFIX = "gutb200"

    def forward(self, stream, cam, n, particles, sph, sph_degree, rays_o, rays_d, out_rgba, out_dist, out_hits, visibility):
        self._check(self._lib.gutb200_forward(self._h, stream, C.byref(cam), n, particles, sph, sph_degree, rays_o, rays_d,
                                              out_rgba, out_dist, out_hits, visibility), "gutb200_forward")

    def backward(self, stream, cam, n, particles, sph, sph_degree, rays_o, rays_d, out_rgba, d_rgba, out_dist, d_dist,
                 d_particles, d_sph):
        self._check(self._lib.gutb200_backward(self._h, stream, C.byref(cam), n, particles, sph, sph_degree, rays_o, rays_d,
                                               out_rgba, d_rgba, out_dist, d_dist, d_particles, d_sph), "gutb200_backward")

    def forward_nht(self, stream, cam, n, particles, features, feature_dim, features_half, rays_o, rays_d, out_features_alpha, out_dist,
                    out_hits, visibility):
        """NHT features instead of SH radiance: out_features_alpha [H,W,feature_dim/2 + 1] (gutb200_forward_nht)."""
        self._check(self._lib.gutb200_forward_nht(self._h, stream, C.byref(cam), n, particles, features, feature_dim, features_half, rays_o,
                                                  rays_d, out_features_alpha, out_dist, out_hits, visibility), "gutb200_forward_nht")

    def backward_nht(self, stream, cam, n, particles, features, feature_dim, features_half, rays_o, rays_d, out_features_alpha,
                     d_features_alpha, out_dist, d_dist, d_particles, d_features):
        """Adjoint of forward_nht: d_particles [N,12], d_features [N,feature_dim] fp32 (gutb200_backward_nht)."""
        self._check(self._lib.gutb200_backward_nht(self._h, stream, C.byref(cam), n, particles, features, feature_dim, features_half, rays_o,
                                                   rays_d, out_features_alpha, d_features_alpha, out_dist, d_dist, d_particles, d_features),
                    "gutb200_backward_nht")

    def backward_compact(self, stream, cam, n, particles, sph, sph_degree, rays_o, rays_d, out_rgba, d_rgba, out_dist, d_dist,
                         d_particles, d_radiance):
        """Like backward, but emits the [N,4] masked radiance gradient instead of the [N,48] SH gradient (view-parallel exchange)."""
        self._check(self._lib.gutb200_backward_compact(self._h, stream, C.byref(cam), n, particles, sph, sph_degree, rays_o, rays_d,
                                                       out_rgba, d_rgba, out_dist, d_dist, d_particles, d_radiance), "gutb200_backward_compact")

    def sph_grad_from_views(self, stream, n, particles, sph_degree, view_positions, d_radiance_all, d_sph):
        """view_positions: float32 numpy [views,3] (host); d_radiance_all: device [views,N,4]; d_sph: device [N,48]."""
        import numpy as np

        vp_ = np.ascontiguousarray(view_positions, dtype=np.float32)
        self._check(self._lib.gutb200_sph_grad_from_views(self._h, stream, n, particles, sph_degree, int(vp_.shape[0]), vp_.ctypes.data,
                                                          d_radiance_all, d_sph), "gutb200_sph_grad_from_views")

    def forward_host(self, cam, n, particles, sph, sph_degree, rays_o, rays_d, out_rgba, out_dist, out_hits, visibility):
        self._check(self._lib.gutb200_forward_host(self._h, C.byref(cam), n, particles, sph, sph_degree, rays_o, rays_d,
                                                   out_rgba, out_dist, out_hits, visibility), "gutb200_forward_host")

    def backward_host(self, cam, n, particles, sph, sph_degree, rays_o, rays_d, out_rgba, d_rgba, out_dist, d_dist,
                      d_particles, d_sph):
        self._check(self._lib.gutb200_backward_host(self._h, C.byref(cam), n, particles, sph, sph_degree, rays_o, rays_d,
                                                    out_rgba, d_rgba, out_dist, d_dist, d_particles, d_sph), "gutb200_backward_host")

    def stats(self):
        n, i, v, t = C.c_int64(), C.c_int64(), C.c_int64(), C.c_int64()
        self._check(self._lib.gutb200_last_stats(self._h, C.byref(n), C.byref(i), C.byref(v), C.byref(t)), "gutb200_last_stats")
        return {"N": n.value, "I": i.value, "V": v.value, "T": t.value}

    def debug_copy(self, what: int):
        import numpy as np

        st = self.stats()
        shape, dt = {
            DBG_TILES_COUNT: ((st["N"],), np.uint32), DBG_SORTED_KEYS: ((st["I"],), np.uint64),
            DBG_SORTED_VALUES: ((st["I"],), np.uint32), DBG_TILE_RANGES: ((st["T"], 2), np.uint32),
            DBG_DEPTH: ((st["N"],), np.float32), DBG_RGB: ((st["N"], 3), np.float32), DBG_PROJ: ((st["N"], 8), np.float32),
        }[what]
        out = np.zeros(shape, dt)
        self._check(self._lib.gutb200_debug_copy(self._h, what, out.ctypes.data, out.nbytes), "gutb200_debug_copy")
        return out

    def collect_times(self):
        f, b = C.c_float(), C.c_float()
        self._check(self._lib.gutb200_collect_times(self._h, C.byref(f), C.byref(b)), "gutb200_collect_times")
        return f.value, b.value

    STAGES = ("project", "scan", "expand", "sort", "tile_ranges", "render", "render_backward", "project_backward")

    def collect_stage_times(self):
        arr = (C.c_float * 8)()
        self._check(self._lib.gutb200_collect_stage_times(self._h, arr), "gutb200_collect_stage_times")
        return dict(zip(self.STAGES, [float(v) for v in arr]))

    def set_timings(self, level: int):
        self._check(self._lib.gutb200_set_timings(self._h, int(level)), "gutb200_set_timings")

    def launch_count(self) -> int:
        return int(self._lib.gutb200_launch_count(self._h))

    COUNTERS = ("tests_ref", "tests_exec", "hits", "fwd_iters", "hit_iters", "screens", "bwd_lanes", "iters16", "iters8", "sub16_hits", "sub8_hits")

    def work_counters(self, particles, rays_o, rays_d):
        """Work counters of the last forward (device pointers as passed to it): dict of ints (gutb200_debug_work_counters)."""
        arr = (C.c_uint64 * 16)()
        self._check(self._lib.gutb200_debug_work_counters(self._h, particles, rays_o, rays_d, arr), "gutb200_debug_work_counters")
        return dict(zip(self.COUNTERS, [int(v) for v in arr]))

    def fma_peak_tflops(self, repeats: int = 5) -> float:
        v = C.c_float()
        self._check(self._lib.gutb200_debug_fma_peak(self._h, int(repeats), C.byref(v)), "gutb200_debug_fma_peak")
        return float(v.value)


# ---------------------------------------------------------------------------------------------------------------
# include/grt_b200.h (3DGRT: LBVH build + ordered ray tracing), same shared library

NHT_FEATURE_DIM = 48  # model.nht_features.dim of the shipped NHT configs (configs/base_gs.yaml): 4 tetrahedron vertices x 12
_NHT_BUILT = (("model.nht_features.dim", NHT_FEATURE_DIM), ("model.nht_features.activation.type", "sincos"),
              ("model.nht_features.activation.num_frequencies", 1), ("model.nht_features.interpolation_type", "barycentric"))


def nht_feature_config(conf, tracer: str):
    """model.feature_type -> None (SH radiance) or the NHT settings both tracers take: {"half": render.particle_feature_half}.
    Only the reference's shipped NHT configuration is built (configs/base_gs.yaml: dim 48, barycentric, sincos with 1 frequency);
    anything else raises NotImplementedError naming the key.  Pure config logic: needs no GPU.  `tracer` names the caller in messages."""
    kind = str(cfg_get(conf, "model.feature_type", "sh")).lower()
    if kind == "sh":
        return None
    if kind != "nht":
        raise NotImplementedError(f"model.feature_type={kind!r}: the {tracer} tracer renders 'sh' or 'nht'")
    for key, want in _NHT_BUILT:
        got = cfg_get(conf, key, want)
        if (str(got).lower() if isinstance(want, str) else int(got)) != want:
            raise NotImplementedError(f"{key}={got!r}: NHT features are built for {key}={want!r} only")
    return {"half": bool(cfg_get(conf, "render.particle_feature_half", False))}


def grt_default_config() -> GrtConfig:
    cfg = GrtConfig()
    load().grtb200_default_config(C.byref(cfg))
    return cfg


class GrtContext(_Handle):
    """Owning wrapper of a grtb200_ctx*."""

    PREFIX = "grtb200"

    def _check_create(self, rc: int, cfg):
        if rc == 5:
            raise ValueError(f"grtb200_create: primitive {cfg.primitive} is not one of {GRT_PRIMITIVES}")
        super()._check_create(rc, cfg)

    def build_bvh(self, stream, n, pos, rot, scl, dns, rebuild=True, allow_update=False):
        self._check(self._lib.grtb200_build_bvh(self._h, stream, n, pos, rot, scl, dns, int(rebuild), int(allow_update)), "grtb200_build_bvh")

    def build_bvh_packed(self, stream, n, particles):
        """The same build from the [N,12] particle record that trace reads (grtb200_build_bvh_packed)."""
        self._check(self._lib.grtb200_build_bvh_packed(self._h, stream, n, particles), "grtb200_build_bvh_packed")

    def trace(self, stream, n, particles, sph, sph_degree, min_t, batch, height, width, rays_o, rays_d, r2w_host, out_rgb, out_alpha,
              out_dist, out_hits, visibility):
        self._check(self._lib.grtb200_trace(self._h, stream, n, particles, sph, sph_degree, min_t, batch, height, width, rays_o, rays_d,
                                            r2w_host, out_rgb, out_alpha, out_dist, out_hits, visibility), "grtb200_trace")

    def trace_normals(self, stream, n, particles, sph, sph_degree, min_t, batch, height, width, rays_o, rays_d, r2w_host, out_rgb, out_alpha,
                      out_dist, out_hits, visibility, out_normals):
        """trace that also writes the unnormalised ray normals out_normals [R,3] (grtb200_trace_normals); trace_bwd replays its hit lists
        as trace's, and the normals get no gradient."""
        self._check(self._lib.grtb200_trace_normals(self._h, stream, n, particles, sph, sph_degree, min_t, batch, height, width, rays_o,
                                                    rays_d, r2w_host, out_rgb, out_alpha, out_dist, out_hits, visibility, out_normals),
                    "grtb200_trace_normals")

    def trace_bwd(self, stream, n, particles, sph, sph_degree, min_t, batch, height, width, rays_o, rays_d, r2w_host, out_rgb, out_alpha,
                  out_dist, d_rgb, d_alpha, d_dist, d_particles, d_sph, accumulate=False):
        """accumulate: add to d_particles / d_sph instead of zeroing them first (grtb200_trace_bwd_accumulate)."""
        name = "grtb200_trace_bwd_accumulate" if accumulate else "grtb200_trace_bwd"
        self._check(getattr(self._lib, name)(self._h, stream, n, particles, sph, sph_degree, min_t, batch, height, width, rays_o, rays_d,
                                             r2w_host, out_rgb, out_alpha, out_dist, d_rgb, d_alpha, d_dist, d_particles, d_sph), name)

    def trace_nht(self, stream, n, particles, features, feature_dim, features_half, min_t, batch, height, width, rays_o, rays_d, r2w_host,
                  out_features, out_alpha, out_dist, out_hits, visibility):
        """NHT features instead of SH radiance: out_features [R,feature_dim/2] (grtb200_trace_nht)."""
        self._check(self._lib.grtb200_trace_nht(self._h, stream, n, particles, features, feature_dim, features_half, min_t, batch, height, width,
                                                rays_o, rays_d, r2w_host, out_features, out_alpha, out_dist, out_hits, visibility),
                    "grtb200_trace_nht")

    def trace_bwd_nht(self, stream, n, particles, features, feature_dim, features_half, min_t, batch, height, width, rays_o, rays_d, r2w_host,
                      out_features, out_alpha, out_dist, d_features_out, d_alpha, d_dist, d_particles, d_features):
        """Adjoint of trace_nht: d_particles [N,12], d_features [N,feature_dim] fp32 (grtb200_trace_bwd_nht)."""
        self._check(self._lib.grtb200_trace_bwd_nht(self._h, stream, n, particles, features, feature_dim, features_half, min_t, batch, height,
                                                    width, rays_o, rays_d, r2w_host, out_features, out_alpha, out_dist, d_features_out, d_alpha,
                                                    d_dist, d_particles, d_features), "grtb200_trace_bwd_nht")

    def scene_aabb(self):
        import numpy as np

        out = np.zeros(6, np.float32)
        self._check(self._lib.grtb200_scene_aabb(self._h, out.ctypes.data), "grtb200_scene_aabb")
        return out

    def set_replay(self, enable: bool):
        """Record hit lists in the forward for the backward's replay (default on); off frees the cache (inference-only rendering)."""
        self._check(self._lib.grtb200_set_replay(self._h, int(bool(enable))), "grtb200_set_replay")

    TRACE_COUNTERS = ("rays", "queries", "node_visits", "box_tests", "proxy_tests", "candidate_hits", "accepted_hits", "packet_rays")

    def trace_counters(self, stream, n, particles, sph, sph_degree, min_t, batch, height, width, rays_o, rays_d, r2w_host, visibility_scratch):
        """Work counters of one forward trace (debug; synchronises): dict of ints."""
        arr = (C.c_uint64 * 8)()
        self._check(self._lib.grtb200_debug_trace_counters(self._h, stream, n, particles, sph, sph_degree, min_t, batch, height, width, rays_o, rays_d,
                                                           r2w_host, visibility_scratch, arr), "grtb200_debug_trace_counters")
        return dict(zip(self.TRACE_COUNTERS, [int(v) for v in arr]))

    def launch_count(self) -> int:
        return int(self._lib.grtb200_launch_count(self._h))

    def trace_playground(self, stream, mesh, n, particles, sph, sph_degree, min_t, batch, height, width, rays_o, rays_d, r2w_host, ray_max_t,
                         background_host, smooth_normals, out_rgb, out_alpha, visibility):
        """Forward render with the meshes of `mesh` (a MeshBvh or None) inserted: out_rgb [R,3], out_alpha [R] (grtb200_trace_playground)."""
        self._check(self._lib.grtb200_trace_playground(self._h, stream, None if mesh is None else mesh._h, n, particles, sph, sph_degree, min_t,
                                                       batch, height, width, rays_o, rays_d, r2w_host, ray_max_t, background_host,
                                                       int(bool(smooth_normals)), out_rgb, out_alpha, visibility), "grtb200_trace_playground")


class MeshBvh(_Handle):
    """Owning wrapper of a grtb200_mesh*: the LBVH over the triangles of the playground meshes."""

    PREFIX = "grtb200_mesh"

    def __init__(self, device: int = 0):
        self._lib = load()
        self._h = C.c_void_p()
        self._check_create(self._lib.grtb200_mesh_create(int(device), C.byref(self._h)), None)

    def build(self, stream, n_vertices, vertices, vertex_normals, n_faces, faces, face_material, n_materials, materials):
        """(Re)build over device arrays: vertices / vertex_normals [V,3] fp32, faces [F,3] int32, face_material [F] int32, materials
        [M,8] fp32 (grtb200_build_mesh_bvh; synchronises the stream, copies everything)."""
        self._check(self._lib.grtb200_build_mesh_bvh(self._h, stream, n_vertices, vertices, vertex_normals, n_faces, faces, face_material,
                                                     n_materials, materials), "grtb200_build_mesh_bvh")

    def closest_hit(self, stream, n_rays, rays_o, rays_d, out_t, out_tri):
        """World rays [R,3] -> out_t [R] fp32 (1e5 where nothing is hit), out_tri [R] int32 (-1) (grtb200_mesh_closest_hit)."""
        self._check(self._lib.grtb200_mesh_closest_hit(self._h, stream, n_rays, rays_o, rays_d, out_t, out_tri), "grtb200_mesh_closest_hit")


# ---------------------------------------------------------------------------------------------------------------
# include/nht_b200.h (NHT feature decoder: fused tensor-core MLP), same shared library

nht_lib = load  # the feature decoder's name for the library; load() binds the nhtb200_* entries with the rest


def nht_check(rc: int, what: str):
    """Raise for a non-zero nhtb200_* return code: NotImplementedError for a configuration that is not built."""
    if rc == 0:
        return
    msg = f"{what}: {nht_lib().nhtb200_last_error().decode()}"
    if rc == NHT_UNSUPPORTED:
        raise NotImplementedError(msg)
    raise RuntimeError(msg)

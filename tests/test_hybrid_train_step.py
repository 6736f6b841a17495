"""Host logic of the 3DGRUT hybrid training step (train_step_hybrid), no GPU: the settings it refuses, the render defaults both tracers
read, the C5 workload and the entry points it adds to the C ABI."""
import numpy as np
import pytest

from helpers import declared

pytest.importorskip("torch")

HYBRID_ENTRIES = ("gutb200_hybrid_rays", "gutb200_hybrid_composite", "gutb200_hybrid_composite_bwd")


def test_nht_features_are_refused_by_key():
    import train_step_hybrid as th

    with pytest.raises(NotImplementedError, match="model.feature_type"):
        th.hybrid_render_conf({"model": {"feature_type": "nht"}, "render": {}})


def test_a_rolling_shutter_sensor_is_refused_by_key():
    import scenes
    import train_step_hybrid as th
    from threedgut_tracer.tracer import ShutterType, fromOpenCVPinholeCameraModelParameters

    sc = scenes.scene_c1(n=10, width=16, height=12)

    def sensor(shutter):
        return fromOpenCVPinholeCameraModelParameters(np.array([sc.width, sc.height]), shutter, np.array([sc.cx, sc.cy]), np.array([sc.fx, sc.fy]),
                                                      np.zeros(6), np.zeros(2), np.zeros(4))

    th.check_sensor(sensor(ShutterType.GLOBAL))
    for shutter in (ShutterType.ROLLING_TOP_TO_BOTTOM, ShutterType.ROLLING_RIGHT_TO_LEFT):
        with pytest.raises(NotImplementedError, match="shutter_type"):
            th.check_sensor(sensor(shutter))


@pytest.mark.parametrize("normal", [(0.0, 0.0, 0.0), (0, 0, 0)])
def test_a_zero_plane_normal_is_refused_by_key(normal):
    import train_step_hybrid as th

    with pytest.raises(NotImplementedError, match="plane_normal"):
        th.mirror_settings(dict(plane_normal=normal))


@pytest.mark.parametrize("reflectivity", [-0.1, 1.5, float("nan")])
def test_a_reflectivity_outside_the_unit_interval_is_refused_by_key(reflectivity):
    import train_step_hybrid as th

    with pytest.raises(NotImplementedError, match="reflectivity"):
        th.mirror_settings(dict(reflectivity=reflectivity))


def test_mirror_defaults_are_render_hybrids_and_the_normal_is_normalised():
    import inspect

    import hybrid
    import scenes
    import train_step_hybrid as th

    sig = inspect.signature(hybrid.render_hybrid).parameters
    m = th.mirror_settings()
    assert tuple(m["plane_point"]) == tuple(np.float32(sig["plane_point"].default))
    assert tuple(m["plane_normal"]) == tuple(np.float32(sig["plane_normal"].default))
    assert m["reflectivity"] == sig["reflectivity"].default
    assert th.mirror_settings(scenes.C5_MIRROR)["reflectivity"] == m["reflectivity"]
    for r in (0.0, 1.0):
        assert th.mirror_settings(dict(reflectivity=r))["reflectivity"] == r
    tilted = th.mirror_settings(dict(plane_normal=(3.0, 0.0, 4.0)))["plane_normal"]
    assert tilted.dtype == np.float32 and np.allclose(tilted, [0.6, 0.0, 0.8], atol=1e-7)
    with pytest.raises(ValueError, match="unknown"):
        th.mirror_settings(dict(normal=(0, 0, 1)))


@pytest.mark.parametrize("render", [{}, {"particle_kernel_degree": 4, "min_transmittance": 0.001}, {"primitive_type": "icosahedron",
                                                                                                     "particle_kernel_density_clamping": False}])
def test_both_tracers_read_the_same_filled_render_section(render):
    """The 3DGUT pass reads the filled section through its config builder, the 3DGRT pass through cfg_get with its own defaults
    (threedgrt_tracer.Tracer): both see the same kernel degree and min_transmittance, 3dgut.yaml's where the user sets none."""
    import train_step_hybrid as th
    from b200_native import cfg_get
    from threedgut_tracer.tracer import _native_config

    user = {"render": dict(render)}
    conf = th.hybrid_render_conf(user)
    assert user == {"render": dict(render)}  # the caller's config is not modified
    gut = _native_config(conf)
    grt_degree = int(cfg_get(conf, "render.particle_kernel_degree", 4))
    grt_min_t = float(cfg_get(conf, "render.min_transmittance", 0.001))
    assert gut.kernel_degree == grt_degree == int(render.get("particle_kernel_degree", 2))
    assert np.float32(gut.min_transmittance) == np.float32(grt_min_t) == np.float32(render.get("min_transmittance", 1e-4))
    assert np.float32(gut.max_alpha) == np.float32(cfg_get(conf, "render.particle_kernel_max_alpha", 0.0)) == np.float32(0.99)
    assert np.float32(gut.min_kernel_density) == np.float32(cfg_get(conf, "render.particle_kernel_min_response", 0.0)) == np.float32(0.0113)
    assert cfg_get(conf, "render.primitive_type", None) == render.get("primitive_type", "instances")
    assert bool(cfg_get(conf, "render.particle_kernel_density_clamping", None)) == render.get("particle_kernel_density_clamping", True)
    assert int(cfg_get(conf, "render.max_consecutive_bvh_update", 0)) == 15


def test_a_min_alpha_the_3dgrt_pass_cannot_take_is_refused_by_key():
    import train_step_hybrid as th

    th.hybrid_render_conf({"render": {"particle_kernel_min_alpha": 1.0 / 255.0}})
    with pytest.raises(NotImplementedError, match="particle_kernel_min_alpha"):
        th.hybrid_render_conf({"render": {"particle_kernel_min_alpha": 0.01}})


def test_c5_is_c3s_generator_with_a_seed_of_its_own():
    import scenes

    c5 = scenes.scene_c5(n=2000)
    c3 = scenes.scene_c3(n=2000)
    assert (c5.width, c5.height, c5.fx, c5.fy, c5.camera_radius) == (1237, 822, c3.fx, c3.fy, c3.camera_radius) and c5.n == 2000
    assert c5.name.startswith("c5") and c3.name.startswith("c3")
    assert not np.array_equal(c5.particles, c3.particles)
    assert np.array_equal(scenes.scene_c3(n=2000, seed=23).particles, c5.particles)


def test_hybrid_entry_points_are_declared_exported_and_bound():
    import b200_native as nat
    import train_step_hybrid as th

    lib = nat.load()
    for name in HYBRID_ENTRIES:
        assert name in declared("gut_b200.h") and name in nat.EXPORTS
        assert hasattr(lib, name), name
    assert "grtb200_trace_bwd_accumulate" in declared("grt_b200.h") and "grtb200_trace_bwd_accumulate" in nat.GRT_EXPORTS
    assert hasattr(lib, "grtb200_trace_bwd_accumulate")
    assert th.PHASES == ("rays", "primary", "build", "secondary", "loss", "backward_primary", "backward_secondary", "exchange", "adam", "densify")


def test_accumulate_is_an_sh_option_of_trace_bwd_with_out():
    from threedgrt_tracer.tracer import OptixTracer

    assert "accumulate" in OptixTracer.trace_bwd.__code__.co_varnames
    ot = OptixTracer.__new__(OptixTracer)  # no context: the refusal comes before any device work
    ot._nht = None
    with pytest.raises(NotImplementedError, match="accumulate"):
        ot.trace_bwd(0, None, None, None, None, None, None, None, None, None, None, None, None, None, 0, 3, 0.001, out=None, accumulate=True)

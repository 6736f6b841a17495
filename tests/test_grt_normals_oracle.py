"""CPU checks of the 3DGRT normals (render.enable_normals with SH radiance): which configurations the tracer accepts, and the float64
normals oracle (tests/grt_normals_oracle.py) on cases worked out by hand from the reference's formula."""
import math

import numpy as np
import pytest

from oracle import gut_oracle as go

torch = pytest.importorskip("torch")
import grt_normals_oracle as gnr  # noqa: E402

F64 = torch.float64


def test_sh_with_normals_passes_the_pipeline_check():
    from threedgrt_tracer.tracer import _check_pipelines, _nht_config

    _check_pipelines("reference", "referenceBwd", False, True)
    assert _nht_config({"render": {"enable_normals": True}}) is None
    assert _nht_config({"model": {"feature_type": "sh"}, "render": {"enable_normals": True, "pipeline_type": "reference"}}) is None


def test_nht_with_normals_is_still_refused():
    from threedgrt_tracer.tracer import _check_pipelines, _nht_config

    with pytest.raises(NotImplementedError, match="render.enable_normals"):
        _check_pipelines("referenceSlang", "referenceSlangBwd", True, True)
    conf = {"model": {"feature_type": "nht"}, "render": {"pipeline_type": "referenceSlang", "backward_pipeline_type": "referenceSlangBwd",
                                                         "enable_normals": True}}
    with pytest.raises(NotImplementedError, match="SH radiance"):
        _nht_config(conf)


def test_hybrid_conf_keeps_the_normals_key():
    from train_step_hybrid import hybrid_render_conf

    assert hybrid_render_conf({"render": {"enable_normals": True}})["render"]["enable_normals"] is True


def _t(row):
    return torch.as_tensor(np.asarray(row, np.float64)[None])


@pytest.mark.parametrize("direction", [(0.0, 0.0, 1.0), (1.0, 2.0, 3.0), (-0.3, 0.9, -0.1)])
def test_isotropic_gaussian_through_its_centre_faces_the_ray(direction):
    """Identity rotation, equal scales, ray through the centre: gro = -t0 d / s, grayDist = 0, gro + grd (t0 / s - 3) = -3 d, so the
    normal is -d whatever the scale."""
    d = np.asarray(direction, np.float64)
    d /= np.linalg.norm(d)
    mu = np.array([0.2, -0.1, 0.4])
    o = mu - 2.5 * d
    n = gnr.hit_normals(_t(o), _t(d), _t(mu), _t([1.0, 0.0, 0.0, 0.0]), _t([0.3, 0.3, 0.3]))[0].numpy()
    assert np.allclose(n, -d, atol=1e-12)


def test_rotated_anisotropic_gaussian_by_hand():
    """90 degrees about z (q = (cos 45, 0, 0, sin 45)), scale (1, 2, 0.5) at the origin, ray o = (0.5, 0, -4), d = +z.  The rows of
    quaternionWXYZToMatrix are m0 = (0, 1, 0), m1 = (-1, 0, 0), m2 = (0, 0, 1), so gro = (m_i . o) / s_i = (0, -0.25, -8), grd = (0, 0, 1),
    gcrod = grd x gro = (0.25, 0, 0), grayDist = 1/16, dot(grd, -gro) = 8; gro + grd (8 - sqrt(9 - 1/16)) = (0, -0.25, -sqrt(8.9375));
    R s = sum_i s_i m_i = (-2, 1, 0.5); the element-wise product is (0, -0.25, -sqrt(8.9375) / 2)."""
    c = math.sqrt(0.5)
    n = gnr.hit_normals(_t([0.5, 0.0, -4.0]), _t([0.0, 0.0, 1.0]), _t([0.0, 0.0, 0.0]), _t([c, 0.0, 0.0, c]), _t([1.0, 2.0, 0.5]))[0].numpy()
    v = np.array([0.0, -0.25, -math.sqrt(8.9375) / 2.0])
    assert np.allclose(n, v / np.linalg.norm(v), atol=1e-12)
    assert np.allclose(n, [0.0, -0.164957, -0.986301], atol=1e-6)


def test_outside_the_ellipsoid_radius_is_nan_as_in_the_reference():
    """grayDist > 9 (reachable only with particle_kernel_min_response < exp(-4.5)): sqrt of a negative number."""
    n = gnr.hit_normals(_t([3.5, 0.0, -4.0]), _t([0.0, 0.0, 1.0]), _t([0.0, 0.0, 0.0]), _t([1.0, 0.0, 0.0, 0.0]), _t([1.0, 1.0, 1.0]))
    assert torch.isnan(n).all()


def _single(x_offset, density, degree=4):
    """One Gaussian (the rotated anisotropic one above, at the origin) and one ray along +z through the oracle's lists."""
    c = math.sqrt(0.5)
    particles = np.array([[0.0, 0.0, 0.0, density, c, 0.0, 0.0, c, 0.1, 0.2, 0.05, 0.0]], np.float32)
    ro = np.array([[[[x_offset, 0.0, -4.0]]]], np.float32)
    rd = np.array([[[[0.0, 0.0, 1.0]]]], np.float32)
    cfg = go.grt_config()
    cfg.kernel_degree = degree
    return gnr.frame(cfg, particles, ro[0], rd[0], np.eye(4, dtype=np.float32)), particles


@pytest.mark.parametrize("degree", [4, 2])
def test_one_hit_through_the_oracle_lists_is_weighted_by_alpha(degree):
    """The sum over the C oracle's lists: one accepted hit, weight = alpha (T = 1) times the hand-derived direction."""
    (nrm, lists), particles = _single(0.05, 0.8, degree)
    assert lists["count"][0] == 1 and lists["alpha"][0, 0] > 0
    alpha = lists["alpha"][0, 0]
    # as above with o = (0.05, 0, -4) and s = (0.1, 0.2, 0.05): gro = (0, -0.25, -80), grayDist = 1/16, R s = (-0.2, 0.1, 0.05)
    gray = 1.0 / 16.0
    resp = math.exp(-gray * gray / 18.0) if degree == 4 else math.exp(-0.5 * gray)
    assert abs(alpha - min(0.99, 0.8 * resp)) < 1e-6
    v = np.array([0.0, -0.25 * 0.1, -math.sqrt(9.0 - gray) * 0.05])
    assert np.allclose(nrm[0], alpha * v / np.linalg.norm(v), atol=1e-6)  # the particle record is float32: 0.05, sqrt(0.5) round


def test_two_hits_compose_with_the_transmittance_between_them():
    """Two isotropic Gaussians on the axis of a ray: the first hit weighs alpha1, the second alpha2 (1 - alpha1); both face -d."""
    particles = np.array([[0.0, 0.0, z, 0.6, 1.0, 0.0, 0.0, 0.0, 0.05, 0.05, 0.05, 0.0] for z in (0.0, 0.5)], np.float32)
    ro = np.array([[[0.0, 0.0, -3.0]]], np.float32)
    rd = np.array([[[0.0, 0.0, 1.0]]], np.float32)
    nrm, lists = gnr.frame(go.grt_config(), particles, ro, rd, np.eye(4, dtype=np.float32))
    assert lists["count"][0] == 2 and (lists["alpha"][0, :2] > 0).all()
    a1, a2 = lists["alpha"][0, 0], lists["alpha"][0, 1]
    assert np.allclose(nrm[0], [0.0, 0.0, -(a1 + a2 * (1 - a1))], atol=1e-12)


def test_rays_that_accept_nothing_have_a_zero_normal():
    particles = np.array([[0.0, 0.0, 0.0, 0.6, 1.0, 0.0, 0.0, 0.0, 0.05, 0.05, 0.05, 0.0]], np.float32)
    ro = np.array([[[2.0, 0.0, -3.0]]], np.float32)
    rd = np.array([[[0.0, 0.0, 1.0]]], np.float32)
    nrm, lists = gnr.frame(go.grt_config(), particles, ro, rd, np.eye(4, dtype=np.float32))
    assert lists["count"][0] == 0 and np.array_equal(nrm, np.zeros((1, 3)))

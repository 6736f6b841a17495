"""The shared record helpers on the CPU: train_step.raw_params (the inverse of train_step.particle_record that the training-step tests
and scripts start from) and scenes.Scene.pinhole_sensor (the 3DGUT sensor of a scene's pinhole rays)."""
import dataclasses

import numpy as np
import pytest

import scenes

torch = pytest.importorskip("torch")


def _records(seed):
    """A C1 record ([N,12]: unit quaternions, zero pad column, densities in [0.05, 0.9]) with a few densities moved onto and past the
    clamp, its [N,48] SH and [N,48] NHT features."""
    sc = scenes.scene_c1(n=300, seed=seed)
    P = torch.from_numpy(sc.particles)
    P[:4, 3] = torch.tensor([0.0, 1.0, 1e-6, 1.0 - 1e-6])
    F = torch.from_numpy(np.random.default_rng(seed).uniform(-np.pi / 2, np.pi / 2, (sc.n, 48)).astype(np.float32))
    return P, torch.from_numpy(sc.sph), F


def _inline(P, S=None, F=None):
    """The inverse as the tests and scripts wrote it out before raw_params."""
    dns = P[:, 3:4].clamp(1e-4, 1 - 1e-4)
    out = {"positions": P[:, 0:3].clone(), "density": torch.log(dns / (1 - dns)), "rotation": P[:, 4:8].clone(), "scale": torch.log(P[:, 8:11])}
    if F is not None:
        out["features"] = F.clone()
    else:
        out.update(features_albedo=S[:, 0:3].clone(), features_specular=S[:, 3:48].clone())
    return out


@pytest.mark.parametrize("kind", ["sh", "nht"])
@pytest.mark.parametrize("seed", [0, 1])
def test_raw_params_is_bit_identical_to_the_inline_inverse(kind, seed):
    import train_step

    P, S, F = _records(seed)
    got = train_step.raw_params(P, S) if kind == "sh" else train_step.raw_params(P, features=F)
    want = _inline(P, S) if kind == "sh" else _inline(P, F=F)
    assert list(got) == list(want)
    for k, w in want.items():
        g = got[k]
        assert g.dtype == torch.float32 and g.shape == w.shape and g.is_contiguous(), k
        assert torch.equal(g.view(torch.int32), w.view(torch.int32)), k
        assert g.untyped_storage().data_ptr() not in (P.untyped_storage().data_ptr(), S.untyped_storage().data_ptr(),
                                                      F.untyped_storage().data_ptr()), f"{k} aliases its input"


def test_raw_params_inverts_particle_record():
    import train_step

    sc = scenes.scene_c1(n=300, seed=3)
    P, S = torch.from_numpy(sc.particles), torch.from_numpy(sc.sph)
    assert float(P[:, 3].min()) > 1e-4 and float(P[:, 3].max()) < 1 - 1e-4
    raw = train_step.raw_params(P, S)
    rec = train_step.particle_record(raw)
    assert torch.equal(rec[:, 11], torch.zeros(sc.n)) and torch.equal(rec[:, 0:3], P[:, 0:3])
    # sigmoid(logit d), exp(log s) and normalize(q) of a unit q round-trip to a few fp32 ulps
    torch.testing.assert_close(rec, P, rtol=1e-6, atol=0.0)
    assert torch.equal(torch.cat([raw["features_albedo"], raw["features_specular"]], 1), S)


def test_raw_params_takes_exactly_one_feature_kind():
    import train_step

    P, S, F = _records(0)
    with pytest.raises(ValueError):
        train_step.raw_params(P)
    with pytest.raises(ValueError):
        train_step.raw_params(P, S, F)


@pytest.mark.parametrize("scene", ["c1", "c3"])
def test_pinhole_sensor_matches_the_hand_built_sensor(scene):
    from threedgut_tracer.tracer import ShutterType, fromOpenCVPinholeCameraModelParameters

    sc = scenes.scene_c1(n=50, width=128, height=96) if scene == "c1" else scenes.scene_c3(n=1000)
    want = fromOpenCVPinholeCameraModelParameters(np.array([sc.width, sc.height]), ShutterType.GLOBAL, np.array([sc.cx, sc.cy], np.float32),
                                                  np.array([sc.fx, sc.fy], np.float32), np.zeros(6, np.float32), np.zeros(2, np.float32),
                                                  np.zeros(4, np.float32))
    got = sc.pinhole_sensor()
    for field in dataclasses.fields(want):
        a, b = getattr(got, field.name), getattr(want, field.name)
        if isinstance(b, np.ndarray):
            assert a.dtype == b.dtype and np.array_equal(a, b), field.name
        else:
            assert type(a) is type(b) and a == b, field.name


def test_pinhole_sensor_refuses_a_fisheye_scene():
    sc = dataclasses.replace(scenes.scene_c1(n=50), fisheye=(0.1, 0.0, 0.0, 0.0, 1.5))
    with pytest.raises(ValueError, match="fisheye"):
        sc.pinhole_sensor()

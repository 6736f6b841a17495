"""CPU checks of the float64 NHT render oracle (tests/nht_render_oracle.py) and of the tracer's NHT config validation."""
import math

import numpy as np
import pytest

import scenes
from helpers import rel_l2
from oracle import gut_oracle as go

torch = pytest.importorskip("torch")
import nht_render_oracle as nro  # noqa: E402


def _slang_features(P, f):
    """Literal numpy restatement of featuresFromParametersBuffer (neuralHarmonicFeaturesParticle.slang:46-66, 123-134, 152-189)."""
    edge, face_h, face_r, height, in_r = math.sqrt(24.0), math.sqrt(24.0) * math.sqrt(3.0) / 2, math.sqrt(2.0), 4.0, 1.0
    v = [np.array([0.5 * edge, -face_r, -1.0]), np.array([-0.5 * edge, -face_r, -1.0]), np.array([0.0, face_h - face_r, -1.0]),
         np.array([0.0, 0.0, height - in_r])]
    e1, e2, e3 = v[1] - v[0], v[2] - v[0], v[3] - v[0]
    c23 = np.cross(e2, e3)
    inv_det = 1.0 / np.dot(e1, c23)
    d = np.asarray(P, np.float64) - v[0]
    wy = np.dot(d, c23) * inv_det
    wz = np.dot(e1, np.cross(d, e3)) * inv_det
    ww = np.dot(e1, np.cross(e2, d)) * inv_det
    w = [1.0 - wy - wz - ww, wy, wz, ww]
    base = [f[n] * w[0] for n in range(12)]
    for k in range(1, 4):
        for n in range(12):
            base[n] += w[k] * f[k * 12 + n]
    out = []
    for k in range(12):
        out += [math.sin(base[k]), math.cos(base[k])]
    return np.array(w), np.array(out)


def test_feature_function_matches_the_slang():
    rng = np.random.default_rng(3)
    f = rng.uniform(-math.pi / 2, math.pi / 2, 48)
    # the weights are one-hot at the vertices and 1/4 at the incentre
    for k in range(4):
        w = nro.barycentric(torch.tensor(nro.TETRA[k], dtype=torch.float64)).numpy()
        assert np.allclose(w, np.eye(4)[k], atol=1e-12)
    assert np.allclose(nro.barycentric(torch.zeros(3, dtype=torch.float64)).numpy(), 0.25, atol=1e-12)
    # inside, outside (extrapolating) and far points
    pts = np.concatenate([rng.normal(size=(20, 3)), 4.0 * rng.normal(size=(10, 3)), nro.TETRA, np.zeros((1, 3))])
    got = nro.features_at(torch.tensor(pts), torch.tensor(f)).numpy()
    for p, g in zip(pts, got):
        w, ref = _slang_features(p, f)
        assert np.allclose(nro.barycentric(torch.tensor(p)).numpy(), w, atol=1e-12)
        assert np.allclose(g, ref, atol=1e-12)


def _scene(seed=20, n=90, w=48, h=40):
    sc = scenes.scene_c1(n=n, seed=seed, width=w, height=h)
    cam = go.make_camera(sc.width, sc.height, sc.fx, sc.fy, sc.cx, sc.cy, scenes.pose7_from_c2w(sc.camera(seed % 5, 5)))
    feats = np.random.default_rng(seed).uniform(-math.pi / 2, math.pi / 2, (sc.n, 48)).astype(np.float32)
    return sc, cam, feats


# render settings off the default the pins run at as well: earlier termination, and the *_3dgut_mcmc_nht configs' sigma-point spread
# (ut_delta follows ut_alpha as threedgut_tracer._native_config sets it)
SETTINGS = {"min_transmittance=0.03": dict(min_transmittance=0.03), "ut_alpha=0.1": dict(ut_alpha=0.1, ut_delta=math.sqrt(0.03))}


def _config(settings=None):
    cfg = go.default_config()
    for k, v in (settings or {}).items():
        setattr(cfg, k, v)
    return cfg


def _alpha_dist_hits(settings=None):
    sc, cam, feats = _scene()
    cfg = _config(settings)
    ro, rd = sc.rays()
    fr = nro.frame(cfg, cam, sc.particles, feats, ro, rd, go)
    assert fr["bn"].sorted_values.size > 200
    rgba, dist, hits = go.render_forward(cfg, cam, ro, rd, sc.particles, fr["pr"], fr["bn"], f64=True)
    assert np.abs(fr["out"][..., 24] - rgba[..., 3]).max() < 1e-6
    assert np.abs(fr["dist"] - dist).max() < 1e-5 * max(1.0, np.abs(dist).max())
    assert np.array_equal(fr["hits"], hits)
    return fr


def test_alpha_dist_hits_equal_the_sh_forward_in_f64():
    _alpha_dist_hits()


def _sh_adjoint(settings=None):
    """d_features = 0 on an unclamped scene: the NHT adjoint of alpha and distance is the SH path's, which the C oracle pins."""
    sc, cam, feats = _scene(seed=21)
    assert sc.particles[:, 3].max() < 0.99  # alpha = response * density never reaches the clamp
    cfg = _config(settings)
    ro, rd = sc.rays()
    rng = np.random.default_rng(5)
    h, w = sc.height, sc.width
    d_out = np.zeros((h, w, 25))
    d_out[..., 24] = rng.normal(size=(h, w))
    d_dist = 0.2 * rng.normal(size=(h, w, 1))
    fr = nro.frame(cfg, cam, sc.particles, feats, ro, rd, go, d_out=d_out, d_dist=d_dist)
    rgba, dist, _ = go.render_forward(cfg, cam, ro, rd, sc.particles, fr["pr"], fr["bn"], f64=True)
    d_rgba = np.zeros((h, w, 4), np.float32)
    d_rgba[..., 3] = d_out[..., 24]
    dp, _ = go.render_backward(cfg, cam, ro, rd, sc.particles, np.zeros((sc.n, 48), np.float32), 0, fr["pr"], fr["bn"], rgba, dist, d_rgba,
                               d_dist.astype(np.float32), f64=True)
    for name, sl in (("pos", slice(0, 3)), ("density", slice(3, 4)), ("quat", slice(4, 8)), ("scale", slice(8, 11))):
        err = rel_l2(fr["dp"][:, sl], dp[:, sl])
        print(f"{name}: rel-L2 {err:.2e}")
        assert err < 1e-6, name
    assert np.abs(fr["df"]).max() == 0.0


def test_density_adjoint_equals_the_sh_adjoint_with_a_zero_rgb_gradient():
    _sh_adjoint()


def _central_differences(settings=None):
    sc, cam, feats = _scene(seed=22, n=40, w=32, h=32)
    particles = sc.particles.copy()
    cfg = _config(settings)
    ro, rd = sc.rays()
    fr0 = nro.frame(cfg, cam, particles, feats, ro, rd, go)
    # the particle with the most hits gets a density high enough to clamp alpha at 0.99 in its centre
    counts = np.bincount(fr0["bn"].sorted_values.astype(np.int64), minlength=sc.n)
    top = int(np.argmax(counts))
    particles[top, 3] = 5.0
    rng = np.random.default_rng(9)
    d_out = rng.normal(size=(sc.height, sc.width, 25))
    d_dist = 0.1 * rng.normal(size=(sc.height, sc.width, 1))
    fr = nro.frame(cfg, cam, particles, feats, ro, rd, go, d_out=d_out, d_dist=d_dist)
    pr, bn = fr["pr"], fr["bn"]
    _, inv, _ = go.sensor_matrices(cam)

    def loss(p_mod, f_mod):
        pos, dns, quat, scl = (torch.tensor(p_mod[:, 0:3]), torch.tensor(p_mod[:, 3]), torch.tensor(p_mod[:, 4:8]), torch.tensor(p_mod[:, 8:11]))
        ft = torch.tensor(f_mod)
        img, dist, _ = nro.render(cfg, inv, cam.width, cam.height, ro, rd, pos, dns, quat, scl, ft, bn.sorted_values, bn.ranges)
        return float((img * torch.tensor(d_out)).sum() + (dist * torch.tensor(d_dist)).sum())

    # the clamped pair's particle must reach the clamp for this check to mean anything
    assert fr["out"][..., 24].max() > 0.98
    p64 = particles.astype(np.float64)
    f64 = feats.astype(np.float64)
    visible = np.nonzero(counts > 0)[0]
    picks = [top] + [int(i) for i in rng.choice(visible, 3, replace=False) if i != top][:2]
    eps = 1e-6
    checked = 0
    for i in picks:
        for col in (0, 1, 2, 3, 4, 6, 8, 10):
            a, b = p64.copy(), p64.copy()
            a[i, col] += eps
            b[i, col] -= eps
            fd = (loss(a, f64) - loss(b, f64)) / (2 * eps)
            ag = fr["dp"][i, col]
            assert abs(fd - ag) <= 1e-5 * max(1.0, abs(fd)), (i, col, fd, ag)
            checked += 1
        for col in (0, 13, 30, 47):
            a, b = f64.copy(), f64.copy()
            a[i, col] += eps
            b[i, col] -= eps
            fd = (loss(p64, a) - loss(p64, b)) / (2 * eps)
            assert abs(fd - fr["df"][i, col]) <= 1e-5 * max(1.0, abs(fd)), (i, col, fd, fr["df"][i, col])
            checked += 1
    assert checked == 36


def test_autograd_matches_central_differences_including_a_clamped_pair():
    _central_differences()


@pytest.mark.parametrize("setting", list(SETTINGS))
def test_oracle_pins_at_other_render_settings(setting):
    """The three pins above at min_transmittance = 0.03 and at ut_alpha = 0.1: the f64 forward against the C oracle, the SH-adjoint
    equality, and central differences including a clamped pair."""
    fr = _alpha_dist_hits(SETTINGS[setting])
    sc, cam, feats = _scene()
    base = nro.frame(go.default_config(), cam, sc.particles, feats, *sc.rays(), go)
    if setting.startswith("min_t"):  # rays stop earlier: fewer composited hits
        assert fr["hits"].sum() < base["hits"].sum()
    else:  # the smaller sigma-point spread changes the lists
        assert not np.array_equal(fr["bn"].ranges, base["bn"].ranges)
    _sh_adjoint(SETTINGS[setting])
    _central_differences(SETTINGS[setting])


def test_tile_subset_backward_is_the_masked_full_frame_backward():
    """The sampling premise of tests/test_nht_render_headline_gpu.py: with output gradients zero outside a set of tiles, the backward of
    the whole frame (one autograd graph over every tile) equals the tile-subset oracle's, and the subset's forward is the full frame's
    at its pixels.  Tiles are independent: each pixel composites its own tile's list only."""
    sc, cam, feats = _scene(seed=23, n=300, w=75, h=53)  # ragged: 5 x 4 tiles, partial on both edges
    particles = sc.particles.copy()
    particles[::7, 3] = 3.0  # clamped pairs
    cfg = _config(SETTINGS["ut_alpha=0.1"])
    ro, rd = sc.rays()
    n_tiles = ((sc.width + 15) // 16) * ((sc.height + 15) // 16)
    tiles = [0, 4, 7, 18, 19]
    mask = np.zeros(sc.width * sc.height, bool)
    for t in tiles:
        mask[nro.tile_pixels(t, sc.width, sc.height)] = True
    mask = mask.reshape(sc.height, sc.width, 1)
    rng = np.random.default_rng(4)
    d_out = rng.normal(size=(sc.height, sc.width, 25)) * mask
    d_dist = 0.1 * rng.normal(size=(sc.height, sc.width, 1)) * mask
    part = nro.frame(cfg, cam, particles, feats, ro, rd, go, d_out=d_out, d_dist=d_dist, tiles=tiles)
    assert part["hits"][mask[..., 0]].sum() > 4 * mask.sum() and np.all(part["hits"][~mask[..., 0]] == 0)
    _, inv, _ = go.sensor_matrices(cam)
    lv = nro.leaves(particles, feats)
    img, dist, hits = nro.render(cfg, inv, cam.width, cam.height, ro, rd, *lv, part["bn"].sorted_values, part["bn"].ranges)
    assert part["bn"].ranges.shape[0] == n_tiles
    for name, a, b in (("out", img, part["out"]), ("dist", dist, part["dist"]), ("hits", hits, part["hits"])):
        assert np.array_equal(a.detach().numpy()[mask[..., 0]], b[mask[..., 0]]), name
    loss = (img * torch.tensor(d_out)).sum() + (dist * torch.tensor(d_dist)).sum()
    gp, gd, gq, gs, gf = torch.autograd.grad(loss, lv)
    full_dp = torch.cat([gp, gd[:, None], gq, gs, torch.zeros((sc.n, 1), dtype=torch.float64)], 1).numpy()
    assert np.abs(part["dp"]).max() > 0 and np.abs(part["df"]).max() > 0 and part["clamped"] > 0
    for name, a, b in (("d_particles", full_dp, part["dp"]), ("d_features", gf.numpy(), part["df"])):
        err = rel_l2(b, a)
        print(f"[sample] NHT {name}: tile subset vs masked full frame rel-L2 {err:.2e}")
        assert err <= 1e-12, name


@pytest.mark.parametrize("key,value", [
    ("model.feature_type", "rgb"),
    ("model.nht_features.dim", 64),
    ("model.nht_features.activation.type", "siren"),
    ("model.nht_features.activation.num_frequencies", 2),
    ("model.nht_features.interpolation_type", "none"),
    ("render.splat.k_buffer_size", 16),
])
def test_unsupported_nht_configs_are_refused(key, value):
    from threedgut_tracer.tracer import _nht_config

    conf = {"model": {"feature_type": "nht", "nht_features": {"dim": 48, "activation": {"type": "sincos", "num_frequencies": 1},
                                                                "interpolation_type": "barycentric"}},
            "render": {"particle_feature_half": True, "splat": {"k_buffer_size": 0}}}
    assert _nht_config(conf) == {"half": True}
    assert _nht_config({"model": {"feature_type": "sh"}}) is None and _nht_config({}) is None
    node = conf
    *path, last = key.split(".")
    for p in path:
        node = node[p]
    node[last] = value
    with pytest.raises(NotImplementedError, match=key.split(".")[-1] if key != "model.feature_type" else "feature_type"):
        _nht_config(conf)

"""CPU checks of the float64 3DGRT NHT oracle (tests/grt_nht_oracle.py) and of the 3DGRT tracer's NHT configuration check.

- The exported hit lists are the ones grt_oracle_trace / grt_ico_oracle_trace integrate: recomposited in numpy with the oracle's
  float32 arithmetic they reproduce its SH images, alpha, distances and hit counts bit for bit.
- Autograd of the oracle agrees with central differences, with a hit clamped at max_alpha = 0.999 and with the last-hit rule.
- With a zero feature gradient on an unclamped scene its density and geometry adjoint is the C oracle's SH adjoint.
- Every pairing the tracer does not build is refused with NotImplementedError naming the key.
"""
import ctypes as C
import math

import numpy as np
import pytest

import scenes
from helpers import rel_l2
from oracle import gut_oracle as go

torch = pytest.importorskip("torch")
import grt_ico_oracle as gio  # noqa: E402
import grt_nht_oracle as gno  # noqa: E402


def _frame(n=300, seed=3, w=24, h=20, cam=2, dist=10):
    sc = scenes.scene_c1(n=n, seed=seed, width=w, height=h)
    c2w = np.asarray(sc.camera(cam, dist), np.float32)
    ro, rd = sc.rays()
    return sc, c2w, ro[0], rd[0]


def _world_dirs_f32(rd, c2w):
    """grt_ray's direction in float32, left to right as the C code evaluates it"""
    m = np.asarray(c2w, np.float32)[:3, :4]
    rd = np.asarray(rd, np.float32).reshape(-1, 3)
    return np.stack([(m[a, 0] * rd[:, 0] + m[a, 1] * rd[:, 1]) + m[a, 2] * rd[:, 2] for a in range(3)], -1).astype(np.float32)


@pytest.mark.parametrize("primitive", ["instances", "icosahedron"])
def test_lists_reproduce_the_oracle_sh_images_exactly(primitive):
    sc, c2w, ro, rd = _frame()
    cfg = go.grt_config()
    rgb, alpha, dist, hits, _ = gio.grt_trace(cfg, sc.particles, sc.sph, 3, ro, rd, c2w, primitive=primitive)
    L = gno.trace_lists(cfg, sc.particles, ro, rd, c2w, primitive=primitive)
    assert L["count"].max() > 4 and (L["alpha"] > 0).sum() > 200
    R = L["count"].shape[0]
    d = _world_dirs_f32(rd, c2w)
    sph_eval = go.lib().gut_oracle_sph_eval
    f32 = np.float32
    T = np.ones(R, f32)
    Cc = np.zeros((R, 3), f32)
    D = np.zeros(R, f32)
    H = np.zeros(R, f32)
    rad = np.zeros(3, np.float32)
    sph = np.ascontiguousarray(sc.sph, np.float32)
    for r in range(R):
        dr = np.ascontiguousarray(d[r])
        for s in range(L["count"][r]):
            a = f32(L["alpha"][r, s])
            if a > 0:
                p = int(L["pid"][r, s])
                sph_eval(C.c_int32(3), sph[p].ctypes.data_as(C.POINTER(C.c_float)), dr.ctypes.data_as(C.POINTER(C.c_float)),
                         rad.ctypes.data_as(C.POINTER(C.c_float)))
                w = f32(a * T[r])
                Cc[r] = Cc[r] + np.maximum(rad, f32(0)) * w
                T[r] = f32(T[r] * f32(f32(1) - a))
                D[r] = f32(D[r] + f32(f32(L["depth"][r, s]) * w))
                H[r] += 1
    assert np.array_equal(Cc, rgb.reshape(R, 3))
    assert np.array_equal(f32(1) - T, alpha.reshape(R))
    assert np.array_equal(D, dist.reshape(R, 2)[:, 0]) and np.array_equal(L["last"], dist.reshape(R, 2)[:, 1])
    assert np.array_equal(H, hits.reshape(R))


def _clamped_scene():
    sc, c2w, ro, rd = _frame(n=60, seed=22, w=16, h=16, cam=1, dist=8)
    cfg = go.grt_config()
    cfg.max_alpha = 0.999
    particles = sc.particles.copy()
    L0 = gno.trace_lists(cfg, particles, ro, rd, c2w)
    counts = np.bincount(L0["pid"][L0["alpha"] > 0].astype(np.int64), minlength=sc.n)
    top = int(np.argmax(counts))
    particles[top, 3] = 5.0  # alpha = min(0.999, response * 5) clamps near its centre
    return sc, cfg, particles, c2w, ro, rd, counts, top


def test_autograd_matches_central_differences_with_a_clamped_hit_and_the_last_hit_rule():
    sc, cfg, particles, c2w, ro, rd, counts, top = _clamped_scene()
    feats = np.random.default_rng(9).uniform(-math.pi / 2, math.pi / 2, (sc.n, 48)).astype(np.float32)
    R = ro.reshape(-1, 3).shape[0]
    rng = np.random.default_rng(10)
    d_feat, d_alpha, d_dist = rng.normal(size=(R, 24)), rng.normal(size=R), 0.1 * rng.normal(size=R)
    fr = gno.frame(cfg, particles, feats, ro, rd, c2w, d_feat=d_feat, d_alpha=d_alpha, d_dist=d_dist)
    L = fr["lists"]
    assert (L["alpha"] == np.float32(0.999)).sum() > 0, "no hit reaches the clamp"
    on = np.arange(L["pid"].shape[1])[None, :] < L["count"][:, None]
    at_last = on & (L["alpha"] > 0) & (L["key"] == L["last"][:, None])
    assert at_last.sum() > 10, "the last-hit rule is not exercised"

    o, d = gno.world_rays(ro, rd, c2w)
    base = gno.leaves(particles, feats, requires_grad=False)

    def loss(p_mod, f_mod):
        live = tuple(torch.as_tensor(x) for x in (p_mod[:, 0:3], p_mod[:, 3:4], p_mod[:, 4:8], p_mod[:, 8:11], f_mod))
        F, A, D, _ = gno.composite(cfg, L, o, d, live, frozen=base)
        return float((F * torch.tensor(d_feat)).sum() + (A * torch.tensor(d_alpha)).sum() + (D * torch.tensor(d_dist)).sum())

    # the rule matters: the full autograd (last hits not frozen) differs from the reference adjoint
    live = gno.leaves(particles, feats)
    F, A, D, _ = gno.composite(cfg, L, o, d, live, frozen=live)
    full = torch.autograd.grad((F * torch.tensor(d_feat)).sum() + (A * torch.tensor(d_alpha)).sum() + (D * torch.tensor(d_dist)).sum(), live)
    assert rel_l2(fr["dp"][:, 0:3], full[0].numpy()) > 1e-3

    p64, f64 = particles.astype(np.float64), feats.astype(np.float64)
    last_pids = np.unique(L["pid"][at_last])
    picks = [top] + [int(i) for i in last_pids if i != top][:2]
    eps = 1e-6
    checked = 0
    for i in picks:
        for col in (0, 1, 2, 3, 4, 6, 8, 10):
            a, b = p64.copy(), p64.copy()
            a[i, col] += eps
            b[i, col] -= eps
            fd = (loss(a, f64) - loss(b, f64)) / (2 * eps)
            assert abs(fd - fr["dp"][i, col]) <= 1e-5 * max(1.0, abs(fd)), (i, col, fd, fr["dp"][i, col])
            checked += 1
        for col in (0, 13, 30, 47):
            a, b = f64.copy(), f64.copy()
            a[i, col] += eps
            b[i, col] -= eps
            fd = (loss(p64, a) - loss(p64, b)) / (2 * eps)
            assert abs(fd - fr["df"][i, col]) <= 1e-5 * max(1.0, abs(fd)), (i, col, fd, fr["df"][i, col])
            checked += 1
    assert checked == 36


def test_density_adjoint_equals_the_sh_adjoint_with_a_zero_feature_gradient():
    """d_features = 0 on an unclamped scene: the NHT adjoint of alpha and distance is the SH path's, which the C oracle pins.
    Instances only: the icosahedron oracle's float64 build compares its double entry t against the float `last` in the re-trace, so
    a last hit whose t rounds up to `last` is differentiated there; the float32 key comparison of the tracer (and of composite()) never
    does that.  The icosahedron lists are pinned by test_lists_reproduce_the_oracle_sh_images_exactly."""
    primitive = "instances"
    sc, c2w, ro, rd = _frame(n=200, seed=21, w=20, h=16, cam=3)
    assert sc.particles[:, 3].max() < 0.99
    cfg = go.grt_config()
    feats = np.random.default_rng(2).uniform(-1, 1, (sc.n, 48)).astype(np.float32)
    R = ro.reshape(-1, 3).shape[0]
    rng = np.random.default_rng(5)
    d_alpha, d_dist = rng.normal(size=R).astype(np.float32), (0.2 * rng.normal(size=R)).astype(np.float32)
    fr = gno.frame(cfg, sc.particles, feats, ro, rd, c2w, d_feat=np.zeros((R, 24)), d_alpha=d_alpha, d_dist=d_dist, primitive=primitive)
    rgb, alpha, dist, _, _ = gio.grt_trace(cfg, sc.particles, sc.sph, 3, ro, rd, c2w, f64=True, primitive=primitive)
    assert np.abs(fr["alpha"] - alpha.reshape(R)).max() < 1e-6
    assert np.array_equal(fr["dist"][:, 1].astype(np.float32), dist.reshape(R, 2)[:, 1])
    dp, _ = gio.grt_trace_bwd(cfg, sc.particles, sc.sph, 3, ro, rd, c2w, rgb, alpha, dist, np.zeros_like(rgb), d_alpha.reshape(alpha.shape),
                              d_dist.reshape(alpha.shape), f64=True, primitive=primitive)
    for name, sl in (("pos", slice(0, 3)), ("density", slice(3, 4)), ("quat", slice(4, 8)), ("scale", slice(8, 11))):
        err = rel_l2(fr["dp"][:, sl], dp[:, sl])
        print(f"{primitive} {name}: rel-L2 {err:.2e}")
        assert err < 1e-6, name
    assert np.abs(fr["df"]).max() == 0.0


def _conf(**render):
    conf = {"model": {"feature_type": "nht", "nht_features": {"dim": 48, "activation": {"type": "sincos", "num_frequencies": 1},
                                                               "interpolation_type": "barycentric"}},
            "render": {"pipeline_type": "referenceSlang", "backward_pipeline_type": "referenceSlangBwd", "particle_feature_half": True}}
    conf["render"].update(render)
    return conf


@pytest.mark.parametrize("change,key", [
    (("model.feature_type", "sh"), "render.pipeline_type"),                  # SH through the Slang pipelines
    (("render.pipeline_type", "reference"), "render.pipeline_type"),         # NHT through the CUDA pipelines
    (("render.backward_pipeline_type", "referenceBwd"), "render.backward_pipeline_type"),
    (("render.enable_normals", True), "render.enable_normals"),
    (("model.feature_type", "rgb"), "feature_type"),
    (("model.nht_features.dim", 64), "dim"),
    (("model.nht_features.activation.type", "siren"), "activation.type"),
    (("model.nht_features.activation.num_frequencies", 2), "num_frequencies"),
    (("model.nht_features.interpolation_type", "none"), "interpolation_type"),
])
def test_unsupported_pairings_are_refused(change, key):
    from threedgrt_tracer.tracer import _nht_config

    assert _nht_config(_conf()) == {"half": True}
    assert _nht_config({}) is None and _nht_config({"model": {"feature_type": "sh"}}) is None
    conf = _conf()
    path, value = change
    *parents, last = path.split(".")
    node = conf
    for p in parents:
        node = node.setdefault(p, {})
    node[last] = value
    with pytest.raises(NotImplementedError, match=key):
        _nht_config(conf)


def test_sh_with_a_slang_backward_is_refused():
    from threedgrt_tracer.tracer import _nht_config

    with pytest.raises(NotImplementedError, match="render.backward_pipeline_type"):
        _nht_config({"render": {"backward_pipeline_type": "referenceSlangBwd"}})

"""NHT features through the CUDA 3DGUT path (gutb200_forward_nht / gutb200_backward_nht, Tracer with model.feature_type: nht) against
the float64 autograd oracle (tests/nht_render_oracle.py) over the C oracle's sorted lists.

Bars (DESIGN.md section 5, applied to all 25 channels): mean |diff| <= 1e-5, |diff| <= 1e-4 on all but max(3, 2e-4 P) pixels, max |diff|
<= 2e-2; hit counts equal on >= 99.9 % of pixels; gradients rel-L2 <= 1e-3 per tensor."""
import math

import numpy as np
import pytest

import scenes
from helpers import dist_grad_blocks, dist_grad_mask, image_error_report, rel_l2
from oracle import gut_oracle as go

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import nht_render_oracle as nro  # noqa: E402


def _native():
    import b200_native

    return b200_native


def _scene(name):
    if name == "c1":
        return scenes.scene_c1(n=1000, seed=42, width=128, height=128)
    if name == "odd":
        return scenes.scene_c1(n=700, seed=5, width=75, height=53)
    sc = scenes.scene_c1(n=5000, seed=8, width=64, height=64)  # dense: tile lists of more than 256 entries
    return sc


def _setup(name, cam_i, deg, half, seed=0):
    sc = _scene(name)
    cfg = go.default_config()
    cfg.kernel_degree = deg
    cam = go.make_camera(sc.width, sc.height, sc.fx, sc.fy, sc.cx, sc.cy, scenes.pose7_from_c2w(sc.camera(cam_i, 5)))
    feats = np.random.default_rng(seed).uniform(-math.pi / 2, math.pi / 2, (sc.n, 48)).astype(np.float32)
    if half:
        feats = feats.astype(np.float16).astype(np.float32)  # what the kernel reads
    return sc, cfg, cam, feats


class _Gpu:
    """One native context and the device buffers of a frame."""

    def __init__(self, sc, deg, cam, feats, half, ro=None, rd=None):
        nat = _native()
        c = nat.default_config()
        c.kernel_degree = deg
        self.nat, self.ctx = nat, nat.Context(c, 0)
        self.cam = nat.Camera.from_buffer_copy(bytes(cam))
        if ro is None:
            ro, rd = sc.rays()
        self.ro = torch.from_numpy(np.ascontiguousarray(ro, np.float32)).cuda()
        self.rd = torch.from_numpy(np.ascontiguousarray(rd, np.float32)).cuda()
        self.p = torch.from_numpy(sc.particles).cuda()
        self.f = torch.from_numpy(feats).cuda().to(torch.float16 if half else torch.float32).contiguous()
        self.half, self.n, self.h, self.w = int(half), sc.n, sc.height, sc.width
        self.stream = torch.cuda.current_stream().cuda_stream

    def forward(self, fill=0.0):
        h, w, n = self.h, self.w, self.n
        self.out = torch.full((h, w, 25), fill, device="cuda")
        self.dist = torch.full((h, w, 1), fill, device="cuda")
        self.hits = torch.full((h, w, 1), fill, device="cuda")
        self.vis = torch.full((n, 1), fill, device="cuda")
        self.ctx.forward_nht(self.stream, self.cam, n, self.p.data_ptr(), self.f.data_ptr(), 48, self.half, self.ro.data_ptr(), self.rd.data_ptr(),
                             self.out.data_ptr(), self.dist.data_ptr(), self.hits.data_ptr(), self.vis.data_ptr())
        torch.cuda.synchronize()
        return self

    def backward(self, d_out, d_dist, cam=None, fill=0.0):
        d_out = torch.as_tensor(d_out, dtype=torch.float32).cuda().contiguous()
        d_dist = torch.as_tensor(d_dist, dtype=torch.float32).cuda().contiguous()
        dp = torch.full((self.n, 12), fill, device="cuda")
        df = torch.full((self.n, 48), fill, device="cuda")
        self.ctx.backward_nht(self.stream, self.cam if cam is None else cam, self.n, self.p.data_ptr(), self.f.data_ptr(), 48, self.half,
                              self.ro.data_ptr(), self.rd.data_ptr(), self.out.data_ptr(), d_out.data_ptr(), self.dist.data_ptr(),
                              d_dist.data_ptr(), dp.data_ptr(), df.data_ptr())
        torch.cuda.synchronize()
        return dp.cpu().numpy(), df.cpu().numpy()


def _check_frame(tag, sc, cfg, cam, feats, g, ro, rd, seed=1, d_dist_mode="random"):
    """d_dist_mode: helpers.dist_grad_mask ("zero" is what training passes: no warp of the backward takes the depth branch)."""
    rng = np.random.default_rng(seed)
    d_out = rng.normal(size=(sc.height, sc.width, 25)).astype(np.float32)
    d_dist = (0.1 * rng.normal(size=(sc.height, sc.width, 1))).astype(np.float32)
    d_dist *= dist_grad_mask(sc.height, sc.width, d_dist_mode, seed)[..., None]
    if d_dist_mode != "random":
        tag = f"{tag} d_dist={d_dist_mode} (warp blocks with / without a distance gradient {dist_grad_blocks(d_dist)})"
    ref = nro.frame(cfg, cam, sc.particles, feats, ro, rd, go, d_out=d_out, d_dist=d_dist, device="cuda")
    g.forward()
    out, dist, hits = g.out.cpu().numpy(), g.dist.cpu().numpy(), g.hits.cpu().numpy()
    P = sc.width * sc.height
    for name, got, want in (("features+alpha", out, ref["out"]), ("dist", dist, ref["dist"])):
        mean, mx, bad = image_error_report(f"{tag} {name}", got, want)
        assert mean <= 1e-5 and mx <= 2e-2 and bad <= max(3, int(2e-4 * P)), (name, mean, mx, bad)
    assert (hits == ref["hits"]).mean() >= 0.999
    dp, df = g.backward(d_out, d_dist)
    for name, a, b in (("d_pos", dp[:, 0:3], ref["dp"][:, 0:3]), ("d_density", dp[:, 3], ref["dp"][:, 3]), ("d_quat", dp[:, 4:8], ref["dp"][:, 4:8]),
                       ("d_scale", dp[:, 8:11], ref["dp"][:, 8:11]), ("d_features", df, ref["df"])):
        err = rel_l2(a, b)
        print(f"[parity] {tag} {name}: rel-L2 {err:.2e}")
        assert err <= 1e-3, (name, err)
    return ref


FRAMES = [("c1", 0, 2, False), ("c1", 3, 4, True), ("odd", 0, 4, False), ("odd", 3, 2, True), ("dense", 0, 2, False), ("dense", 3, 4, True)]
CASES = [pytest.param(*f, "random", id="-".join(map(str, f))) for f in FRAMES] \
    + [pytest.param(*f, m, id="-".join(map(str, f)) + f"-{m}_d_dist") for m in ("zero", "mixed") for f in FRAMES]


@pytest.mark.parametrize("name,cam_i,deg,half,d_dist", CASES)
def test_nht_matches_the_f64_oracle(name, cam_i, deg, half, d_dist):
    sc, cfg, cam, feats = _setup(name, cam_i, deg, half)
    ro, rd = sc.rays()
    g = _Gpu(sc, deg, cam, feats, half)
    ref = _check_frame(f"{name} cam{cam_i} deg{deg} {'fp16' if half else 'fp32'}", sc, cfg, cam, feats, g, ro, rd, d_dist_mode=d_dist)
    if name == "dense":
        assert np.diff(ref["bn"].ranges.astype(np.int64), axis=1).max() > 256


def test_nht_with_per_pixel_origins():
    sc, cfg, cam, feats = _setup("c1", 1, 2, False)
    ro, rd = sc.rays()
    ro = ro + 0.01 * np.random.default_rng(4).normal(size=ro.shape).astype(np.float32)
    _check_frame("c1 jittered origins", sc, cfg, cam, feats, _Gpu(sc, 2, cam, feats, False, ro, rd), ro, rd)


def test_alpha_dist_hits_visibility_equal_the_sh_forward():
    sc, cfg, cam, feats = _setup("c1", 2, 2, False)
    g = _Gpu(sc, 2, cam, feats, False).forward()
    rgba = torch.empty((sc.height, sc.width, 4), device="cuda")
    dist, hits, vis = torch.empty_like(g.dist), torch.empty_like(g.hits), torch.empty_like(g.vis)
    sph = torch.from_numpy(sc.sph).cuda()
    g.ctx.forward(g.stream, g.cam, sc.n, g.p.data_ptr(), sph.data_ptr(), 3, g.ro.data_ptr(), g.rd.data_ptr(), rgba.data_ptr(), dist.data_ptr(),
                  hits.data_ptr(), vis.data_ptr())
    torch.cuda.synchronize()
    same = {k: bool(torch.equal(a, b)) for k, a, b in (("alpha", g.out[..., 24], rgba[..., 3]), ("dist", g.dist, dist), ("hits", g.hits, hits),
                                                        ("visibility", g.vis, vis))}
    print(f"[parity] NHT vs SH forward bit-identical: {same}")
    assert (g.out[..., 24] - rgba[..., 3]).abs().max().item() <= 1e-6
    assert (g.dist - dist).abs().max().item() <= 1e-5
    assert torch.equal(g.hits, hits) and torch.equal(g.vis, vis)


def test_outputs_prefilled_with_nan_are_all_written():
    sc, cfg, cam, feats = _setup("odd", 1, 2, True)
    g = _Gpu(sc, 2, cam, feats, True).forward(fill=float("nan"))
    for t in (g.out, g.dist, g.hits, g.vis):
        assert not torch.isnan(t).any()
    rng = np.random.default_rng(2)
    dp, df = g.backward(rng.normal(size=(sc.height, sc.width, 25)), rng.normal(size=(sc.height, sc.width, 1)), fill=float("nan"))
    assert not np.isnan(dp).any() and not np.isnan(df).any()


def test_backward_after_another_camera_or_kind_is_refused():
    sc, cfg, cam, feats = _setup("odd", 0, 2, False)
    g = _Gpu(sc, 2, cam, feats, False).forward()
    other = g.nat.Camera.from_buffer_copy(bytes(g.cam))
    other.pose_start[0] += 0.1
    other.pose_end[0] += 0.1
    z = np.zeros((sc.height, sc.width, 25), np.float32)
    with pytest.raises(RuntimeError, match="camera"):
        g.backward(z, z[..., :1], cam=other)
    sph = torch.zeros((sc.n, 48), device="cuda")
    d = torch.zeros((sc.height, sc.width, 4), device="cuda")
    dp = torch.empty((sc.n, 12), device="cuda")
    with pytest.raises(RuntimeError, match="NHT"):
        g.ctx.backward(g.stream, g.cam, sc.n, g.p.data_ptr(), sph.data_ptr(), 3, g.ro.data_ptr(), g.rd.data_ptr(), d.data_ptr(), d.data_ptr(),
                       g.dist.data_ptr(), g.dist.data_ptr(), dp.data_ptr(), sph.data_ptr())


def _conf(half):
    return {"model": {"feature_type": "nht", "nht_features": {"dim": 48, "activation": {"type": "sincos", "num_frequencies": 1},
                                                               "interpolation_type": "barycentric"}},
            "render": {"particle_feature_half": half}}


class _Gaussians:
    def __init__(self, particles, feats):
        p = torch.from_numpy(np.asarray(particles, np.float32)).cuda()
        self.positions = p[:, 0:3].clone().requires_grad_(True)
        self.dns = p[:, 3:4].clone().requires_grad_(True)
        self.rot = p[:, 4:8].clone().requires_grad_(True)
        self.scl = p[:, 8:11].clone().requires_grad_(True)
        self.feats = torch.from_numpy(np.asarray(feats, np.float32)).cuda().requires_grad_(True)
        self.n_active_features = 0
        self.ray_feature_dim = 24

    def get_rotation(self):
        return self.rot

    def get_scale(self):
        return self.scl

    def get_density(self):
        return self.dns

    def get_features(self):
        return self.feats

    def params(self):
        return [self.positions, self.dns, self.rot, self.scl, self.feats]


class _Batch:
    def __init__(self, sc, c2w):
        ro, rd = sc.rays()
        self.rays_ori = torch.from_numpy(ro).cuda()
        self.rays_dir = torch.from_numpy(rd).cuda()
        self.T_to_world = torch.from_numpy(np.asarray(c2w, np.float32))[None]
        self.intrinsics_OpenCVPinholeCameraModelParameters = dict(
            resolution=np.array([sc.width, sc.height]), shutter_type="GLOBAL", principal_point=np.array([sc.cx, sc.cy], np.float32),
            focal_length=np.array([sc.fx, sc.fy], np.float32), radial_coeffs=np.zeros(6, np.float32),
            tangential_coeffs=np.zeros(2, np.float32), thin_prism_coeffs=np.zeros(4, np.float32))


@pytest.mark.parametrize("half", [False, True])
def test_tracer_render_autograd_equals_trace_bwd(half):
    import threedgut_tracer

    sc = _scene("odd")
    feats = np.random.default_rng(3).uniform(-1.5, 1.5, (sc.n, 48)).astype(np.float32)
    tr = threedgut_tracer.Tracer(_conf(half))
    gs = _Gaussians(sc.particles, feats)
    batch = _Batch(sc, sc.camera(1, 5))
    out = tr.render(gs, batch)
    assert out["pred_features"].shape == (1, sc.height, sc.width, 24) and out["pred_opacity"].shape == (1, sc.height, sc.width, 1)
    rng = np.random.default_rng(6)
    gf = torch.from_numpy(rng.normal(size=(1, sc.height, sc.width, 24)).astype(np.float32)).cuda()
    go_ = torch.from_numpy(rng.normal(size=(1, sc.height, sc.width, 1)).astype(np.float32)).cuda()
    gd = torch.from_numpy((0.1 * rng.normal(size=(1, sc.height, sc.width, 1))).astype(np.float32)).cuda()
    ((out["pred_features"] * gf).sum() + (out["pred_opacity"] * go_).sum() + (out["pred_dist"] * gd).sum()).backward()
    # the same backward called directly
    sr = tr.tracer_wrapper
    sensor, poses = threedgut_tracer.Tracer._create_camera_parameters(batch)
    pd = torch.cat([gs.positions, gs.dns, gs.rot, gs.scl, torch.zeros_like(gs.dns)], 1).detach().contiguous()
    fa, dist, _, _ = sr.trace(0, 0, pd, gs.feats.detach(), batch.rays_ori, batch.rays_dir, None, sensor, 0, 1, poses.T_world_sensors[0],
                              poses.T_world_sensors[1])
    d_fa = torch.cat([gf[0], go_[0]], -1).contiguous()
    dp, df = sr.trace_bwd(0, 0, pd, gs.feats.detach(), batch.rays_ori, batch.rays_dir, None, sensor, 0, 1, poses.T_world_sensors[0],
                          poses.T_world_sensors[1], fa, d_fa, dist, gd[0].contiguous())
    assert torch.equal(fa, torch.cat([out["pred_features"][0], out["pred_opacity"][0]], -1))
    for got, want in ((gs.positions.grad, dp[:, 0:3]), (gs.dns.grad, dp[:, 3:4]), (gs.rot.grad, dp[:, 4:8]), (gs.scl.grad, dp[:, 8:11]),
                      (gs.feats.grad, df)):
        assert rel_l2(got.cpu().numpy(), want.cpu().numpy()) <= 1e-5  # float atomics: two backwards differ in the last bits


def test_fit_a_perturbed_scene_through_the_decoder():
    """Tracer.render -> FeatureDecoder -> L1 -> Adam over the Gaussians and the decoder: the loss falls at least 4x in 150 steps."""
    import feature_decoder as fdm
    import threedgut_tracer

    torch.manual_seed(0)
    sc = scenes.scene_c1(n=400, seed=13, width=64, height=64)
    rng = np.random.default_rng(13)
    feats = rng.uniform(-math.pi / 2, math.pi / 2, (sc.n, 48)).astype(np.float32)
    tr = threedgut_tracer.Tracer(_conf(False))
    dec = fdm.FeatureDecoder(24, hidden_dim=128, num_layers=2).cuda()
    batches = [_Batch(sc, sc.camera(i, 5)) for i in range(3)]
    target = _Gaussians(sc.particles, feats)
    with torch.no_grad():
        targets = []
        for b in batches:
            o = tr.render(target, b)
            targets.append(dec(o["pred_features"], b.rays_dir))
    pert = sc.particles.copy()
    pert[:, 0:3] += 0.03 * rng.normal(size=(sc.n, 3)).astype(np.float32)
    gs = _Gaussians(pert, feats + 0.5 * rng.normal(size=feats.shape).astype(np.float32))
    opt = torch.optim.Adam([{"params": gs.params(), "lr": 5e-3}, {"params": dec.parameters(), "lr": 1e-4}])
    losses = []
    for step in range(150):
        b = step % 3
        o = tr.render(gs, batches[b])
        rgb = dec(o["pred_features"], batches[b].rays_dir)
        loss = (rgb - targets[b]).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        with torch.no_grad():
            gs.dns.clamp_(0.01, 0.98)
            gs.scl.clamp_(min=1e-3)
        losses.append(loss.item())
    first, last = np.mean(losses[:3]), np.mean(losses[-3:])
    print(f"[fit] L1 {first:.4e} -> {last:.4e} ({first / last:.1f}x)")
    assert last * 4 <= first

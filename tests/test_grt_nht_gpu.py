"""NHT features through the CUDA 3DGRT path (grtb200_trace_nht / grtb200_trace_bwd_nht, Tracer with model.feature_type: nht) against the
float64 autograd oracle (tests/grt_nht_oracle.py) over the brute-force oracle's hit lists.

Bars (DESIGN.md sections 5, 13): features + alpha (25 channels) mean |diff| <= 1e-5, |diff| <= 1e-4 on all but max(3, 2e-4 P) rays,
max <= 2e-2; distance the same relative to the scene's distance scale; hit counts equal on >= 99.9 % of rays; gradients rel-L2 <= 1e-3
per tensor."""
import math

import numpy as np
import pytest

import scenes
from helpers import image_error_report, rel_l2
from oracle import gut_oracle as go

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import grt_nht_oracle as gno  # noqa: E402

MIN_T = 1e-3


def _nat():
    import b200_native

    return b200_native


def _scene(name):
    if name == "c1":
        return scenes.scene_c1(n=1000, seed=42, width=128, height=128)
    if name == "odd":
        return scenes.scene_c1(n=700, seed=5, width=75, height=53)
    return scenes.scene_c1(n=5000, seed=8, width=64, height=64)  # dense


def _setup(name, cam_i, deg, half, max_alpha=0.99, seed=0):
    sc = _scene(name)
    particles = sc.particles.copy()
    if max_alpha > 0.99:  # make hits reach the clamp: every 7th particle gets a density far above 1
        particles[::7, 3] = 3.0
    c2w = np.asarray(sc.camera(cam_i, 10), np.float32)
    feats = np.random.default_rng(seed).uniform(-math.pi / 2, math.pi / 2, (sc.n, 48)).astype(np.float32)
    if half:
        feats = feats.astype(np.float16).astype(np.float32)  # what the kernel reads
    ro, rd = sc.rays()
    cfg = go.grt_config()
    cfg.kernel_degree = deg
    cfg.max_alpha = max_alpha
    return sc, particles, feats, c2w, ro, rd, cfg


class _Gpu:
    """One native 3DGRT context, a BVH over the particles and the device buffers of a frame."""

    def __init__(self, particles, feats, c2w, ro, rd, deg, half, prim="instances", max_alpha=0.99):
        nat = _nat()
        c = nat.grt_default_config()
        c.kernel_degree, c.max_alpha, c.primitive = deg, max_alpha, nat.GRT_PRIMITIVES[prim]
        self.nat, self.ctx = nat, nat.GrtContext(c, 0)
        self.stream = torch.cuda.current_stream().cuda_stream
        self.n = int(particles.shape[0])
        self.p = torch.from_numpy(np.ascontiguousarray(particles if self.n else np.zeros((1, 12)), np.float32)).cuda()
        f = np.ascontiguousarray(feats if self.n else np.zeros((1, 48)), np.float32)
        self.f = torch.from_numpy(f).cuda().to(torch.float16 if half else torch.float32).contiguous()
        self.half = int(half)
        self.ro = torch.from_numpy(np.ascontiguousarray(ro, np.float32)).cuda()
        self.rd = torch.from_numpy(np.ascontiguousarray(rd, np.float32)).cuda()
        self.b, self.h, self.w = (int(v) for v in self.ro.shape[:3])
        self.R = self.b * self.h * self.w
        self.r2w = np.ascontiguousarray(np.asarray(c2w, np.float32)[:3, :4])
        self.ctx.build_bvh_packed(self.stream, self.n, self.p.data_ptr())

    def forward(self, fill=0.0):
        R, n = self.R, max(self.n, 1)
        self.feat, self.alpha = torch.full((R, 24), fill, device="cuda"), torch.full((R,), fill, device="cuda")
        self.dist, self.hits = torch.full((R, 2), fill, device="cuda"), torch.full((R,), fill, device="cuda")
        self.vis = torch.full((n,), fill, device="cuda")
        self.ctx.trace_nht(self.stream, self.n, self.p.data_ptr(), self.f.data_ptr(), 48, self.half, MIN_T, self.b, self.h, self.w,
                           self.ro.data_ptr(), self.rd.data_ptr(), self.r2w.ctypes.data, self.feat.data_ptr(), self.alpha.data_ptr(),
                           self.dist.data_ptr(), self.hits.data_ptr(), self.vis.data_ptr())
        torch.cuda.synchronize()
        return self

    def forward_sh(self, sph):
        R, n = self.R, max(self.n, 1)
        out = [torch.empty((R, 3), device="cuda"), torch.empty(R, device="cuda"), torch.empty((R, 2), device="cuda"),
               torch.empty(R, device="cuda"), torch.empty(n, device="cuda")]
        self.ctx.trace(self.stream, self.n, self.p.data_ptr(), sph.data_ptr(), 3, MIN_T, self.b, self.h, self.w, self.ro.data_ptr(),
                       self.rd.data_ptr(), self.r2w.ctypes.data, *[t.data_ptr() for t in out])
        torch.cuda.synchronize()
        return out

    def backward(self, d_feat, d_alpha, d_dist, fill=0.0):
        t = lambda a: torch.as_tensor(np.asarray(a, np.float32)).cuda().contiguous()  # noqa: E731
        d_feat, d_alpha, d_dist = t(d_feat).reshape(self.R, 24), t(d_alpha).reshape(self.R), t(d_dist).reshape(self.R)
        n = max(self.n, 1)
        dp, df = torch.full((n, 12), fill, device="cuda"), torch.full((n, 48), fill, device="cuda")
        self.ctx.trace_bwd_nht(self.stream, self.n, self.p.data_ptr(), self.f.data_ptr(), 48, self.half, MIN_T, self.b, self.h, self.w,
                               self.ro.data_ptr(), self.rd.data_ptr(), self.r2w.ctypes.data, self.feat.data_ptr(), self.alpha.data_ptr(),
                               self.dist.data_ptr(), d_feat.data_ptr(), d_alpha.data_ptr(), d_dist.data_ptr(), dp.data_ptr(), df.data_ptr())
        torch.cuda.synchronize()
        return dp.cpu().numpy()[: self.n], df.cpu().numpy()[: self.n]


def _grads(R, seed=1):
    rng = np.random.default_rng(seed)
    return (rng.normal(size=(R, 24)).astype(np.float32), rng.normal(size=R).astype(np.float32), (0.1 * rng.normal(size=R)).astype(np.float32))


FRAMES = [("c1", 1, 4, False, "instances", 0.99), ("c1", 6, 2, True, "icosahedron", 0.999), ("odd", 3, 2, False, "icosahedron", 0.99),
          ("odd", 0, 4, True, "instances", 0.999), ("dense", 0, 4, False, "instances", 0.999), ("dense", 3, 2, True, "icosahedron", 0.999)]


@pytest.mark.parametrize("name,cam_i,deg,half,prim,max_alpha", FRAMES)
def test_nht_matches_the_f64_oracle(name, cam_i, deg, half, prim, max_alpha):
    sc, particles, feats, c2w, ro, rd, cfg = _setup(name, cam_i, deg, half, max_alpha)
    tag = f"{name} cam{cam_i} deg{deg} {prim} {'fp16' if half else 'fp32'} max_alpha {max_alpha}"
    R = sc.width * sc.height
    d_feat, d_alpha, d_dist = _grads(R)
    ref = gno.frame(cfg, particles, feats, ro[0], rd[0], c2w, d_feat=d_feat, d_alpha=d_alpha, d_dist=d_dist, primitive=prim, device="cuda")
    if max_alpha > 0.99:
        clamped = int((ref["lists"]["alpha"] == np.float32(max_alpha)).sum())
        print(f"[parity] {tag}: {clamped} hits clamped at {max_alpha}")
        assert clamped > 0
    g = _Gpu(particles, feats, c2w, ro, rd, deg, half, prim, max_alpha).forward()
    got = np.concatenate([g.feat.cpu().numpy(), g.alpha.cpu().numpy()[:, None]], -1).reshape(sc.height, sc.width, 25)
    want = np.concatenate([ref["feat"], ref["alpha"][:, None]], -1).reshape(sc.height, sc.width, 25)
    mean, mx, bad = image_error_report(f"{tag} features+alpha", got, want)
    assert mean <= 1e-5 and mx <= 2e-2 and bad <= max(3, int(2e-4 * R)), (mean, mx, bad)
    scale = max(1.0, float(np.abs(ref["dist"][:, 0]).max()))
    mean, mx, bad = image_error_report(f"{tag} dist", g.dist.cpu().numpy()[:, :1].reshape(sc.height, sc.width, 1),
                                       ref["dist"][:, :1].reshape(sc.height, sc.width, 1), atol=1e-4 * scale)
    assert mean <= 1e-5 * scale and mx <= 2e-2 * scale and bad <= max(3, int(2e-4 * R)), (mean, mx, bad)
    assert (g.hits.cpu().numpy() == ref["hits"]).mean() >= 0.999
    dp, df = g.backward(d_feat, d_alpha, d_dist)
    for nm, a, b in (("d_pos", dp[:, 0:3], ref["dp"][:, 0:3]), ("d_density", dp[:, 3], ref["dp"][:, 3]), ("d_quat", dp[:, 4:8], ref["dp"][:, 4:8]),
                     ("d_scale", dp[:, 8:11], ref["dp"][:, 8:11]), ("d_features", df, ref["df"])):
        err = rel_l2(a, b)
        print(f"[parity] {tag} {nm}: rel-L2 {err:.2e}")
        assert err <= 1e-3, (nm, err)


def _grad_run(g, grads):
    g.forward()
    return g.backward(*grads)


@pytest.mark.parametrize("prim", ["instances", "icosahedron"])
def test_replay_overflow_and_retrace_give_the_same_gradients(monkeypatch, prim):
    """Replay, the re-trace of overflowed rays and the full re-trace.  Icosahedra: the same hits with the same per-ray arithmetic, only
    the order of the float atomics differs.  Instances: a hit whose t* lies before its box entry survives a query or not depending on
    where the query starts, which differs between the forward's chunks and the re-trace's (the SH path has the same ambiguity, and
    test_grt_parity_gpu.test_traversal_variants_give_the_same_image the same 1e-3 bar)."""
    sc, particles, feats, c2w, ro, rd, _ = _setup("odd", 1, 4, False)
    grads = _grads(sc.width * sc.height, 3)
    g = _Gpu(particles, feats, c2w, ro, rd, 4, False, prim)
    dp0, df0 = _grad_run(g, grads)
    assert int(g.hits.max().item()) > 4  # some lists overflow a capacity of 4
    monkeypatch.setenv("GRTB200_HITCAP", "4")
    dp1, df1 = _grad_run(g, grads)
    monkeypatch.delenv("GRTB200_HITCAP")
    g.ctx.set_replay(False)
    dp2, df2 = _grad_run(g, grads)
    errs = [rel_l2(a, b) for a, b in ((dp1, dp0), (df1, df0), (dp2, dp0), (df2, df0))]
    print(f"[paths] {prim} overflow / re-trace vs replay rel-L2: {errs}")
    assert max(errs) <= (1e-5 if prim == "icosahedron" else 1e-3)


def test_batch_of_two_images():
    sc, particles, feats, c2w, ro, rd, _ = _setup("odd", 2, 2, True)
    ro2 = np.concatenate([ro, ro], 0)
    rd2 = np.concatenate([rd, rd + 0.01 * np.random.default_rng(1).normal(size=rd.shape).astype(np.float32)], 0)
    R = sc.width * sc.height
    grads = _grads(2 * R, 4)
    g2 = _Gpu(particles, feats, c2w, ro2, rd2, 2, True)
    dp2, df2 = _grad_run(g2, grads)
    dps, dfs = [], []
    for i in range(2):
        g = _Gpu(particles, feats, c2w, ro2[i:i + 1], rd2[i:i + 1], 2, True)
        dp, df = _grad_run(g, tuple(x[i * R:(i + 1) * R] for x in grads))
        assert torch.equal(g.feat, g2.feat[i * R:(i + 1) * R]) and torch.equal(g.alpha, g2.alpha[i * R:(i + 1) * R])
        dps.append(dp)
        dfs.append(df)
    assert rel_l2(dp2, dps[0] + dps[1]) <= 1e-6 and rel_l2(df2, dfs[0] + dfs[1]) <= 1e-6


@pytest.mark.parametrize("prim", ["instances", "icosahedron"])
def test_alpha_dist_hits_visibility_equal_the_sh_trace(prim):
    sc, particles, feats, c2w, ro, rd, _ = _setup("c1", 2, 4, False, 0.999)
    g = _Gpu(particles, feats, c2w, ro, rd, 4, False, prim, 0.999).forward()
    rgb, alpha, dist, hits, vis = g.forward_sh(torch.from_numpy(sc.sph).cuda())
    for nm, a, b in (("alpha", g.alpha, alpha), ("dist", g.dist, dist), ("hits", g.hits, hits), ("visibility", g.vis, vis)):
        assert torch.equal(a, b), nm


def test_outputs_prefilled_with_nan_are_all_written_and_invisible_particles_get_zero_rows():
    sc, particles, feats, c2w, ro, rd, _ = _setup("odd", 1, 2, True)
    g = _Gpu(particles, feats, c2w, ro, rd, 2, True).forward(fill=float("nan"))
    for t in (g.feat, g.alpha, g.dist, g.hits, g.vis):
        assert not torch.isnan(t).any()
    dp, df = g.backward(*_grads(sc.width * sc.height, 2), fill=float("nan"))
    assert not np.isnan(dp).any() and not np.isnan(df).any()
    invisible = g.vis.cpu().numpy().view(np.int32) == 0
    assert invisible.sum() > 0 and (~invisible).sum() > 0
    assert np.abs(df[invisible]).max() == 0.0 and np.abs(dp[invisible]).max() == 0.0
    assert np.abs(df[~invisible]).max() > 0.0


@pytest.mark.parametrize("n", [0, 1])
def test_empty_and_single_particle_scenes(n):
    sc, particles, feats, c2w, ro, rd, cfg = _setup("odd", 0, 4, False)
    # the single particle: the one closest to the centre ray of the image, made large enough to cover part of it
    m = np.asarray(c2w, np.float64)
    d = m[:3, :3] @ rd[0, sc.height // 2, sc.width // 2]
    d /= np.linalg.norm(d)
    v = particles[:, 0:3] - m[:3, 3]
    near = int(np.argmin(np.linalg.norm(v - (v @ d)[:, None] * d, axis=1) + 1e3 * ((v @ d) < 1.0)))
    p, f = particles[near:near + n].copy(), feats[near:near + n]
    p[:, 8:11] = 0.5
    g = _Gpu(p, f, c2w, ro, rd, 4, False).forward(fill=float("nan"))
    grads = _grads(sc.width * sc.height, 5)
    dp, df = g.backward(*grads)
    if n == 0:
        assert float(g.feat.abs().max()) == 0 and float(g.alpha.abs().max()) == 0 and float(g.hits.max()) == 0
        assert dp.shape == (0, 12) and df.shape == (0, 48)
        return
    ref = gno.frame(cfg, p, f, ro[0], rd[0], c2w, *grads, device="cuda")
    assert ref["hits"].sum() > 20
    assert np.abs(g.feat.cpu().numpy() - ref["feat"]).max() <= 1e-4 and (g.hits.cpu().numpy() == ref["hits"]).mean() >= 0.999
    assert rel_l2(dp, ref["dp"]) <= 1e-3 and rel_l2(df, ref["df"]) <= 1e-3


def test_backward_after_a_forward_of_the_other_kind_retraces(monkeypatch):
    """The hit lists of the last forward are replayed only by a backward of the same kind; after a forward of the other kind the
    backward re-traces, so it equals a backward with the lists switched off (GRTB200_HITCAP=0) up to the order of the float atomics."""
    sc, particles, feats, c2w, ro, rd, _ = _setup("odd", 3, 2, False)
    grads = _grads(sc.width * sc.height, 6)
    g = _Gpu(particles, feats, c2w, ro, rd, 2, False)
    sph = torch.from_numpy(sc.sph).cuda()
    d_rgb = torch.from_numpy(grads[0][:, :3].copy()).cuda()
    d_a, d_d = torch.from_numpy(grads[1]).cuda(), torch.from_numpy(grads[2]).cuda()

    def sh_bwd(rgb, alpha, dist):
        dp, ds = torch.empty((g.n, 12), device="cuda"), torch.empty((g.n, 48), device="cuda")
        g.ctx.trace_bwd(g.stream, g.n, g.p.data_ptr(), sph.data_ptr(), 3, MIN_T, 1, g.h, g.w, g.ro.data_ptr(), g.rd.data_ptr(), g.r2w.ctypes.data,
                        rgb.data_ptr(), alpha.data_ptr(), dist.data_ptr(), d_rgb.data_ptr(), d_a.data_ptr(), d_d.data_ptr(), dp.data_ptr(),
                        ds.data_ptr())
        torch.cuda.synchronize()
        return dp.cpu().numpy(), ds.cpu().numpy()

    monkeypatch.setenv("GRTB200_HITCAP", "0")  # reference: both kinds re-trace
    dp0, df0 = _grad_run(g, grads)
    sh = g.forward_sh(sph)
    sdp0, sds0 = sh_bwd(*sh[:3])
    monkeypatch.delenv("GRTB200_HITCAP")
    g.forward()
    g.forward_sh(sph)  # the context's lists now belong to an SH forward
    dp1, df1 = g.backward(*grads)
    sh = g.forward_sh(sph)
    g.forward()  # ... and now to an NHT forward
    sdp1, sds1 = sh_bwd(*sh[:3])
    errs = [rel_l2(dp1, dp0), rel_l2(df1, df0), rel_l2(sdp1, sdp0), rel_l2(sds1, sds0)]
    print(f"[kinds] backward after the other kind vs re-trace rel-L2: {errs}")
    assert max(errs) <= 1e-6


def test_other_feature_dims_are_refused():
    sc, particles, feats, c2w, ro, rd, _ = _setup("odd", 0, 2, False)
    g = _Gpu(particles, feats, c2w, ro, rd, 2, False)
    g.forward()
    with pytest.raises(RuntimeError, match="feature_dim"):
        g.ctx.trace_nht(g.stream, g.n, g.p.data_ptr(), g.f.data_ptr(), 32, 0, MIN_T, 1, g.h, g.w, g.ro.data_ptr(), g.rd.data_ptr(),
                        g.r2w.ctypes.data, g.feat.data_ptr(), g.alpha.data_ptr(), g.dist.data_ptr(), g.hits.data_ptr(), g.vis.data_ptr())


def _conf(half):
    return {"model": {"feature_type": "nht", "nht_features": {"dim": 48, "activation": {"type": "sincos", "num_frequencies": 1},
                                                               "interpolation_type": "barycentric"}},
            "render": {"pipeline_type": "referenceSlang", "backward_pipeline_type": "referenceSlangBwd", "particle_kernel_max_alpha": 0.999,
                       "particle_feature_half": half, "min_transmittance": MIN_T}}


class _Gaussians:
    def __init__(self, particles, feats):
        p = torch.from_numpy(np.asarray(particles, np.float32)).cuda()
        self.positions = p[:, 0:3].clone().requires_grad_(True)
        self.density = p[:, 3:4].clone().requires_grad_(True)
        self.rotation = p[:, 4:8].clone().requires_grad_(True)
        self.scale = p[:, 8:11].clone().requires_grad_(True)
        self.feats = torch.from_numpy(np.asarray(feats, np.float32)).cuda().requires_grad_(True)
        self.n_active_features = 0
        ident = lambda t: t  # noqa: E731  (parameters here are already post-activation)
        self.rotation_activation = self.scale_activation = self.density_activation = ident

    def get_rotation(self):
        return self.rotation

    def get_scale(self):
        return self.scale

    def get_density(self):
        return self.density

    def get_features(self):
        return self.feats

    def params(self):
        return [self.positions, self.density, self.rotation, self.scale, self.feats]


class _Batch:
    def __init__(self, sc, c2w):
        ro, rd = sc.rays()
        self.rays_ori = torch.from_numpy(ro).cuda()
        self.rays_dir = torch.from_numpy(rd).cuda()
        self.T_to_world = torch.from_numpy(np.asarray(c2w, np.float32))[None].cuda()


@pytest.mark.parametrize("half", [False, True])
def test_tracer_render_autograd_equals_trace_bwd(half):
    import threedgrt_tracer

    sc = _scene("odd")
    feats = np.random.default_rng(3).uniform(-1.5, 1.5, (sc.n, 48)).astype(np.float32)
    tr = threedgrt_tracer.Tracer(_conf(half))
    gs = _Gaussians(sc.particles, feats)
    tr.build_acc(gs, rebuild=True)
    batch = _Batch(sc, sc.camera(1, 10))
    out = tr.render(gs, batch, train=True)
    assert out["pred_features"].shape == (1, sc.height, sc.width, 24) and out["pred_opacity"].shape == (1, sc.height, sc.width, 1)
    rng = np.random.default_rng(6)
    gf = torch.from_numpy(rng.normal(size=(1, sc.height, sc.width, 24)).astype(np.float32)).cuda()
    ga = torch.from_numpy(rng.normal(size=(1, sc.height, sc.width, 1)).astype(np.float32)).cuda()
    gd = torch.from_numpy((0.1 * rng.normal(size=(1, sc.height, sc.width, 1))).astype(np.float32)).cuda()
    ((out["pred_features"] * gf).sum() + (out["pred_opacity"] * ga).sum() + (out["pred_dist"] * gd).sum()).backward()
    ow = tr.tracer_wrapper
    pd = torch.cat([gs.positions, gs.density, gs.rotation, gs.scale, torch.zeros_like(gs.density)], 1).detach().contiguous()
    feat, alpha, hit, nrm, _, _ = ow.trace(0, batch.T_to_world, batch.rays_ori, batch.rays_dir, pd, gs.feats.detach(), 0, 0, MIN_T)
    assert torch.equal(feat, out["pred_features"]) and torch.equal(alpha, out["pred_opacity"])
    dp, df = ow.trace_bwd(0, batch.T_to_world, batch.rays_ori, batch.rays_dir, feat, alpha, hit, nrm, pd, gs.feats.detach(), gf, ga, gd,
                          None, 0, 0, MIN_T)
    for got, want in ((gs.positions.grad, dp[:, 0:3]), (gs.density.grad, dp[:, 3:4]), (gs.rotation.grad, dp[:, 4:8]),
                      (gs.scale.grad, dp[:, 8:11]), (gs.feats.grad, df)):
        assert rel_l2(got.cpu().numpy(), want.cpu().numpy()) <= 1e-5  # float atomics: two backwards differ in the last bits


def test_fit_a_perturbed_scene_through_the_decoder():
    """Tracer.render -> FeatureDecoder -> L1 -> Adam over the Gaussians and the decoder: the loss falls at least 4x in 150 steps."""
    import feature_decoder as fdm
    import threedgrt_tracer

    torch.manual_seed(0)
    sc = scenes.scene_c1(n=400, seed=13, width=64, height=64)
    rng = np.random.default_rng(13)
    feats = rng.uniform(-math.pi / 2, math.pi / 2, (sc.n, 48)).astype(np.float32)
    tr = threedgrt_tracer.Tracer(_conf(False))
    dec = fdm.FeatureDecoder(24, hidden_dim=128, num_layers=2).cuda()
    batches = [_Batch(sc, sc.camera(i, 10)) for i in range(3)]
    target = _Gaussians(sc.particles, feats)
    tr.build_acc(target)
    with torch.no_grad():
        targets = [dec(tr.render(target, b)["pred_features"], b.rays_dir) for b in batches]
    pert = sc.particles.copy()
    pert[:, 0:3] += 0.03 * rng.normal(size=(sc.n, 3)).astype(np.float32)
    gs = _Gaussians(pert, feats + 0.5 * rng.normal(size=feats.shape).astype(np.float32))
    opt = torch.optim.Adam([{"params": gs.params(), "lr": 5e-3}, {"params": dec.parameters(), "lr": 1e-4}])
    losses = []
    for step in range(150):
        b = step % 3
        tr.build_acc(gs)
        o = tr.render(gs, batches[b], train=True)
        loss = (dec(o["pred_features"], batches[b].rays_dir) - targets[b]).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        with torch.no_grad():
            gs.density.clamp_(0.01, 0.98)
            gs.scale.clamp_(min=1e-3)
        losses.append(loss.item())
    first, last = np.mean(losses[:3]), np.mean(losses[-3:])
    print(f"[fit] L1 {first:.4e} -> {last:.4e} ({first / last:.1f}x)")
    assert last * 4 <= first

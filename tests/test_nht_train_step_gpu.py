"""The NHT training steps (train_step_nht.GaussianTrainStepNHT on 3DGUT, GaussianTrainStepGRTNHT on 3DGRT) and the device code they add:
one step against Tracer.render -> FeatureDecoder -> composite / mask -> L1 + SSIM -> regularisers -> autograd, the fused NHT Adam
against torch.optim.Adam, the tracers' trace_bwd(out=...) with NHT features, fits with and without MCMC densification, colour refinement
and two ranks."""
import math
import os

import numpy as np
import pytest

from helpers import rel_l2
from test_grt_train_step_gpu import _free_port, _setup
from test_loss_terms_step_gpu import _ImageLoss
from test_nht_train_step import _einsum_dirs
from train_step import raw_params

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

LRS = dict(positions=2e-3, density=0.05, rotation=1e-3, scale=5e-3, features=2e-2, decoder=1e-3)
GEOMETRY = ("positions", "density", "rotation", "scale")


def _conf(half=False, **top):
    # the 3DGRT tracer takes NHT features through the Slang pipelines only (the *_3dgrt_mcmc_nht apps); 3DGUT does not read these keys
    return {"model": {"feature_type": "nht", "nht_features": {"dim": 48, "activation": {"type": "sincos", "num_frequencies": 1},
                                                               "interpolation_type": "barycentric"}},
            "render": {"particle_feature_half": half, "pipeline_type": "referenceSlang", "backward_pipeline_type": "referenceSlangBwd"}, **top}


def _decoder(seed=0):
    import feature_decoder as fdm

    torch.manual_seed(seed)
    return fdm.FeatureDecoder(24, hidden_dim=128, num_layers=3, sh_scale=3.0).cuda()  # the shipped net (configs/base_gs.yaml)


class _Harness:
    """C1, 600 Gaussians, 96x96, 6 views, random NHT features, through either NHT step."""

    def __init__(self, kind, half=False):
        import scenes

        self.kind, self.half = kind, half
        self.sc, self.rays_o, self.rays_d, self.P, _, self.poses = _setup()
        self.dev = self.P.device
        self.H, self.W = self.sc.height, self.sc.width
        rng = np.random.default_rng(5)
        self.F = torch.from_numpy(rng.uniform(-math.pi / 2, math.pi / 2, (self.sc.n, 48)).astype(np.float32)).to(self.dev)
        sc = self.sc
        self.sensor = sc.pinhole_sensor()
        self.views = [scenes.pose7_from_c2w(sc.camera(i, 6)) for i in range(6)]

    def make(self, raw, decoder, conf=None, **kw):
        import train_step_nht as tsn

        cls = tsn.GaussianTrainStepNHT if self.kind == "gut" else tsn.GaussianTrainStepGRTNHT
        return cls(raw, LRS, decoder, conf if conf is not None else _conf(self.half), **kw)

    def step(self, st, v, target, mask=None, **kw):
        if self.kind == "gut":
            return st.step(self.rays_o, self.rays_d, self.sensor, self.views[v], target, mask=mask, **kw)
        return st.step(self.rays_o, self.rays_d, self.poses[v], target, mask=mask, **kw)

    def render(self, st, v):
        if self.kind == "gut":
            return st.render(self.rays_o, self.rays_d, self.sensor, self.views[v])
        return st.render(self.rays_o, self.rays_d, self.poses[v])

    def autograd_render(self, leaves, v):
        """Tracer.render's autograd node on the activated raw leaves: (features [1,H,W,24], alpha [H,W,1])."""
        act = (leaves["positions"], torch.nn.functional.normalize(leaves["rotation"]), torch.exp(leaves["scale"]), torch.sigmoid(leaves["density"]))
        if self.kind == "gut":
            from threedgut_tracer.tracer import SensorPose3D, SplatRaster, Tracer

            pose = self.views[v]
            out, _, _, _ = Tracer._Autograd.apply(SplatRaster(_conf(self.half)), 0, 0, self.rays_o, self.rays_d, *act, leaves["features"],
                                                  self.sensor, SensorPose3D(T_world_sensors=[pose, pose], timestamps_us=[0, 1]))
            out = out.reshape(self.H, self.W, 25)
            return out[None, ..., :24], out[..., 24:]
        import threedgrt_tracer

        tracer = threedgrt_tracer.Tracer(_conf(self.half))
        ot = tracer.tracer_wrapper
        ot.set_replay(True, self.dev)
        pos, rot, scl, dns = act
        ot.build_bvh(pos.detach().contiguous(), rot.detach().contiguous(), scl.detach().contiguous(), dns.detach().contiguous())
        feat, alpha, _, _, _, _ = threedgrt_tracer.Tracer._Autograd.apply(ot, 0, self.poses[v], self.rays_o, self.rays_d, pos, rot, scl, dns,
                                                                         leaves["features"], 0, 0, tracer._min_transmittance)
        return feat, alpha[0]

    def c2w(self, v):
        return np.asarray(self.sc.camera(v, 6), np.float32)


def _step_against_autograd(hz, composite):
    import feature_decoder as fdm

    H, W, dev = hz.H, hz.W, hz.dev
    weights, lo, ls = ((0.8, 0.2), 0.01, 0.02) if composite else ((1.0, 0.0), 0.0, 0.0)
    dec = _decoder()
    params0 = dec.network.params.detach().clone()
    raw = raw_params(hz.P, features=hz.F)
    kw = dict(background="white", lambda_opacity=lo, lambda_scale=ls) if composite else {}
    st = hz.make({k: v.clone() for k, v in raw.items()}, dec, lambda_l1=weights[0], lambda_ssim=weights[1], **kw)
    gen = torch.Generator(device=dev).manual_seed(3)
    target = (torch.rand((H, W, 3), device=dev, generator=gen) * 0.8).contiguous()
    mask = (torch.rand((H, W), device=dev, generator=gen) > 0.25).float() if composite else None
    got_loss = float(hz.step(st, 1, target, mask=mask))

    def autograd(dirs):
        leaves = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
        dparams = params0.clone().requires_grad_(True)
        feats, alpha = hz.autograd_render(leaves, 1)
        x = fdm.decode(feats.reshape(-1, 24), dirs, dparams, dec.config).reshape(H, W, 3)
        y = target
        if composite:
            x = x + 1.0 * (1.0 - alpha)                       # apply_background after the decoder (utils/render.py), white
            x, y = x * mask[..., None], y * mask[..., None]   # trainer.py:693-694
        loss = _ImageLoss.apply(torch.cat([x, torch.zeros_like(alpha)], -1), y, *weights)
        loss = loss + lo * torch.sigmoid(leaves["density"]).abs().mean() + ls * torch.exp(leaves["scale"]).abs().mean()
        loss.backward()
        grads = {k: leaves[k].grad.cpu().numpy() for k in raw}
        grads["decoder"] = dparams.grad.cpu().numpy()
        return grads, float(loss.detach())

    import train_step_nht as tsn

    dirs = _einsum_dirs(hz.c2w(1), hz.rays_d.cpu()).to(dev)
    want, want_loss = autograd(dirs)
    again, _ = autograd(dirs)
    # the 3DGUT step has only the world -> sensor pose: its R_c2w comes from the pose's quaternion and differs from the camera-to-world
    # matrix in the last bits; the reference run on those directions shows how far that alone moves the gradients
    R = tsn.c2w_rotation_from_pose7(hz.views[1]) if hz.kind == "gut" else tsn.c2w_rotation_from_T(hz.poses[1])
    alt, _ = autograd(tsn.world_ray_directions(R, hz.rays_d))
    one_minus_b1 = float(np.float32(1) - np.float32(0.9))
    got = {k: st.optimizer.exp_avg[k].cpu().numpy() / one_minus_b1 for k in raw}
    got["decoder"] = st.optimizer.decoder_exp_avg.cpu().numpy() / one_minus_b1
    errs, floor = {}, {}
    for k in want:
        assert float(np.abs(want[k]).max()) > 0, k
        errs[k] = rel_l2(got[k], want[k])
        floor[k] = max(rel_l2(again[k], want[k]), rel_l2(alt[k], want[k]))
    return errs, floor, got_loss, want_loss


@pytest.mark.parametrize("kind,half,composite", [("gut", False, True), ("gut", True, True), ("gut", False, False),
                                                 ("grt", False, True), ("grt", True, True), ("grt", False, False)])
def test_one_step_matches_autograd(kind, half, composite):
    errs, floor, got_loss, want_loss = _step_against_autograd(_Harness(kind, half), composite)
    assert abs(got_loss - want_loss) <= 1e-5 * max(1.0, abs(want_loss)), (got_loss, want_loss)
    for k, err in errs.items():
        # `floor`: how far the reference moves by itself -- run twice (the renderers' backwards sum with float atomics) and run on the
        # step's own ray directions, which equal apply_feature_decoder's to ~1e-7.  The decoder encodes the directions in fp16, so such a
        # last-bit change can flip roundings of the encoding; with fp16 features the 3DGUT position gradient of this scene is sensitive
        # enough to that to pass 1e-5 on its own.  The step must be as close to the reference as the reference is to itself.
        bar = max(1e-5, 2.0 * floor[k])
        print(f"[nht step] {kind} {'fp16' if half else 'fp32'} {'composited+masked+reg' if composite else 'L1'} {k}: exp_avg / (1 - b1) "
              f"vs autograd rel-L2 {err:.2e} (reference vs itself {floor[k]:.2e}, bar {bar:.2e})")
        assert err <= bar, k


# ---------------------------------------------------------------------------------------------------------------------------------
# the fused NHT Adam against torch.optim.Adam


def _raw_grads(leaves, dp, lo, ls):
    """Autograd of the activations: the raw-parameter gradients of <record, d_particles> (+ the regularisers)."""
    import train_step

    rec = {k: v.detach().clone().requires_grad_(True) for k, v in leaves.items() if k in GEOMETRY}
    obj = (train_step.particle_record(rec) * dp).sum() + lo * torch.sigmoid(rec["density"]).mean() + ls * torch.exp(rec["scale"]).mean()
    obj.backward()
    return {k: rec[k].grad for k in GEOMETRY}


@pytest.mark.parametrize("selective,reg", [(False, False), (True, False), (False, True), (True, True)])
def test_fused_nht_adam_matches_torch_adam(selective, reg):
    import optimizers

    dev = torch.device("cuda", 0)
    n, n_dec, wd = 4099, 40960, 1e-3
    g = torch.Generator(device=dev).manual_seed(2)
    leaves = {"positions": torch.randn(n, 3, device=dev, generator=g), "density": torch.randn(n, 1, device=dev, generator=g),
              "rotation": torch.randn(n, 4, device=dev, generator=g), "scale": torch.randn(n, 3, device=dev, generator=g) - 3,
              "features": torch.randn(n, 48, device=dev, generator=g)}
    dec = torch.randn(n_dec, device=dev, generator=g) * 0.05
    ref = {k: torch.nn.Parameter(v.clone()) for k, v in leaves.items()}
    ref_dec = torch.nn.Parameter(dec.clone())
    # The kernel takes the betas as fp32 and forms 1 - beta in fp32 (1 - 0.999f = 0.00099998713...); torch forms it in double from the
    # Python float.  Handing torch the fp32 values of the betas gives both the same hyper-parameters (1 - b is exact in either precision).
    b1, b2 = float(np.float32(0.9)), float(np.float32(0.999))
    opt = optimizers.FusedNHTAdam({k: v.clone() for k, v in leaves.items()}, dec.clone(), LRS, betas=(b1, b2), eps=1e-15, selective=selective,
                                  decoder_betas=(b1, b2), decoder_weight_decay=wd)
    torch_g = torch.optim.Adam([{"params": [ref[k]], "lr": LRS[k]} for k in optimizers.NHT_GROUPS], betas=(b1, b2), eps=1e-15)
    torch_d = torch.optim.Adam([ref_dec], lr=LRS["decoder"], betas=(b1, b2), eps=1e-8, weight_decay=wd)
    ms = {k: torch.zeros_like(v) for k, v in leaves.items()}
    vs = {k: torch.zeros_like(v) for k, v in leaves.items()}
    lo, ls = (0.3, 0.2) if reg else (0.0, 0.0)
    for t in range(3):
        dp = torch.randn(n, 12, device=dev, generator=g)
        df = torch.randn(n, 48, device=dev, generator=g)
        dd = torch.randn(n_dec, device=dev, generator=g) * 1e-2
        vis = (torch.rand(n, device=dev, generator=g) > 0.3).float()
        grads = _raw_grads(opt.params, dp, lo, ls)
        grads["features"] = df
        opt.step(dp, df, dd, visibility=vis if selective else None, lambda_opacity=lo, lambda_scale=ls)
        if selective:  # the reference plugin's rule: no bias correction, visible rows only (optimizers.cu:49-83)
            with torch.no_grad():
                for k in optimizers.NHT_GROUPS:
                    rows = vis.bool()
                    gk = grads[k]
                    ms[k][rows] = b1 * ms[k][rows] + (1 - b1) * gk[rows]
                    vs[k][rows] = b2 * vs[k][rows] + (1 - b2) * gk[rows] * gk[rows]
                    ref[k].data[rows] -= LRS[k] * ms[k][rows] / (vs[k][rows].sqrt() + 1e-15)
        else:
            for k in optimizers.NHT_GROUPS:
                ref[k].grad = grads[k].clone()
            torch_g.step()
        ref_dec.grad = dd.clone()
        torch_d.step()
    torch.cuda.synchronize()
    for k in optimizers.NHT_GROUPS:
        m = ms[k] if selective else torch_g.state[ref[k]]["exp_avg"]
        v = vs[k] if selective else torch_g.state[ref[k]]["exp_avg_sq"]
        for what, a, b in (("param", opt.params[k], ref[k].detach()), ("exp_avg", opt.exp_avg[k], m), ("exp_avg_sq", opt.exp_avg_sq[k], v)):
            err = rel_l2(a.cpu().numpy(), b.cpu().numpy())
            assert err <= 1e-6, (k, what, err)
    st = torch_d.state[ref_dec]
    for what, a, b in (("param", opt.decoder_params, ref_dec.detach()), ("exp_avg", opt.decoder_exp_avg, st["exp_avg"]),
                       ("exp_avg_sq", opt.decoder_exp_avg_sq, st["exp_avg_sq"])):
        err = rel_l2(a.cpu().numpy(), b.cpu().numpy())
        assert err <= 1e-6, ("decoder", what, err)


def test_frozen_groups_are_untouched_bit_for_bit():
    import optimizers

    dev = torch.device("cuda", 0)
    n = 1001
    g = torch.Generator(device=dev).manual_seed(4)
    leaves = {k: torch.randn(n, w, device=dev, generator=g) for k, w in zip(optimizers.NHT_GROUPS, optimizers.NHT_WIDTHS)}
    opt = optimizers.FusedNHTAdam(leaves, torch.randn(40960, device=dev, generator=g), LRS)
    step = lambda **kw: opt.step(torch.randn(n, 12, device=dev, generator=g), torch.randn(n, 48, device=dev, generator=g),  # noqa: E731
                                 torch.randn(40960, device=dev, generator=g), **kw)
    step()
    before = {k: (opt.params[k].clone(), opt.exp_avg[k].clone(), opt.exp_avg_sq[k].clone()) for k in optimizers.NHT_GROUPS}
    dec_before = opt.decoder_params.clone()
    for _ in range(3):
        step(frozen=GEOMETRY, lambda_opacity=0.5)
    for k in GEOMETRY:
        for a, b in zip(before[k], (opt.params[k], opt.exp_avg[k], opt.exp_avg_sq[k])):
            assert torch.equal(a, b), k
        assert opt.steps[k] == 1
    assert not torch.equal(before["features"][0], opt.params["features"]) and not torch.equal(dec_before, opt.decoder_params)
    assert opt.steps["features"] == opt.steps["decoder"] == 4
    step(frozen=("decoder",))
    assert opt.steps["decoder"] == 4 and opt.steps["positions"] == 2


# ---------------------------------------------------------------------------------------------------------------------------------
# trace_bwd(out=...) with NHT features


@pytest.mark.parametrize("kind", ["gut", "grt"])
def test_trace_bwd_into_out_equals_the_plain_call(kind):
    import view_parallel

    hz = _Harness(kind)
    dev = hz.dev
    raw = raw_params(hz.P, features=hz.F)
    st = hz.make(raw, _decoder())
    particles, feats = st.activated()
    g = torch.Generator(device=dev).manual_seed(8)
    ex = view_parallel.FlatGradientExchange(hz.sc.n, dev, tail=7)
    if kind == "gut":
        r = st.raster
        out, dst, _, _ = r.trace(0, 0, particles, feats, hz.rays_o, hz.rays_d, None, hz.sensor, 0, 1, hz.views[2], hz.views[2])
        d_out = torch.randn(out.shape, device=dev, generator=g)
        d_dist = torch.randn(dst.shape, device=dev, generator=g) * 0.1
        args = (0, 0, particles, feats, hz.rays_o, hz.rays_d, None, hz.sensor, 0, 1, hz.views[2], hz.views[2], out, d_out, dst, d_dist)
        plain = r.trace_bwd(*args)
        into = r.trace_bwd(*args, out=ex.out())
    else:
        ot = st.tracer.tracer_wrapper
        ot.build_bvh_packed(particles)
        feat, alpha, dst, nrm, _, _ = ot.trace(0, hz.poses[2], hz.rays_o, hz.rays_d, particles, feats, 0, 0, 0.001)
        gf = torch.randn(feat.shape, device=dev, generator=g)
        ga = torch.randn(alpha.shape, device=dev, generator=g)
        args = (0, hz.poses[2], hz.rays_o, hz.rays_d, feat, alpha, dst, nrm, particles, feats, gf, ga, torch.zeros_like(alpha),
                torch.zeros_like(nrm), 0, 0, 0.001)
        plain = ot.trace_bwd(*args)
        into = ot.trace_bwd(*args, out=ex.out())
    assert into[0].data_ptr() == ex.d_particles.data_ptr() and into[1].data_ptr() == ex.d_sph.data_ptr()
    for a, b in zip(plain, into):
        assert float(a.abs().max()) > 0
        assert rel_l2(b.cpu().numpy(), a.cpu().numpy()) <= 1e-5  # float atomics: two backwards differ in the last bits


# ---------------------------------------------------------------------------------------------------------------------------------
# fits


FIT_LRS = dict(positions=5e-3, density=0.05, rotation=1e-3, scale=5e-3, features=5e-3, decoder=1e-4)
FIT_VIEWS = 3


def _fit_decoder():
    import feature_decoder as fdm

    torch.manual_seed(0)
    return fdm.FeatureDecoder(24, hidden_dim=128, num_layers=2).cuda()  # the net of test_nht_render_gpu.py's autograd fit


def _targets(hz, dec, views=6):
    truth = hz.make(raw_params(hz.P, features=hz.F), dec)
    return [hz.render(truth, v)[0].clone() for v in range(views)]


def _perturbed(hz):
    rng = np.random.default_rng(13)
    P2 = hz.P.clone()
    P2[:, 0:3] += torch.from_numpy(0.03 * rng.normal(size=(hz.sc.n, 3)).astype(np.float32)).to(hz.dev)
    F2 = hz.F + torch.from_numpy(0.5 * rng.normal(size=(hz.sc.n, 48)).astype(np.float32)).to(hz.dev)
    return raw_params(P2, features=F2)


def _mean_l1(hz, st, targets):
    return float(np.mean([float((hz.render(st, v)[0] - t).abs().mean()) for v, t in enumerate(targets)]))


@pytest.mark.parametrize("kind", ["gut", "grt"])
@pytest.mark.parametrize("mcmc", [False, True])
def test_fit_a_perturbed_scene(kind, mcmc, monkeypatch):
    import densify

    monkeypatch.setitem(globals(), "LRS", FIT_LRS)
    hz = _Harness(kind)
    targets = _targets(hz, _fit_decoder(), FIT_VIEWS)
    kw = {}
    if mcmc:
        kw["densify_conf"] = densify.MCMCConfig(relocate_start=5, relocate_frequency=20, add_start=5, add_frequency=20, perturb_start=0,
                                                noise_lr=5e3, seed=2)
    fit = hz.make(_perturbed(hz), _fit_decoder(), **kw)
    n0, ex0 = fit.n, fit.exchange
    before = _mean_l1(hz, fit, targets)
    for it in range(90):
        hz.step(fit, it % FIT_VIEWS, targets[it % FIT_VIEWS])
    after = _mean_l1(hz, fit, targets)
    print(f"[nht fit] {kind} {'mcmc' if mcmc else 'plain'}: N {n0} -> {fit.n}, mean L1 over {FIT_VIEWS} views {before:.5f} -> {after:.5f} "
          f"({before / after:.1f}x) after 90 steps")
    # plain: the bar of test_nht_render_gpu.py's fit; with MCMC the Gaussians relocated and added every 20 steps start from zero moments
    assert np.isfinite(after) and after * (2 if mcmc else 4) <= before
    if mcmc:
        assert fit.n > n0 and fit.exchange is not ex0 and fit.exchange.n == fit.n
        assert fit.exchange.d_tail.numel() == fit.decoder.network.params.numel()


# ---------------------------------------------------------------------------------------------------------------------------------
# colour refinement


@pytest.mark.parametrize("kind", ["gut", "grt"])
def test_color_refinement_freezes_the_geometry(kind):
    import densify

    hz = _Harness(kind)
    conf = _conf(n_iterations=5, model={**_conf()["model"], "nht_decoder": {"color_refine_steps": 5}})
    gen = torch.Generator(device=hz.dev).manual_seed(6)
    target = (torch.rand((hz.H, hz.W, 3), device=hz.dev, generator=gen) * 0.8).contiguous()
    mcmc = densify.MCMCConfig(relocate_start=0, relocate_frequency=1, add_start=0, add_frequency=1, perturb_start=0, noise_lr=5e3, seed=2)
    st = hz.make(raw_params(hz.P, features=hz.F), _decoder(), conf=conf, lambda_opacity=0.01, lambda_scale=0.01, densify_conf=mcmc)
    plain = hz.make(raw_params(hz.P, features=hz.F), _decoder(), conf=conf)
    assert st.color_refine_start == 0
    geo = {k: st.params[k].clone() for k in GEOMETRY}
    feats, dec = st.params["features"].clone(), st.decoder.network.params.detach().clone()
    n0 = st.n
    for it in range(5):
        loss = float(hz.step(st, it, target))
        if it == 0:
            want = float(hz.step(plain, it, target))
            assert abs(loss - want) <= 1e-6 * max(1.0, abs(want)), (loss, want)  # no regulariser while refining
    assert st.n == n0
    for k in GEOMETRY:
        assert torch.equal(st.params[k], geo[k]), k
        assert not st.optimizer.exp_avg[k].any() and not st.optimizer.exp_avg_sq[k].any(), k
    assert not torch.equal(st.params["features"], feats) and not torch.equal(st.decoder.network.params.detach(), dec)


# ---------------------------------------------------------------------------------------------------------------------------------
# two ranks


def _rank_worker(rank, world, port, out_dir):
    import torch.distributed as dist

    import view_parallel as vp

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        hz = _Harness("grt")
        targets = torch.from_numpy(np.load(os.path.join(out_dir, "targets.npy"))).to(hz.dev)
        fit = hz.make(_perturbed(hz), _decoder(), selective=True, background="random")
        for it in range(10):
            views = [vp.views_for_rank(it, r, world, 6)[0] for r in range(world)]
            positions = np.stack([fit.sensor_position(hz.poses[v]) for v in views])
            hz.step(fit, views[rank], targets[views[rank]], all_sensor_positions=positions)
        torch.cuda.synchronize()
        np.savez(os.path.join(out_dir, f"rank{rank}.npz"), decoder=fit.decoder.network.params.detach().cpu().numpy(),
                 **{k: v.detach().cpu().numpy() for k, v in fit.params.items()})
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_stay_bit_identical(tmp_path):
    import torch.multiprocessing as mp

    hz = _Harness("grt")
    np.save(tmp_path / "targets.npy", torch.stack(_targets(hz, _decoder())).cpu().numpy())
    mp.spawn(_rank_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    outs = [np.load(tmp_path / f"rank{r}.npz") for r in range(2)]
    for k in outs[0].files:
        assert np.array_equal(outs[0][k], outs[1][k]), k

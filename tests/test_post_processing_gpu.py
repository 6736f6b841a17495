"""The linear-to-sRGB post-processing (post_processing.method: linear-to-srgb) on the GPU: the loss entry against the float64 oracle
(tests/post_processing_oracle.py) on both layouts, every background mode, with and without a mask and SSIM; post_processing=None bit for
bit the existing entries; one step of each of the five training steps against autograd of the reference chain (render -> background ->
linear_to_srgb -> mask -> L1 + SSIM); and fits to sRGB-encoded targets through 3DGUT and 3DGRT."""
import numpy as np
import pytest

import post_processing_oracle as ppo
from helpers import rel_l2
from train_step import raw_params

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

POST = "linear-to-srgb"
BACKGROUNDS = ("black", "white", "image")


def _case(h, w, background, masked, seed):
    """Linear radiance (dark values on the linear branch of the encode, a few HDR values above 1) against an sRGB target."""
    rng = np.random.default_rng(seed)
    y = rng.uniform(0, 1, (h, w, 3)).astype(np.float32)
    rgb = (1.2 * rng.uniform(0, 1, (h, w, 3)) ** 2.2 - 0.002).astype(np.float32)
    alpha = rng.uniform(0.05, 1.0, (h, w, 1)).astype(np.float32)
    bg = {"black": None, "white": (1.0, 1.0, 1.0), "image": rng.uniform(0, 1, (h, w, 3)).astype(np.float32)}[background]
    m = (rng.uniform(size=(h, w)) > 0.3).astype(np.float32) if masked else None
    return rgb, alpha, y, bg, m


def _dev(a, dev):
    return None if a is None else (torch.from_numpy(np.ascontiguousarray(a)).to(dev) if isinstance(a, np.ndarray) else a)


def _run(layout, rgb, alpha, y, bg, m, weights, dev, post=POST):
    import losses

    t_rgb, t_alpha, t_y, t_bg, t_m = (_dev(a, dev) for a in (rgb, alpha, y, bg, m))
    if layout == 4:
        loss, _, _, d = losses.image_loss(torch.cat([t_rgb, t_alpha], -1).contiguous(), t_y, *weights, background=t_bg, mask=t_m,
                                          post_processing=post)
        return float(loss), d[..., :3].cpu().numpy(), d[..., 3:].cpu().numpy()
    loss, _, _, d_rgb, d_alpha = losses.image_loss_rgb_alpha(t_rgb, t_alpha, t_y, *weights, background=t_bg, mask=t_m, post_processing=post)
    return float(loss), d_rgb.cpu().numpy(), d_alpha.cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------------------
# the loss entry


@pytest.mark.parametrize("size", [(96, 96), (61, 97)])
@pytest.mark.parametrize("layout", [4, 3])
@pytest.mark.parametrize("background", BACKGROUNDS)
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("lambda_ssim", [0.0, 0.2])
def test_loss_matches_the_float64_oracle(size, layout, background, masked, lambda_ssim):
    h, w = size
    dev = torch.device("cuda", 0)
    rgb, alpha, y, bg, m = _case(h, w, background, masked, seed=h * 100 + w + 7 * BACKGROUNDS.index(background) + 3 * masked)
    weights = (1.0 - lambda_ssim, lambda_ssim)
    loss, d_rgb, d_alpha = _run(layout, rgb, alpha, y, bg, m, weights, dev)
    r_loss, r_rgb, r_alpha = ppo.loss_and_gradients(rgb, alpha, y, *weights, background=bg, mask=m)
    e_rgb = rel_l2(d_rgb, r_rgb)
    e_alpha = rel_l2(d_alpha, r_alpha) if background != "black" else 0.0
    print(f"[post] {size} layout {layout} {background} mask {masked} ssim {lambda_ssim}: loss {loss:.7f} vs {r_loss:.7f}, "
          f"d_rgb rel-L2 {e_rgb:.2e}, d_alpha rel-L2 {e_alpha:.2e}")
    assert abs(loss - r_loss) <= 1e-5 * abs(r_loss)
    assert e_rgb <= 1e-5 and e_alpha <= 1e-5
    if background == "black":
        assert not d_alpha.any()


def test_none_is_bit_identical_to_the_existing_entries():
    import ctypes

    import b200_native as nat
    import losses

    dev = torch.device("cuda", 0)
    lib = nat.load()
    stream = torch.cuda.current_stream(dev).cuda_stream
    h, w = 61, 97
    for background in BACKGROUNDS:
        for masked in (False, True):
            rgb, alpha, y, bg, m = _case(h, w, background, masked, seed=5)
            t_rgb, t_alpha, t_y, t_bg, t_m = (_dev(a, dev) for a in (rgb, alpha, y, bg, m))
            rgba = torch.cat([t_rgb, t_alpha], -1).contiguous()
            # the Python entries: post_processing=None runs exactly the launches they ran before
            # (the gradients are deterministic; the loss terms are sums of per-block atomics in any order: within the 1e-6 of the loss tests)
            a = losses.image_loss(rgba, t_y, 0.8, 0.2, background=t_bg, mask=t_m)
            b = losses.image_loss(rgba, t_y, 0.8, 0.2, background=t_bg, mask=t_m, post_processing=None)
            assert torch.equal(a[3], b[3]) and abs(float(a[0]) - float(b[0])) <= 1e-6
            want = {4: b}
            a = losses.image_loss_rgb_alpha(t_rgb, t_alpha, t_y, 0.8, 0.2, background=t_bg, mask=t_m)
            b = losses.image_loss_rgb_alpha(t_rgb, t_alpha, t_y, 0.8, 0.2, background=t_bg, mask=t_m, post_processing=None)
            assert torch.equal(a[3], b[3]) and torch.equal(a[4], b[4]) and abs(float(a[0]) - float(b[0])) <= 1e-6
            want[3] = b
            # the C entry called directly with post_processing 0 against what losses.* returned above, both layouts
            bg_rgb = (ctypes.c_float * 3)(*bg) if isinstance(bg, tuple) else None
            bg_img = t_bg.data_ptr() if isinstance(t_bg, torch.Tensor) else None
            mask = None if t_m is None else t_m.data_ptr()
            for layout, pred in ((4, rgba), (3, t_rgb)):
                scratch = torch.empty(int(lib.gutb200_image_loss_scratch_bytes(h, w)) // 4 + 1, device=dev)
                d = torch.empty((h, w, layout), device=dev)
                d_alpha = torch.empty((h, w, 1), device=dev)
                sums = torch.empty(2, device=dev)
                rc = lib.gutb200_image_loss(stream, h, w, layout, pred.data_ptr(), None if layout == 4 else t_alpha.data_ptr(), t_y.data_ptr(),
                                            bg_rgb, bg_img, mask, 0.8, 0.2, scratch.data_ptr(), d.data_ptr(),
                                            None if layout == 4 else d_alpha.data_ptr(), sums.data_ptr(), 0)
                assert rc == 0
                assert torch.equal(d, want[layout][3]), (background, masked, layout)
                means = torch.tensor([3.0 * h * w, 3.0 * (h - 10) * (w - 10)], device=dev)   # l1 and ssim of the sums
                l1_ssim = torch.stack([want[layout][1], want[layout][2]]).to(torch.float32)
                assert float((sums / means - l1_ssim).abs().max()) <= 1e-6, (background, masked, layout)
                if layout == 3:
                    assert torch.equal(d_alpha, want[layout][4]), (background, masked, layout)


def test_rgb_entry_and_refusals():
    import b200_native as nat
    import losses

    dev = torch.device("cuda", 0)
    rgb, alpha, y, _, _ = _case(40, 56, "black", False, seed=2)
    t_rgb, t_alpha, t_y = (_dev(a, dev) for a in (rgb, alpha, y))
    # image_loss_rgb (no alpha) with the encode is the split entry on black: the alpha is never read
    a = losses.image_loss_rgb(t_rgb, t_y, 0.8, 0.2, post_processing=POST)
    b = losses.image_loss_rgb_alpha(t_rgb, t_alpha, t_y, 0.8, 0.2, post_processing=POST)
    assert torch.equal(a[3], b[3]) and abs(float(a[0]) - float(b[0])) <= 1e-6 and not bool(b[4].any())
    for method in ("ppisp", "srgb"):
        for call in (lambda: losses.image_loss(torch.cat([t_rgb, t_alpha], -1).contiguous(), t_y, post_processing=method),
                     lambda: losses.image_loss_rgb(t_rgb, t_y, post_processing=method),
                     lambda: losses.image_loss_rgb_alpha(t_rgb, t_alpha, t_y, post_processing=method)):
            with pytest.raises(NotImplementedError, match="post_processing.method"):
                call()
    lib = nat.load()
    scratch = torch.empty(int(lib.gutb200_image_loss_scratch_bytes(40, 56)) // 4 + 1, device=dev)
    d = torch.empty((40, 56, 3), device=dev)
    d_alpha = torch.empty((40, 56), device=dev)
    sums = torch.empty(2, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    rc = lib.gutb200_image_loss(stream, 40, 56, 3, t_rgb.data_ptr(), t_alpha.data_ptr(), t_y.data_ptr(), None, None, None, 0.8, 0.2,
                                scratch.data_ptr(), d.data_ptr(), d_alpha.data_ptr(), sums.data_ptr(), 7)
    assert rc == 1 and "post_processing=7" in lib.gutb200_last_error(None).decode()


# ---------------------------------------------------------------------------------------------------------------------------------
# one step of each training step against autograd


def _target_and_mask(H, W, dev, use_mask):
    gen = torch.Generator(device=dev).manual_seed(3)
    target = (torch.rand((H, W, 3), device=dev, generator=gen) * 0.8).contiguous()
    mask = (torch.rand((H, W), device=dev, generator=gen) > 0.25).float() if use_mask else None
    return target, mask


def _encoded_loss(rgb, alpha, target, bg, mask, weights):
    """background -> linear_to_srgb -> mask -> L1 + SSIM as autograd (the kernel L1 + SSIM node of test_grt_train_step_gpu)."""
    import losses
    from test_grt_train_step_gpu import _ImageLoss

    x, y = rgb, target
    if bg is not None:
        x = x + bg * (1.0 - alpha)                # background.py:91 / 93
    x = losses.linear_to_srgb(x)                  # trainer.py:1165-1172, post_processing_linear_to_srgb.py:43-67
    if mask is not None:
        x, y = x * mask[..., None], y * mask[..., None]   # trainer.py:693-694
    return _ImageLoss.apply(torch.cat([x, torch.zeros_like(alpha)], -1), y, *weights)


SH_CASES = [("gut", "white", True, (0.8, 0.2)), ("gut", "black", False, (1.0, 0.0)), ("grt_instances", "random", True, (0.8, 0.2)),
            ("grt_instances", "black", False, (1.0, 0.0))]


@pytest.mark.parametrize("kind,background,use_mask,weights", SH_CASES)
def test_sh_step_matches_autograd(kind, background, use_mask, weights):
    """GaussianTrainStep (3DGUT) and GaussianTrainStepGRT: exp_avg / (1 - b1) after one bias-corrected step against the autograd gradient,
    at the bars of test_loss_terms_step_gpu.py."""
    from test_loss_terms_step_gpu import _Harness, _step_against_autograd

    hz = _Harness(kind)
    H, W, dev = hz.H, hz.W, hz.dev
    raw = raw_params(hz.P, hz.S)
    st = hz.make({k: v.clone() for k, v in raw.items()}, lambda_l1=weights[0], lambda_ssim=weights[1], background=background, background_seed=5,
                 post_processing=POST)
    target, mask = _target_and_mask(H, W, dev, use_mask)
    got_loss = float(hz.step(st, 1, target, mask=mask))
    bg = None
    if background == "random":
        bg = st.background.image.clone()
    elif background == "white":
        bg = torch.ones((H, W, 3), device=dev)
    leaves = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
    rgb, alpha = hz.autograd_render(leaves, 1)
    loss = _encoded_loss(rgb, alpha, target, bg, mask, weights)
    loss.backward()
    assert abs(got_loss - float(loss)) <= 1e-5, (got_loss, float(loss))
    floor = {}
    if kind.startswith("gut"):
        floor, _, _ = _step_against_autograd(hz, "black", False, 0.0, 0.0)  # the compact-vs-full floor of the plain 3DGUT step
    one_minus_b1 = float(np.float32(1) - np.float32(0.9))
    for k in raw:
        want = leaves[k].grad.cpu().numpy()
        assert float(np.abs(want).max()) > 0, k
        err = rel_l2(st.optimizer.exp_avg[k].cpu().numpy() / one_minus_b1, want)
        bar = max(1e-5, 2.0 * floor.get(k, 0.0))
        print(f"[post step] {kind} {background} mask {use_mask} {weights} {k}: rel-L2 {err:.2e} (bar {bar:.2e})")
        assert err <= bar, k


@pytest.mark.parametrize("kind", ["gut", "grt"])
def test_nht_step_matches_autograd(kind):
    """GaussianTrainStepNHT / GaussianTrainStepGRTNHT: the decoded rgb composited onto white, encoded, masked; bars of
    test_nht_train_step_gpu.py (the reference against itself)."""
    import feature_decoder as fdm
    import train_step_nht as tsn
    from test_nht_train_step import _einsum_dirs
    from test_nht_train_step_gpu import _decoder, _Harness

    hz = _Harness(kind)
    H, W, dev = hz.H, hz.W, hz.dev
    weights = (0.8, 0.2)
    dec = _decoder()
    params0 = dec.network.params.detach().clone()
    raw = raw_params(hz.P, features=hz.F)
    st = hz.make({k: v.clone() for k, v in raw.items()}, dec, lambda_l1=weights[0], lambda_ssim=weights[1], background="white",
                 post_processing=POST)
    target, mask = _target_and_mask(H, W, dev, True)
    got_loss = float(hz.step(st, 1, target, mask=mask))
    white = torch.ones((H, W, 3), device=dev)

    def autograd(dirs):
        leaves = {k: v.clone().requires_grad_(True) for k, v in raw.items()}
        dparams = params0.clone().requires_grad_(True)
        feats, alpha = hz.autograd_render(leaves, 1)
        rgb = fdm.decode(feats.reshape(-1, 24), dirs, dparams, dec.config).reshape(H, W, 3)
        loss = _encoded_loss(rgb, alpha, target, white, mask, weights)   # decoder -> background -> linear_to_srgb -> mask -> loss
        loss.backward()
        grads = {k: leaves[k].grad.cpu().numpy() for k in raw}
        grads["decoder"] = dparams.grad.cpu().numpy()
        return grads, float(loss.detach())

    want, want_loss = autograd(_einsum_dirs(hz.c2w(1), hz.rays_d.cpu()).to(dev))
    again, _ = autograd(_einsum_dirs(hz.c2w(1), hz.rays_d.cpu()).to(dev))
    R = tsn.c2w_rotation_from_pose7(hz.views[1]) if kind == "gut" else tsn.c2w_rotation_from_T(hz.poses[1])
    alt, _ = autograd(tsn.world_ray_directions(R, hz.rays_d))
    assert abs(got_loss - want_loss) <= 1e-5 * max(1.0, abs(want_loss)), (got_loss, want_loss)
    one_minus_b1 = float(np.float32(1) - np.float32(0.9))
    got = {k: st.optimizer.exp_avg[k].cpu().numpy() / one_minus_b1 for k in raw}
    got["decoder"] = st.optimizer.decoder_exp_avg.cpu().numpy() / one_minus_b1
    for k in want:
        assert float(np.abs(want[k]).max()) > 0, k
        err = rel_l2(got[k], want[k])
        floor = max(rel_l2(again[k], want[k]), rel_l2(alt[k], want[k]))
        bar = max(1e-5, 2.0 * floor)
        print(f"[post nht step] {kind} {k}: rel-L2 {err:.2e} (reference vs itself {floor:.2e}, bar {bar:.2e})")
        assert err <= bar, k


@pytest.mark.parametrize("background", ["black", "white+mask"])
def test_hybrid_step_matches_autograd(background):
    """GaussianTrainStepHybrid: the final composite (primary + reflection, then the background with the primary alpha) encoded; the
    gradients handed to Adam against autograd through both reference-facing tracers, bar 1e-5 as test_hybrid_train_step_gpu.py's."""
    import threedgrt_tracer
    import threedgut_tracer
    import train_step_hybrid as th
    from test_hybrid_train_step_gpu import CONFIGS, LRS, _Batch, _capture_adam, _Gaussians, _SecondaryBatch, _setup

    sc, rays_o, rays_d, P, S, poses, sensor = _setup()
    dev = P.device
    H, W = sc.height, sc.width
    white = background != "black"
    weights = (0.8, 0.2) if white else (1.0, 0.0)
    target, mask = _target_and_mask(H, W, dev, white)
    step = th.GaussianTrainStepHybrid(raw_params(P, S), LRS, conf=CONFIGS["instances"], lambda_l1=weights[0], lambda_ssim=weights[1],
                                      background="white" if white else "black", post_processing=POST)
    particles, sph = step.activated()
    seen = _capture_adam(step)
    c2w = poses[1]
    got_loss = float(step.step(rays_o, rays_d, sensor, c2w, target, mask=mask))
    d_particles, d_sph = seen[0]

    conf = th.hybrid_render_conf(CONFIGS["instances"])
    g = _Gaussians(particles, sph, 3)
    primary = threedgut_tracer.Tracer(conf).render(g, _Batch(sc, rays_o, rays_d, c2w), train=True)
    m = th.mirror_settings()
    so, sd, hit = th.hybrid_rays(rays_o, rays_d, c2w, m["plane_point"], m["plane_normal"])
    grt = threedgrt_tracer.Tracer(conf)
    grt.build_acc(g, rebuild=True)
    secondary = grt.render(g, _SecondaryBatch(so, sd), train=True)
    rgb = primary["pred_features"] + m["reflectivity"] * (1.0 - primary["pred_opacity"]) * hit.view(1, H, W, 1) * secondary["pred_features"]
    loss = _encoded_loss(rgb[0], primary["pred_opacity"][0], target, torch.ones((H, W, 3), device=dev) if white else None, mask, weights)
    loss.backward()
    assert abs(got_loss - float(loss)) <= 1e-5, (got_loss, float(loss))
    ref = {"positions": (g.positions.grad, d_particles[:, 0:3]), "density": (g.density.grad, d_particles[:, 3:4]),
           "rotation": (g.rotation.grad, d_particles[:, 4:8]), "scale": (g.scale.grad, d_particles[:, 8:11]), "sph": (g._sph.grad, d_sph)}
    for name, (want, got) in ref.items():
        err = rel_l2(got.cpu().numpy(), want.cpu().numpy())
        print(f"[post hybrid step] {background} {name}: rel-L2 {err:.2e} (bar 1e-5)")
        assert float(want.abs().max()) > 0 and err <= 1e-5, name


# ---------------------------------------------------------------------------------------------------------------------------------
# fits to sRGB targets


@pytest.mark.parametrize("kind", ["gut", "grt_instances"])
def test_fit_to_srgb_targets(kind):
    """Targets rendered sRGB-encoded from the unperturbed scene; 90 steps of the perturbed scene with the encode in the loss bring the
    encoded L1 down by the factor of the existing fits."""
    from test_grt_train_step_gpu import _perturb
    from test_loss_terms_step_gpu import _Harness, _mean_composited_l1

    hz = _Harness(kind)
    truth = hz.make(raw_params(hz.P, hz.S), post_processing=POST)
    targets = [hz.render(truth, v)[0].clone() for v in range(6)]   # render() returns the encoded rgb
    P2, S2 = _perturb(hz.sc, hz.P.clone(), hz.S.clone())
    fit = hz.make(raw_params(P2, S2), post_processing=POST)
    before = _mean_composited_l1(hz, fit, targets)
    for it in range(90):
        hz.step(fit, it % 6, targets[it % 6])
    after = _mean_composited_l1(hz, fit, targets)
    print(f"[post fit] {kind}: mean encoded L1 over 6 views {before:.5f} -> {after:.5f} after 90 steps")
    assert np.isfinite(after) and after < 0.6 * before

"""evaluate.evaluate / validate / from_checkpoint on the GPU, through the five training steps on C1: per-frame metrics against the float64
restatement applied to each step's own renders, the PNG files, metrics.json, the training state left untouched, the NHT decoder's EMA,
checkpoints of both tracers and the LPIPS hook."""
import copy
import json

import numpy as np
import pytest

import metrics_oracle as mo
from helpers import rel_l2
from test_checkpoint import _same
from test_metrics_gpu import _assert_bytes
from test_schedule_step_gpu import KINDS, LRS_NHT, LRS_SH, _compressed, _nht_step_conf, _Run

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

# the background and post-processing each step is evaluated with: every evaluation mode is met by some step
SETTINGS = {"gut": dict(background="white"), "grt": dict(background=(0.2, 0.5, 0.9)), "gut_nht": dict(background="random"),
            "grt_nht": dict(post_processing="linear-to-srgb"), "hybrid": dict(background="white", post_processing="linear-to-srgb")}
VIEWS = 4


def _args(run, v):
    if run.kind in ("gut", "gut_nht"):
        return (run.rays_o, run.rays_d, run.sensor, run.views7[v])
    if run.kind == "hybrid":
        return (run.rays_o, run.rays_d, run.sensor, run.poses[v])
    return (run.rays_o, run.rays_d, run.poses[v])


def _views(run, n=VIEWS):
    return [(_args(run, v), run.targets[v]) for v in range(n)]


def _lrs(run):
    return LRS_NHT if run.nht else LRS_SH


def _x(inputs, bg, post):
    """float64 composite of the step's own render (and the float32 x the device computes, for the colour correction and the bytes)."""
    import evaluate
    import metrics as M

    pred = inputs["pred"].reshape(inputs["pred"].shape[-3:]).double().cpu().numpy()
    rgb = pred[..., :3]
    alpha = pred[..., 3:] if inputs["alpha"] is None else inputs["alpha"].reshape(rgb.shape[0], rgb.shape[1], 1).double().cpu().numpy()
    x32 = evaluate._x_of({"pred": inputs["pred"].reshape(inputs["pred"].shape[-3:]), "alpha": inputs["alpha"]}, bg, post)
    return mo.prediction(rgb, alpha, M.background_rgb(bg), post), x32.cpu().numpy()


@pytest.mark.parametrize("kind", KINDS)
def test_every_step_end_to_end(kind, tmp_path):
    from PIL import Image

    import evaluate

    run = _Run(kind)
    st = run.make(run.start(), _lrs(run), **SETTINGS[kind])
    for it in range(3):
        run.step(st, it % 6)
    out = evaluate.evaluate(st, _views(run), out_dir=str(tmp_path))
    assert len(out["psnr"]) == VIEWS and out["inference_time_ms"].shape == (VIEWS,) and (out["inference_time_ms"] > 0).all()
    table = json.loads((tmp_path / "metrics.json").read_text())
    assert list(table) == ["mean_psnr", "mean_ssim", "mean_cc_psnr", "mean_cc_ssim", "mean_inference_time_ms"]
    assert out["std_psnr"] == pytest.approx(float(np.std(out["psnr"])))
    bg, post = st.background, st.post_processing
    for v in range(VIEWS):
        x, x32 = _x(st.metrics_inputs(*_args(run, v)), bg, post)
        y = run.targets[v].double().cpu().numpy()
        want = mo.frame_metrics(x, y, x32=x32)
        assert abs(out["psnr"][v] - want["psnr"]) <= 1e-4 and abs(out["cc_psnr"][v] - want["cc_psnr"]) <= 1e-4, (v, out["psnr"][v], want)
        assert abs(out["ssim"][v] - want["ssim"]) <= 2e-6 and abs(out["cc_ssim"][v] - want["cc_ssim"]) <= 2e-6, (v, out["ssim"][v], want)
        png = np.asarray(Image.open(str(tmp_path / f"ours_{st.frame}" / "renders" / f"{v:05d}.png")).convert("RGB"))
        _assert_bytes(png, x32)
        gt = np.asarray(Image.open(str(tmp_path / f"ours_{st.frame}" / "gt" / f"{v:05d}.png")).convert("RGB"))
        np.testing.assert_array_equal(gt, mo.quantise(run.targets[v].cpu().numpy()))
    val = evaluate.validate(st, _views(run))
    np.testing.assert_array_equal(val["per_view"]["psnr"], out["psnr"])
    assert val["mean"]["hits_max"] >= val["mean"]["hits_mean"] >= val["mean"]["hits_min"] >= 0


def _lockstep(run, kind, evaluate_b):
    """A trains 2k steps; B trains k steps, is evaluated, and trains k more, handed A's gradients after checking they agree (the
    backwards add with float atomics).  Everything else -- frame, schedule, densification, generators, BVH cadence -- must match bit for
    bit."""
    from test_checkpoint_gpu import _build, _grads

    conf = _compressed(kind)
    a, b = _build(run, kind, conf), _build(run, kind, conf)
    seen, worst = {}, [0.0]
    real_a, real_b = a._update, b._update

    def update_a(*args, **kw):
        seen["grads"] = [t.clone() for t in _grads(a)]
        return real_a(*args, **kw)

    def update_b(*args, **kw):
        for mine, theirs in zip(_grads(b), seen["grads"]):
            worst[0] = max(worst[0], rel_l2(mine.cpu(), theirs.cpu()))
            mine.copy_(theirs)
        return real_b(*args, **kw)

    a._update, b._update = update_a, update_b
    k = 12
    for it in range(2 * k):
        if it == k:
            before = copy.deepcopy(b.state_dict())
            evaluate_b(b)
            _same(b.state_dict(), before, "after the evaluation")
        run.step(a, it % 6)
        run.step(b, it % 6)
        _same(b.state_dict(), a.state_dict(), f"step {it}")
    assert worst[0] <= 1e-4


@pytest.mark.parametrize("kind", ["gut", "grt", "gut_nht"])
def test_evaluation_leaves_the_training_state_untouched(kind):
    import evaluate

    run = _Run(kind)
    _lockstep(run, kind, lambda b: evaluate.evaluate(b, _views(run, 2)))


def test_nht_scores_the_ema_weights_and_restores_the_live_ones():
    import evaluate
    import feature_decoder as fdm
    import metrics as M
    import train_step_nht

    run = _Run("gut_nht")
    torch.manual_seed(0)
    dec = fdm.FeatureDecoder(24, hidden_dim=128, num_layers=3, sh_scale=3.0, ema_decay=0.5).to(run.dev)
    st = train_step_nht.GaussianTrainStepNHT(run.start(), LRS_NHT, dec, _nht_step_conf())
    for it in range(4):
        run.step(st, it % 6)
    live = dec.network.params.detach().clone()
    shadow = dec.ema_state_dict()["network.params"]
    assert not torch.equal(live, shadow)
    out = evaluate.evaluate(st, _views(run, 2))
    assert torch.equal(dec.network.params.detach(), live)
    for v in range(2):
        dec.network.params.data.copy_(shadow)
        want_ema = M.as_dict(M.image_metrics(**_metric_args(st, run, v)).cpu().numpy())
        dec.network.params.data.copy_(live)
        want_live = M.as_dict(M.image_metrics(**_metric_args(st, run, v)).cpu().numpy())
        assert out["psnr"][v] == want_ema["psnr"] and out["psnr"][v] != want_live["psnr"]


def _metric_args(st, run, v):
    inp = st.metrics_inputs(*_args(run, v))
    return dict(pred=inp["pred"], target=run.targets[v], alpha=inp["alpha"], background=st.background, post_processing=st.post_processing,
                hits=inp["hits"])


@pytest.mark.parametrize("kind", ["gut", "grt"])
def test_from_checkpoint_reproduces_the_live_evaluation(kind, tmp_path):
    import checkpoint
    import evaluate

    run = _Run(kind)
    conf = _compressed(kind)
    conf["render"]["method"] = "3dgut" if kind == "gut" else "3dgrt"
    kw = dict(background="white")
    if kind == "grt":  # the live step traces with the overrides evaluation applies
        import train_step_grt

        live_conf = {"render": dict(evaluate.GRT_OVERRIDES)}
        st = train_step_grt.GaussianTrainStepGRT(run.start(), LRS_SH, conf=live_conf, **kw)
    else:
        st = run.make(run.start(), LRS_SH, **kw)
    for it in range(5):
        run.step(st, it % 6)
    path = str(tmp_path / "ckpt_5.pt")
    checkpoint.save(st, path, conf=conf)
    loaded = evaluate.from_checkpoint(path)
    assert loaded.frame == st.frame and type(loaded) is type(st)
    if kind == "grt":
        assert loaded.tracer._clamping and loaded.min_transmittance == pytest.approx(0.03)
    a, b = evaluate.evaluate(st, _views(run)), evaluate.evaluate(loaded, _views(run))
    for key in ("psnr", "ssim", "cc_psnr", "cc_ssim"):
        np.testing.assert_array_equal(a[key], b[key])


def test_lpips_hook_receives_clipped_and_corrected_images():
    import evaluate
    import metrics as M

    run = _Run("gut")
    st = run.make(run.start(), LRS_SH, background="white")
    calls = []

    def lpips(x, y):
        calls.append((x.clone(), y.clone()))
        return (x - y).abs().mean()

    out = evaluate.evaluate(st, _views(run, 2), lpips=lpips)
    assert len(calls) == 4 and "mean_lpips" in out["metrics"] and "mean_cc_lpips" in out["metrics"]
    H, W = run.sc.height, run.sc.width
    for v in range(2):
        (x, y), (xcc, y2) = calls[2 * v], calls[2 * v + 1]
        assert x.shape == (1, 3, H, W) and xcc.shape == (1, 3, H, W) and torch.equal(y, y2)
        assert x.min() >= 0 and x.max() <= 1 and xcc.min() >= 0 and xcc.max() <= 1
        inp = st.metrics_inputs(*_args(run, v))
        x_full = evaluate._x_of(inp, st.background, None)
        assert torch.equal(x[0].permute(1, 2, 0), x_full.clip(0, 1))
        row = M.as_dict(M.image_metrics(**_metric_args(st, run, v)).cpu().numpy())
        a = torch.tensor([row["a_r"], row["a_g"], row["a_b"]], device=x.device).float()
        b = torch.tensor([row["b_r"], row["b_g"], row["b_b"]], device=x.device).float()
        assert torch.equal(xcc[0].permute(1, 2, 0), ((x_full - b) / a).clip(0, 1))
        assert out["lpips"][v] == pytest.approx(float((x - y).abs().mean()))
    assert out["metrics"]["mean_lpips"] == pytest.approx(float(np.mean(out["lpips"])))

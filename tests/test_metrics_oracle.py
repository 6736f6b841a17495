"""The float64 restatement of the test-set metrics (tests/metrics_oracle.py) and evaluate's host logic, on the CPU: identical pairs, SSIM
against loss_oracle, the colour correction against a transcription of color_correct_affine, the quantisation against
torchvision.utils.save_image, metrics.json and the checkpoint overrides."""
import io
import json
import os

import numpy as np
import pytest

import metrics_oracle as mo
from oracle import loss_oracle as lo


def _images(seed, H=37, W=53, lo_=-0.2, hi=1.3):
    rng = np.random.default_rng(seed)
    return rng.uniform(lo_, hi, (H, W, 3)), rng.uniform(0.0, 1.0, (H, W, 3))


def test_an_identical_pair_scores_infinite_psnr_and_unit_ssim():
    _, y = _images(0)
    y = y.astype(np.float32).astype(np.float64)  # as the device holds it: the colour correction applies a = 1, b = 0 exactly
    m = mo.frame_metrics(y, y)
    assert m["psnr"] == float("inf") and m["cc_psnr"] == float("inf")
    assert m["ssim"] == pytest.approx(1.0, abs=1e-12) and m["cc_ssim"] == pytest.approx(1.0, abs=1e-12)
    np.testing.assert_allclose(m["a"], 1.0, atol=1e-9)
    np.testing.assert_allclose(m["b"], 0.0, atol=1e-9)
    assert m["l1"] == 0.0


def test_ssim_is_the_loss_oracles_valid_mean_where_no_variance_is_negative():
    x, y = _images(1, lo_=0.0, hi=1.0)
    full, (mu1, mu2, s1, s2, *_rest) = lo.ssim_map(x, y)
    inner = (slice(5, -5), slice(5, -5))
    assert (s1[inner] >= 0).all() and (s2[inner] >= 0).all()
    assert mo.ssim(x, y) == pytest.approx(float(full[inner].mean()), abs=1e-14)


def test_ssim_clamps_negative_variances():
    # a constant channel has a zero variance that rounds slightly negative in the windowed moments: the clamp keeps it at 0
    x, y = _images(2, lo_=0.0, hi=1.0)
    x[..., 1] = 0.7
    m = mo.ssim_map(x, y)
    assert np.isfinite(m).all()
    with pytest.raises(ValueError):
        mo.ssim(x[:10], y[:10])


def _color_correct_affine(img, ref):
    """threedgrut/utils/color_correct.py:96-145, line by line in numpy float64."""
    img_mat, ref_mat = img.reshape(-1, 3), ref.reshape(-1, 3)
    ref_mean, img_mean = ref_mat.mean(0), img_mat.mean(0)
    ref_img_mean, ref_ref_mean = (ref_mat * img_mat).mean(0), (ref_mat * ref_mat).mean(0)
    var_ref = np.maximum(ref_ref_mean - ref_mean * ref_mean, 1e-8)
    a = (ref_img_mean - ref_mean * img_mean) / var_ref
    b = img_mean - a * ref_mean
    a = np.where(np.abs(a) < 1e-8, np.ones_like(a), a)
    return np.clip((img_mat - b) / a, 0, 1).reshape(img.shape)


@pytest.mark.parametrize("case", ["plain", "constant_target", "uncorrelated"])
def test_color_correction_matches_color_correct_affine(case):
    x, y = _images(3)
    if case == "constant_target":  # var_ref clamps at 1e-8
        y[..., 0] = 0.25
    if case == "uncorrelated":  # |a| < 1e-8 -> 1 (b keeps the slope it was computed with)
        x[..., 2] = 0.5
    a, b = mo.affine(x, y)
    if case == "constant_target":
        ym = y.reshape(-1, 3)
        assert (ym * ym).mean(0)[0] - ym.mean(0)[0] ** 2 < 1e-8
    if case == "uncorrelated":
        assert a[2] == 1.0
    want = _color_correct_affine(x, y)
    got = np.clip((x - b) / a, 0, 1)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12)
    # the float32 application: a few float32 roundings of (x - b) / a, amplified by 1 / a where the fit is weak
    np.testing.assert_allclose(mo.color_correct(x, y), want, rtol=0, atol=1e-5)


def test_quantisation_is_byte_identical_to_save_image():
    torch = pytest.importorskip("torch")
    tvu = pytest.importorskip("torchvision.utils")
    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(4)
    v = rng.uniform(-0.5, 1.5, (19, 23, 3)).astype(np.float32)
    # the half-way points of every byte, just below and above them, and the ends
    edges = (np.arange(256, dtype=np.float32) + 0.5) / np.float32(255.0)
    v.reshape(-1)[: 3 * 256] = np.concatenate([edges, np.nextafter(edges, np.float32(0)), np.nextafter(edges, np.float32(2))])
    v.reshape(-1)[-4:] = [0.0, 1.0, -0.0, 255.0]
    buf = io.BytesIO()
    tvu.save_image(torch.from_numpy(v).permute(2, 0, 1), buf, format="png")
    want = np.asarray(Image.open(io.BytesIO(buf.getvalue())).convert("RGB"))
    np.testing.assert_array_equal(mo.quantise(v), want)


def test_write_png_decodes_to_its_bytes(tmp_path):
    import evaluate

    Image = pytest.importorskip("PIL.Image")
    rng = np.random.default_rng(5)
    u8 = rng.integers(0, 256, (13, 29, 3), dtype=np.uint8)
    evaluate.write_png(str(tmp_path / "a.png"), u8)
    np.testing.assert_array_equal(np.asarray(Image.open(str(tmp_path / "a.png")).convert("RGB")), u8)


def _rows(F=5, seed=6):
    import metrics as M

    rng = np.random.default_rng(seed)
    rows = rng.uniform(0, 40, (F, M.K))
    return rows


def test_metrics_json_keys_and_aggregation(tmp_path):
    import evaluate
    import metrics as M

    rows, times = _rows(), [1.0, 2.0, 3.0, 4.0, 5.0]
    out = evaluate.summarise(rows, times)
    assert list(out["metrics"]) == ["mean_psnr", "mean_ssim", "mean_cc_psnr", "mean_cc_ssim", "mean_inference_time_ms"]
    for k in ("psnr", "ssim", "cc_psnr", "cc_ssim"):
        np.testing.assert_array_equal(out[k], rows[:, M.FIELDS.index(k)])
        assert out["metrics"][f"mean_{k}"] == pytest.approx(np.mean(rows[:, M.FIELDS.index(k)]))
    assert out["std_psnr"] == pytest.approx(np.std(rows[:, 0]))  # population std, as render_all
    assert out["mean_inference_time"] == 3.0
    with_lpips = evaluate.summarise(rows, times, scores=[(0.1 * i, 0.2 * i) for i in range(5)])
    assert list(with_lpips["metrics"]) == ["mean_psnr", "mean_ssim", "mean_lpips", "mean_cc_psnr", "mean_cc_ssim", "mean_cc_lpips",
                                           "mean_inference_time_ms"]
    assert with_lpips["metrics"]["mean_cc_lpips"] == pytest.approx(0.4)
    u8 = np.zeros((12, 11, 3), np.uint8)
    evaluate.write_outputs(str(tmp_path), 7, [(u8, u8 + 1)], out["metrics"])
    assert os.path.exists(tmp_path / "ours_7" / "renders" / "00000.png") and os.path.exists(tmp_path / "ours_7" / "gt" / "00000.png")
    assert json.loads((tmp_path / "metrics.json").read_text()) == out["metrics"]


def test_eval_config_applies_the_3dgrt_overrides():
    import evaluate

    conf = {"render": {"method": "3dgrt", "particle_kernel_density_clamping": False, "min_transmittance": 0.001}, "model": {}}
    got = evaluate.eval_config(conf)
    assert got["render"]["particle_kernel_density_clamping"] is True and got["render"]["min_transmittance"] == 0.03
    assert conf["render"]["min_transmittance"] == 0.001  # the caller's config is not changed
    gut = evaluate.eval_config({"render": {"method": "3dgut", "min_transmittance": 0.001}})
    assert gut["render"]["min_transmittance"] == 0.001
    with pytest.raises(NotImplementedError, match="post_processing"):
        evaluate.eval_config({"render": {"method": "3dgut"}, "post_processing": {"method": "ppisp"}})


def test_background_of_evaluation():
    import metrics as M

    assert M.background_rgb("random") is None and M.background_rgb("black") is None and M.background_rgb(None) is None
    assert M.background_rgb("white") == (1.0, 1.0, 1.0) and M.background_rgb([0.1, 0.2, 0.3]) == (0.1, 0.2, 0.3)
    with pytest.raises(ValueError):
        M.background_rgb("grey")

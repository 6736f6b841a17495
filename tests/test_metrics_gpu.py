"""gutb200_image_metrics (metrics.image_metrics) against the float64 restatement (tests/metrics_oracle.py): both layouts, black, white and
colour backgrounds, no post-processing and linear-to-sRGB, predictions outside [0, 1], constant channels, the hit statistics, the PNG
bytes, determinism, the size limit, and torchmetrics where it is installed."""
import numpy as np
import pytest
import torch

import metrics_oracle as mo

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
SIZES = [(11, 11), (37, 130), (75, 53), (800, 800)]
BACKGROUNDS = {"black": None, "white": "white", "colour": (0.2, 0.55, 0.9)}


def _frame(H, W, seed, constant=False):
    rng = np.random.default_rng(seed)
    rgb = rng.uniform(-0.15, 1.2, (H, W, 3)).astype(np.float32)  # above 1 and below 0
    alpha = rng.uniform(0.0, 1.0, (H, W, 1)).astype(np.float32)
    # a smooth target with some texture, correlated with the prediction
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    target = (0.5 + 0.3 * np.sin(xx[..., None] / 7.0 + np.arange(3) + yy[..., None] / 11.0)).astype(np.float32)
    target = np.clip(target + 0.1 * rng.normal(size=target.shape).astype(np.float32), 0, 1).astype(np.float32)
    rgb = (0.6 * rgb + 0.4 * target).astype(np.float32)
    if constant:
        target[..., 0] = 0.25  # a constant target channel: var_ref clamps
        rgb[..., 2] = 0.5      # a constant prediction channel
    hits = rng.integers(0, 40, (H, W)).astype(np.int32)
    return rgb, alpha, target, hits


def _x32(rgb, alpha, bg, post):
    """x as the device computes it (float32 composite and encode, torch on the GPU), for the colour-corrected image and the bytes."""
    import losses
    import metrics as M

    r, a = torch.from_numpy(rgb).to(DEV), torch.from_numpy(alpha).to(DEV)
    b = M.background_rgb(bg)
    x = r if b is None else r + torch.tensor(b, device=DEV) * (1.0 - a)
    return (x if post is None else losses.linear_to_srgb(x)).cpu().numpy()


def _check(got, rgb, alpha, target, hits, bg, post, u8=None):
    import metrics as M

    x = mo.prediction(rgb, alpha, M.background_rgb(bg), post)
    want = mo.frame_metrics(x, target, x32=_x32(rgb, alpha, bg, post))
    g = M.as_dict(got)
    assert abs(g["psnr"] - want["psnr"]) <= 1e-4, (g["psnr"], want["psnr"])
    assert abs(g["ssim"] - want["ssim"]) <= 2e-6, (g["ssim"], want["ssim"])
    assert abs(g["cc_ssim"] - want["cc_ssim"]) <= 2e-6, (g["cc_ssim"], want["cc_ssim"])
    assert abs(g["cc_psnr"] - want["cc_psnr"]) <= 1e-4, (g["cc_psnr"], want["cc_psnr"])
    assert abs(g["l1"] - want["l1"]) <= 1e-6
    np.testing.assert_allclose([g["a_r"], g["a_g"], g["a_b"]], want["a"], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose([g["b_r"], g["b_g"], g["b_b"]], want["b"], rtol=1e-5, atol=1e-7)
    if hits is not None:
        hs = mo.hit_stats(hits)
        for k in ("hits_mean", "hits_min", "hits_max"):
            assert g[k] == hs[k], k
        assert g["hits_std"] == pytest.approx(hs["hits_std"], rel=1e-12)
    if u8 is not None:
        _assert_bytes(u8[0].cpu().numpy(), _x32(rgb, alpha, bg, post))
        np.testing.assert_array_equal(u8[1].cpu().numpy(), mo.quantise(target))


def _assert_bytes(got, x32):
    """The kernel's bytes are the quantisation of x.  x32 is x as torch computes it in float32; where the encode's power (post-processing)
    rounds one ulp apart from it, the byte may differ by one exactly at a rounding boundary -- and only there."""
    want = mo.quantise(x32)
    diff = got.astype(np.int32) - want
    if not diff.any():
        return
    bad = np.nonzero(diff)
    lo, hi = mo.quantise(np.nextafter(x32, np.float32(-np.inf))), mo.quantise(np.nextafter(x32, np.float32(np.inf)))
    assert (np.abs(diff[bad]) == 1).all() and ((got[bad] == lo[bad]) | (got[bad] == hi[bad])).all(), (len(bad[0]), got[bad][:8], want[bad][:8])


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.parametrize("post", [None, "linear-to-srgb"])
@pytest.mark.parametrize("bg", list(BACKGROUNDS))
@pytest.mark.parametrize("layout", [4, 3])
@pytest.mark.parametrize("size", SIZES, ids=[f"{h}x{w}" for h, w in SIZES])
def test_kernel_matches_the_oracle(size, layout, bg, post):
    import metrics as M

    H, W = size
    for constant in (False, True):
        rgb, alpha, target, hits = _frame(H, W, seed=H * 7 + W + layout, constant=constant)
        if layout == 4:
            pred, a = _t(np.concatenate([rgb, alpha], -1)), None
        else:
            pred, a = _t(rgb), _t(alpha)
        out, pu8, tu8 = M.image_metrics(pred, _t(target), alpha=a, background=BACKGROUNDS[bg], post_processing=post, hits=_t(hits), png=True)
        _check(out.cpu().numpy(), rgb, alpha, target, hits, BACKGROUNDS[bg], post, (pu8, tu8))


def test_two_calls_give_the_same_bits_and_rows_of_one_tensor():
    import metrics as M

    rgb, alpha, target, hits = _frame(800, 800, seed=3)
    pred = _t(np.concatenate([rgb, alpha], -1))
    rows = torch.empty((2, M.K), dtype=torch.float64, device=DEV)
    for i in range(2):
        M.image_metrics(pred, _t(target), background="white", post_processing="linear-to-srgb", hits=_t(hits), out=rows[i])
    r = rows.cpu().numpy()
    assert r[0].tobytes() == r[1].tobytes()


def test_identical_pair_and_no_hits():
    import metrics as M

    _, _, target, _ = _frame(64, 48, seed=4)
    got = M.as_dict(M.image_metrics(_t(target), _t(target), alpha=_t(np.ones((64, 48, 1), np.float32))).cpu().numpy())
    assert got["psnr"] == float("inf") and got["cc_psnr"] == float("inf")
    assert got["ssim"] == pytest.approx(1.0, abs=1e-6) and got["cc_ssim"] == pytest.approx(1.0, abs=1e-6)
    assert np.isnan(got["hits_mean"]) and np.isnan(got["hits_max"])


@pytest.mark.parametrize("size", [(10, 40), (40, 10), (5, 5)])
def test_below_11_pixels_is_refused(size):
    import metrics as M

    H, W = size
    x = torch.zeros((H, W, 4), device=DEV)
    with pytest.raises(ValueError, match="11"):
        M.image_metrics(x, torch.zeros((H, W, 3), device=DEV))


def test_torchmetrics_agrees():
    tm = pytest.importorskip("torchmetrics")
    import metrics as M

    rgb, alpha, target, _ = _frame(75, 53, seed=5)
    rgb = np.clip(rgb, 0, 1)
    got = M.as_dict(M.image_metrics(_t(rgb), _t(target), alpha=_t(alpha)).cpu().numpy())
    x, y = _t(rgb).permute(2, 0, 1)[None], _t(target).permute(2, 0, 1)[None]
    psnr = float(tm.image.PeakSignalNoiseRatio(data_range=1.0).to(DEV)(x, y))
    ssim = float(tm.image.StructuralSimilarityIndexMeasure(data_range=1.0).to(DEV)(x, y))
    assert abs(got["psnr"] - psnr) <= 1e-4 and abs(got["ssim"] - ssim) <= 2e-6

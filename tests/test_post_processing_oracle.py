"""CPU checks of the linear-to-sRGB post-processing: the encode at fixed points, its derivative against central differences, the float64
oracle (tests/post_processing_oracle.py) against the numpy loss oracle with the chain rule written out, and the refusal of methods that
are not built (PPISP and unknown names)."""
import numpy as np
import pytest

import post_processing_oracle as ppo
from oracle import loss_oracle as lo

torch = pytest.importorskip("torch")


def _s(x):
    return float(ppo.linear_to_srgb(torch.tensor([x], dtype=torch.float64))[0])


def test_encode_at_fixed_points():
    import losses

    limit = 0.0031308
    assert _s(0.0) == 0.0
    assert _s(limit) == 12.92 * limit                        # the branch point itself takes the linear branch
    above = np.nextafter(limit, 1.0)
    assert _s(above) == pytest.approx(1.055 * above ** (1 / 2.4) - 0.055, rel=1e-15)
    assert abs(_s(above) - _s(limit)) < 1e-7                # the two branches meet there (to the precision of the standard's constants)
    assert _s(-0.25) == -0.25 * 12.92                        # negatives stay on the linear branch, unclamped
    assert _s(1.0) == pytest.approx(1.0, abs=1e-15)
    for hdr in (1.5, 4.0, 100.0):                            # HDR: no clamp to [0, 1]
        assert _s(hdr) == pytest.approx(1.055 * hdr ** (1 / 2.4) - 0.055, rel=1e-15) and _s(hdr) > 1.0
    x = torch.tensor([-1.0, 0.0, 1e-9, limit, 0.01, 0.5, 1.0, 3.0], dtype=torch.float64)
    assert torch.equal(losses.linear_to_srgb(x), ppo.linear_to_srgb(x))   # the public encode is the oracle's
    x32 = x.float()
    got = losses.linear_to_srgb(x32)
    assert got.dtype == torch.float32 and torch.allclose(got.double(), ppo.linear_to_srgb(x), rtol=1e-6, atol=1e-7)


def test_derivative_matches_central_differences():
    xs = np.concatenate([np.linspace(-1.0, 0.003, 41), np.linspace(0.0032, 0.05, 41), np.linspace(0.05, 8.0, 81)])
    h = 1e-7
    fd = np.array([(_s(x + h) - _s(x - h)) / (2 * h) for x in xs])
    np.testing.assert_allclose(ppo.linear_to_srgb_slope(xs), fd, rtol=1e-6)
    # autograd through torch.where takes the same branch
    t = torch.tensor(xs, dtype=torch.float64, requires_grad=True)
    ppo.linear_to_srgb(t).sum().backward()
    np.testing.assert_allclose(t.grad.numpy(), ppo.linear_to_srgb_slope(xs), rtol=1e-12)


@pytest.mark.parametrize("background", ["black", "white", "image"])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("lambda_ssim", [0.0, 0.2])
def test_oracle_is_the_chain_rule_on_the_numpy_loss(background, masked, lambda_ssim):
    """d rgb = m s'(c) dL/dx and d alpha = -sum_c bg_c m s'(c_c) dL/dx_c, with dL/dx from oracle/loss_oracle.py."""
    rng = np.random.default_rng(7 + 3 * masked + 11 * ["black", "white", "image"].index(background) + int(10 * lambda_ssim))
    h, w = 29, 33
    rgb = rng.uniform(-0.02, 1.3, (h, w, 3))
    alpha = rng.uniform(0.05, 1.0, (h, w, 1))
    y = rng.uniform(0, 1, (h, w, 3))
    bg = {"black": None, "white": (1.0, 1.0, 1.0), "image": rng.uniform(0, 1, (h, w, 3))}[background]
    m = (rng.uniform(size=(h, w)) > 0.3).astype(np.float64) if masked else None
    loss, d_rgb, d_alpha = ppo.loss_and_gradients(rgb, alpha, y, 0.8, lambda_ssim, bg, m)

    c = rgb if bg is None else rgb + np.broadcast_to(bg, rgb.shape) * (1.0 - alpha)
    x = ppo.linear_to_srgb(torch.as_tensor(c)).numpy()
    mm = np.ones((h, w, 1)) if m is None else m[..., None]
    r_loss, _, _, gx = lo.loss_and_gradient(x * mm, y * mm, 0.8, lambda_ssim)
    g = mm * ppo.linear_to_srgb_slope(c) * gx
    assert loss == pytest.approx(r_loss, rel=1e-12)
    np.testing.assert_allclose(d_rgb, g, rtol=1e-9, atol=1e-14)
    want_alpha = np.zeros((h, w, 1)) if bg is None else -(np.broadcast_to(bg, rgb.shape) * g).sum(-1, keepdims=True)
    np.testing.assert_allclose(d_alpha, want_alpha, rtol=1e-9, atol=1e-14)


@pytest.mark.parametrize("method", ["ppisp", "linear_to_srgb", "srgb", "Linear-To-SRGB", 1, True])
def test_methods_that_are_not_built_are_refused_by_name(method):
    import losses
    import train_step

    with pytest.raises(NotImplementedError, match="post_processing.method"):
        losses.post_processing_code(method)
    # the training steps refuse at construction, before they touch their arguments
    with pytest.raises(NotImplementedError, match="post_processing.method"):
        train_step.GaussianTrainStep({}, {}, post_processing=method)


def test_built_methods_map_to_their_device_codes():
    import losses

    assert losses.post_processing_code(None) == 0
    assert losses.post_processing_code("linear-to-srgb") == 1

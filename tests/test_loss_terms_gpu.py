"""GPU parity of the composited / masked image loss (gutb200_image_loss_composited) and of the fused Adam step with the opacity and scale
regularisers (gutb200_gaussian_adam_step_reg) against tests/loss_terms_oracle.py.
Bars as in test_loss_gpu.py / test_adam_gpu.py: loss terms 1e-6 absolute; gradient |diff| <= 2e-6 * max|grad| + 1e-10; Adam 2e-6 relative."""
import numpy as np
import pytest

import loss_terms_oracle as lto
from oracle import adam_oracle as ao
from test_adam_gpu import _close
from test_adam_oracle import LRS, _state

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

BACKGROUNDS = ("black", "white", "colour", "random")
MASKS = ("none", "random", "zeros", "ones")


def _case(h, w, background, mask, seed):
    rng = np.random.default_rng(seed)
    y = rng.uniform(0, 1, (h, w, 3)).astype(np.float32)
    rgb = np.clip(0.7 * y + 0.1 * rng.normal(size=(h, w, 3)), 0, 1.2).astype(np.float32)
    alpha = rng.uniform(0.05, 1.0, (h, w, 1)).astype(np.float32)
    bg = {"black": None, "white": (1.0, 1.0, 1.0), "colour": (0.2, 0.5, 0.9), "random": rng.uniform(0, 1, (h, w, 3)).astype(np.float32)}[background]
    m = {"none": None, "random": (rng.uniform(size=(h, w)) > 0.3).astype(np.float32), "zeros": np.zeros((h, w), np.float32),
         "ones": np.ones((h, w), np.float32)}[mask]
    return rgb, alpha, y, bg, m


def _dev(a, dev):
    return None if a is None else (torch.from_numpy(np.ascontiguousarray(a)).to(dev) if isinstance(a, np.ndarray) else a)


def _run(layout, rgb, alpha, y, bg, m, weights, dev):
    import losses

    t_rgb, t_alpha, t_y, t_bg, t_m = (_dev(a, dev) for a in (rgb, alpha, y, bg, m))
    if layout == 4:
        loss, l1, ssim, d = losses.image_loss(torch.cat([t_rgb, t_alpha], -1).contiguous(), t_y, *weights, background=t_bg, mask=t_m)
        assert d.shape == rgb.shape[:2] + (4,)
        d = d.cpu().numpy()
        return float(loss), float(l1), float(ssim), d[..., :3], d[..., 3:]
    loss, l1, ssim, d_rgb, d_alpha = losses.image_loss_rgb_alpha(t_rgb, t_alpha, t_y, *weights, background=t_bg, mask=t_m)
    assert d_rgb.shape == rgb.shape and d_alpha.shape == alpha.shape
    return float(loss), float(l1), float(ssim), d_rgb.cpu().numpy(), d_alpha.cpu().numpy()


@pytest.mark.parametrize("size", [(96, 96), (61, 97), (800, 800)])
@pytest.mark.parametrize("layout", [4, 3])
@pytest.mark.parametrize("background", BACKGROUNDS)
@pytest.mark.parametrize("mask", MASKS)
def test_composited_loss_matches_oracle(size, layout, background, mask):
    h, w = size
    dev = torch.device("cuda", 0)
    rgb, alpha, y, bg, m = _case(h, w, background, mask, seed=h * 1000 + w + 10 * BACKGROUNDS.index(background) + MASKS.index(mask))
    weights = (0.8, 0.2)
    loss, l1, ssim, d_rgb, d_alpha = _run(layout, rgb, alpha, y, bg, m, weights, dev)
    r_loss, r_l1, r_ssim, r_rgb, r_alpha = lto.composited_loss_and_gradients(rgb, alpha, y, *weights, background=bg, mask=m,
                                                                            device_rounding=True)
    assert abs(l1 - r_l1) <= 1e-6 and abs(ssim - r_ssim) <= 1e-6 and abs(loss - r_loss) <= 1e-6, (l1 - r_l1, ssim - r_ssim, loss - r_loss)
    e_rgb, e_alpha = np.abs(d_rgb - r_rgb).max(), np.abs(d_alpha - r_alpha).max()
    print(f"[loss-terms] {size} layout {layout} {background} mask {mask}: max |d_rgb diff| {e_rgb:.2e} (max {np.abs(r_rgb).max():.2e}), "
          f"max |d_alpha diff| {e_alpha:.2e} (max {np.abs(r_alpha).max():.2e})")
    assert e_rgb <= 2e-6 * np.abs(r_rgb).max() + 1e-10
    assert e_alpha <= 2e-6 * np.abs(r_alpha).max() + 1e-10
    if background == "black":
        assert not d_alpha.any()
    if mask == "zeros":
        assert not d_rgb.any() and not d_alpha.any()


@pytest.mark.parametrize("size", [(96, 96), (61, 97), (800, 800)])
@pytest.mark.parametrize("weights", [(0.8, 0.2), (1.0, 0.0)])
def test_black_and_all_ones_mask_are_bit_identical_to_the_plain_entries(size, weights):
    import losses

    h, w = size
    dev = torch.device("cuda", 0)
    rgb, alpha, y, _, ones = _case(h, w, "black", "ones", seed=h + w)
    t_rgb, t_alpha, t_y, t_ones = (torch.from_numpy(a).to(dev) for a in (rgb, alpha, y, ones))
    rgba = torch.cat([t_rgb, t_alpha], -1).contiguous()
    plain4 = losses.image_loss(rgba, t_y, *weights)[3]
    plain3 = losses.image_loss_rgb(t_rgb, t_y, *weights)[3]
    for mask in (None, t_ones, t_ones[None, :, :, None]):
        for background in ((0.0, 0.0, 0.0), None):
            if mask is None and background is None:
                continue  # that is the plain entry itself
            d4 = losses.image_loss(rgba, t_y, *weights, background=background, mask=mask)[3]
            assert torch.equal(d4, plain4)
            _, _, _, d_rgb, d_alpha = losses.image_loss_rgb_alpha(t_rgb, t_alpha, t_y, *weights, background=background, mask=mask)
            assert torch.equal(d_rgb, plain3) and not bool(d_alpha.any())


def test_all_zeros_mask_gives_a_zero_gradient():
    import losses

    dev = torch.device("cuda", 0)
    rgb, alpha, y, bg, zeros = _case(80, 72, "random", "zeros", seed=1)
    t_rgb, t_alpha, t_y, t_bg, t_z = (torch.from_numpy(a).to(dev) for a in (rgb, alpha, y, bg, zeros))
    loss, l1, ssim, d_rgb, d_alpha = losses.image_loss_rgb_alpha(t_rgb, t_alpha, t_y, 0.8, 0.2, background=t_bg, mask=t_z)
    assert not bool(d_rgb.any()) and not bool(d_alpha.any())
    assert float(l1) == 0.0 and abs(float(ssim) - 1.0) <= 1e-6
    d4 = losses.image_loss(torch.cat([t_rgb, t_alpha], -1).contiguous(), t_y, 0.8, 0.2, background=(1.0, 1.0, 1.0), mask=t_z)[3]
    assert not bool(d4.any())


def test_composited_loss_rejects_bad_arguments():
    import ctypes

    import b200_native as nat
    import losses

    dev = torch.device("cuda", 0)
    rgb = torch.rand((16, 16, 3), device=dev)
    alpha = torch.rand((16, 16, 1), device=dev)
    tgt = torch.rand((16, 16, 3), device=dev)
    for bad in (torch.ones((16, 15), device=dev), torch.ones((2, 16, 16, 1), device=dev), torch.ones((16, 16), dtype=torch.uint8, device=dev),
                torch.ones((16, 16))):
        with pytest.raises(RuntimeError):
            losses.image_loss_rgb_alpha(rgb, alpha, tgt, mask=bad)
    with pytest.raises(RuntimeError):
        losses.image_loss_rgb_alpha(rgb, alpha, tgt, background=torch.rand((16, 16, 3)))
    with pytest.raises(ValueError):
        losses.Background("grey")
    lib = nat.load()
    scratch = torch.empty(int(lib.gutb200_image_loss_scratch_bytes(16, 16)) // 4 + 1, device=dev)
    sums = torch.empty(2, device=dev)
    d = torch.empty(16 * 16 * 4 + 1, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    bg = (ctypes.c_float * 3)(1.0, 1.0, 1.0)
    rgba = torch.cat([rgb, alpha], -1).contiguous()
    call = lib.gutb200_image_loss_composited
    assert call(stream, 16, 16, 4, rgba.data_ptr(), None, tgt.data_ptr(), bg, None, None, 0.8, 0.2, scratch.data_ptr(), d.data_ptr() + 4, None,
                sums.data_ptr()) == 3  # the 4-wide gradient is stored 16 bytes at a time
    assert call(stream, 16, 16, 3, rgb.data_ptr(), None, tgt.data_ptr(), bg, None, None, 0.8, 0.2, scratch.data_ptr(), d.data_ptr(), d.data_ptr(),
                sums.data_ptr()) == 1  # split layout without its alpha
    assert call(stream, 16, 16, 3, rgb.data_ptr(), alpha.data_ptr(), tgt.data_ptr(), bg, None, None, 0.8, 0.2, scratch.data_ptr(), d.data_ptr(),
                None, sums.data_ptr()) == 1  # ... or without d_alpha
    assert call(stream, 16, 16, 5, rgba.data_ptr(), None, tgt.data_ptr(), bg, None, None, 0.8, 0.2, scratch.data_ptr(), d.data_ptr(), None,
                sums.data_ptr()) == 1
    assert call(stream, 0, 16, 4, rgba.data_ptr(), None, tgt.data_ptr(), bg, None, None, 0.8, 0.2, scratch.data_ptr(), d.data_ptr(), None,
                sums.data_ptr()) == 1
    assert call(stream, 16, 16, 4, rgba.data_ptr(), None, None, bg, None, None, 0.8, 0.2, scratch.data_ptr(), d.data_ptr(), None,
                sums.data_ptr()) == 1


@pytest.mark.parametrize("selective", [False, True])
def test_regularised_adam_matches_oracle(selective):
    import optimizers

    dev = torch.device("cuda", 0)
    n = 4099
    params, _, _ = _state(n=n, seed=3)
    rng = np.random.default_rng(12)
    leaves = {k: torch.from_numpy(v.copy()).to(dev) for k, v in params.items()}
    opt = optimizers.FusedGaussianAdam(leaves, LRS, eps=1e-15, selective=selective)
    p = {k: v.copy() for k, v in params.items()}
    m = {k: np.zeros_like(v) for k, v in params.items()}
    v = {k: np.zeros_like(vv) for k, vv in params.items()}
    never = np.ones(n, bool)
    for t in range(1, 4):
        dp = (0.01 * rng.normal(size=(n, 12))).astype(np.float32)  # of the order of the regulariser terms
        ds = rng.normal(size=(n, 48)).astype(np.float32)
        vis_bits = (rng.uniform(size=n) > 0.3).astype(np.int32)
        never &= vis_bits == 0
        vis = torch.from_numpy(vis_bits.view(np.float32).copy()).to(dev)
        opt.step(torch.from_numpy(dp).to(dev), torch.from_numpy(ds).to(dev), visibility=vis if selective else None, lambda_opacity=0.3,
                 lambda_scale=0.2)
        p, m, v = lto.gaussian_adam_step(p, m, v, LRS, dp, ds, eps=1e-15, step=t, selective=selective, visibility=vis_bits != 0,
                                         lambda_opacity=0.3, lambda_scale=0.2)
    torch.cuda.synchronize()
    for k in ao.GROUPS:
        _close(leaves[k].cpu().numpy(), p[k], f"param {k}")
        _close(opt.exp_avg[k].cpu().numpy(), m[k], f"exp_avg {k}")
        _close(opt.exp_avg_sq[k].cpu().numpy(), v[k], f"exp_avg_sq {k}")
    if selective:
        assert never.sum() > 0
        for k in ao.GROUPS:  # rows never visible are untouched bit for bit, regulariser or not
            assert np.array_equal(leaves[k].cpu().numpy()[never], params[k][never]), k
            assert not opt.exp_avg[k].cpu().numpy()[never].any(), k


def test_zero_lambdas_are_the_plain_step():
    import optimizers

    dev = torch.device("cuda", 0)
    n = 1031
    params, _, _ = _state(n=n, seed=4)
    rng = np.random.default_rng(13)
    dp = torch.from_numpy(rng.normal(size=(n, 12)).astype(np.float32)).to(dev)
    ds = torch.from_numpy(rng.normal(size=(n, 48)).astype(np.float32)).to(dev)
    outs = []
    for kw in ({}, {"lambda_opacity": 0.0, "lambda_scale": 0.0}):
        leaves = {k: torch.from_numpy(v.copy()).to(dev) for k, v in params.items()}
        opt = optimizers.FusedGaussianAdam(leaves, LRS, eps=1e-15)
        opt.step(dp, ds, **kw)
        outs.append(torch.cat([leaves[k].reshape(-1) for k in ao.GROUPS]))
    assert torch.equal(outs[0], outs[1])

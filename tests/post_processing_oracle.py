"""Float64 torch restatement of the training loss with the reference's linear-to-sRGB post-processing -- TEST INFRASTRUCTURE ONLY.

The chain of the reference trainer (threedgrut/trainer.py:1150-1178, get_losses at :677-712), differentiated by torch autograd:

    c = rgb + bg (1 - alpha)                      model/background.py:80-93 (black: nothing is composited)
    x = s(c),  s = linear_to_srgb                 utils/post_processing_linear_to_srgb.py:43-67
    x, y = x m, target m                          trainer.py:691-694
    loss = lambda_l1 mean|x - y| + lambda_ssim (1 - SSIM(x, y))   trainer.py:698-739 (SSIM as oracle/loss_oracle.py states it)

with s(c) = 1.055 max(c, 1e-8)^(1/2.4) - 0.055 for c > 0.0031308 and 12.92 c otherwise (no clamp to [0, 1]).  SSIM is written here with
conv2d (11x11 Gaussian window, sigma 1.5, zero padding, 5-pixel border cropped before the mean), independently of the numpy oracle."""
import numpy as np
import torch

from oracle import loss_oracle as lo

LIMIT = 0.0031308


def linear_to_srgb(x: torch.Tensor) -> torch.Tensor:
    """The reference's encode, in the dtype of x."""
    return torch.where(x > LIMIT, 1.055 * torch.pow(torch.clamp(x, min=1e-8), 1.0 / 2.4) - 0.055, 12.92 * x)


def linear_to_srgb_slope(x):
    """s'(x) through the branch torch.where takes: (1.055 / 2.4) x^(1/2.4 - 1) above the limit, 12.92 at or below it (float64 numpy)."""
    x = np.asarray(x, np.float64)
    return np.where(x > LIMIT, (1.055 / 2.4) * np.power(np.maximum(x, 1e-8), 1.0 / 2.4 - 1.0), 12.92)


def _ssim(x, y):
    """Mean SSIM of [H,W,3] images over the valid region (conv2d restatement, float64)."""
    H, W, C = x.shape
    g = torch.as_tensor(lo.gaussian_window(), dtype=x.dtype)
    win = (g[:, None] * g[None, :]).expand(C, 1, 11, 11).contiguous()
    conv = lambda t: torch.nn.functional.conv2d(t.permute(2, 0, 1)[None], win, padding=5, groups=C)[0]  # noqa: E731
    mu1, mu2 = conv(x), conv(y)
    s1, s2, s12 = conv(x * x) - mu1 * mu1, conv(y * y) - mu2 * mu2, conv(x * y) - mu1 * mu2
    m = (2 * mu1 * mu2 + lo.C1) * (2 * s12 + lo.C2) / ((mu1 * mu1 + mu2 * mu2 + lo.C1) * (s1 + s2 + lo.C2))
    if H <= 10 or W <= 10:
        return m.sum() * 0.0
    return m[:, 5:-5, 5:-5].mean()


def loss(rgb, alpha, target, lambda_l1=0.8, lambda_ssim=0.2, background=None, mask=None, post_processing="linear-to-srgb"):
    """The scalar loss (torch, differentiable in rgb and alpha).  rgb [H,W,3], alpha [H,W,1], target [H,W,3], background None | (r, g, b) |
    [H,W,3], mask None | [H,W]; post_processing None or "linear-to-srgb"."""
    x, y = rgb, target
    if background is not None:
        x = x + torch.as_tensor(background, dtype=x.dtype).expand_as(x) * (1.0 - alpha)
    if post_processing is not None:
        x = linear_to_srgb(x)
    if mask is not None:
        m = torch.as_tensor(mask, dtype=x.dtype).reshape(x.shape[0], x.shape[1], 1)
        x, y = x * m, y * m
    l1 = (x - y).abs().mean()
    return lambda_l1 * l1 + lambda_ssim * (1.0 - _ssim(x, y))


def loss_and_gradients(rgb, alpha, target, lambda_l1=0.8, lambda_ssim=0.2, background=None, mask=None, post_processing="linear-to-srgb"):
    """numpy in, float64 out: (loss, d_rgb [H,W,3], d_alpha [H,W,1]) by autograd."""
    t = lambda a: None if a is None else torch.as_tensor(np.asarray(a, np.float64))  # noqa: E731
    r = t(rgb).requires_grad_(True)
    a = t(alpha).reshape(r.shape[0], r.shape[1], 1).clone().requires_grad_(True)
    bg = background if background is None or isinstance(background, tuple) else t(background)
    value = loss(r, a, t(target), lambda_l1, lambda_ssim, bg, t(mask), post_processing)
    value.backward()
    d_alpha = np.zeros(a.shape) if a.grad is None else a.grad.numpy()  # black: alpha takes no part
    return float(value), r.grad.numpy(), d_alpha

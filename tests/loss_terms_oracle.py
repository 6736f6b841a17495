"""CPU restatement (numpy) of the parts of the reference training loss beyond L1 + SSIM -- TEST INFRASTRUCTURE ONLY.

Builds on oracle/loss_oracle.py and oracle/adam_oracle.py, which it leaves as they are:
  * background compositing (threedgrut/model/background.py:80-93):  x = rgb + bg (1 - alpha)   (black: nothing is composited)
  * image mask (threedgrut/trainer.py:691-694):                      x, y = x m, y m
    d rgb = m dL/dx,  d alpha = -sum_c bg_c m dL/dx_c
  * opacity and scale regularisers (trainer.py:722-736):
        lambda_opacity mean|sigmoid(raw density)| + lambda_scale mean|exp(raw scale)|
    i.e. + lambda_opacity / N on every activated density gradient and + lambda_scale / (3 N) on every activated scale gradient, before the
    activation chain rule.
Pinned by tests/test_loss_terms_oracle.py against torch autograd of the reference's formulas."""
import numpy as np

from oracle import adam_oracle as ao
from oracle import loss_oracle as lo

f32 = np.float32


def composite(rgb, alpha, background=None, mask=None, target=None, dtype=np.float64, device_rounding=False):
    """(x, y) as the loss sees them.  rgb [H,W,3], alpha [H,W,1], background None | (r, g, b) | [H,W,3], mask None | [H,W].
    device_rounding: round the composite to float32 once, as the device's fused multiply-add does (x + bg * (1 - alpha) with 1 - alpha
    in float32), so that the L1 term takes the sign of the same x - y where the two are within an ulp of each other."""
    x = np.asarray(rgb, dtype)
    if background is not None:
        bg = np.broadcast_to(np.asarray(background, dtype), x.shape)
        a = np.asarray(alpha, dtype).reshape(x.shape[:2] + (1,))
        if device_rounding:
            one_minus = (f32(1) - a.astype(f32)).astype(np.float64)
            x = (x.astype(np.float64) + bg.astype(f32).astype(np.float64) * one_minus).astype(f32).astype(dtype)
        else:
            x = x + bg * (1.0 - a)
    y = None if target is None else np.asarray(target, dtype)
    if mask is not None:
        m = np.asarray(mask, dtype).reshape(x.shape[:2] + (1,))
        x = x * m
        y = None if y is None else y * m
    return x, y


def composited_loss_and_gradients(rgb, alpha, target, lambda_l1=0.8, lambda_ssim=0.2, background=None, mask=None, dtype=np.float64,
                                  device_rounding=False):
    """Returns (loss, l1, ssim, d_rgb [H,W,3], d_alpha [H,W,1]).  With no background and no mask this is loss_oracle.loss_and_gradient
    with a zero alpha gradient."""
    x, y = composite(rgb, alpha, background, mask, target, dtype, device_rounding)
    loss, l1, ssim, gx = lo.loss_and_gradient(x, y, lambda_l1, lambda_ssim, dtype)
    if mask is not None:
        gx = gx * np.asarray(mask, dtype).reshape(x.shape[:2] + (1,))
    d_alpha = np.zeros(x.shape[:2] + (1,), dtype)
    if background is not None:
        bg = np.broadcast_to(np.asarray(background, dtype), x.shape)
        d_alpha = -(bg * gx).sum(-1, keepdims=True)
    return loss, l1, ssim, gx, d_alpha


def regulariser_loss(params, lambda_opacity=0.0, lambda_scale=0.0):
    """lambda_opacity mean|sigmoid(density)| + lambda_scale mean|exp(scale)| on the raw parameters (float64)."""
    d = np.asarray(params["density"], np.float64)
    s = np.asarray(params["scale"], np.float64)
    return lambda_opacity * np.abs(1.0 / (1.0 + np.exp(-d))).mean() + lambda_scale * np.abs(np.exp(s)).mean()


def raw_gradients(params, d_particles, d_sph, lambda_opacity=0.0, lambda_scale=0.0):
    """adam_oracle.raw_gradients with the regularisers added to the activated density / scale gradients before the chain rule."""
    dp = np.array(d_particles, f32)
    n = dp.shape[0]
    if lambda_opacity != 0.0:
        dp[:, 3] = dp[:, 3] + f32(lambda_opacity / n)
    if lambda_scale != 0.0:
        dp[:, 8:11] = dp[:, 8:11] + f32(lambda_scale / (3 * n))
    return ao.raw_gradients(params, dp, d_sph)


def gaussian_adam_step(params, moments_m, moments_v, lrs, d_particles, d_sph, b1=0.9, b2=0.999, eps=1e-15, step=1, selective=False,
                       visibility=None, lambda_opacity=0.0, lambda_scale=0.0):
    """adam_oracle.gaussian_adam_step with the regularisers.  Returns new (params, m, v) dicts."""
    grads = raw_gradients(params, d_particles, d_sph, lambda_opacity, lambda_scale)
    out_p, out_m, out_v = {}, {}, {}
    for name in ao.GROUPS:
        out_p[name], out_m[name], out_v[name] = ao.adam_update(params[name], grads[name], moments_m[name], moments_v[name], lrs[name], b1, b2,
                                                               eps, step, selective, visibility)
    return out_p, out_m, out_v

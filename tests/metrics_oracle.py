"""Float64 numpy restatement of the test-set metrics of a frame (csrc/gut_metrics.cu) -- TEST INFRASTRUCTURE ONLY.

    x = s(rgb + bg (1 - alpha))          composite (model/background.py:80-93; black adds nothing), then post-processing (render.py:294-307)
    psnr = 10 log10(1 / mean (x - y)^2)  torchmetrics PeakSignalNoiseRatio(data_range=1), x unclipped (render.py:327)
    ssim                                 torchmetrics StructuralSimilarityIndexMeasure(data_range=1.0): loss_oracle's window and constants,
                                         both variances clamped at 0, mean over the interior (reflect pad 5 + crop 5 = the valid region)
    color_correct_affine(x, y)           threedgrut/utils/color_correct.py:96-145, moments over all HW pixels
    quantise(v)                          torchvision.utils.save_image: trunc(clamp(fl32(fl32(v 255) + 0.5), 0, 255))

torchmetrics and torchvision are not needed: the definitions above are the pin, and tests/test_metrics_oracle.py checks the pieces that
can be checked here against loss_oracle and a transcription of color_correct.py."""
import numpy as np

from oracle import loss_oracle as lo


def linear_to_srgb(x):
    x = np.asarray(x, np.float64)
    return np.where(x > 0.0031308, 1.055 * np.power(np.maximum(x, 1e-8), 1.0 / 2.4) - 0.055, 12.92 * x)


def prediction(rgb, alpha=None, background=None, post_processing=None):
    """x of the metrics in float64: rgb [H,W,3] composited onto the constant background (None = black) with alpha [H,W] / [H,W,1], then
    post-processed (None or "linear-to-srgb")."""
    x = np.asarray(rgb, np.float64)
    if background is not None:
        a = np.asarray(alpha, np.float64).reshape(x.shape[0], x.shape[1], 1)
        x = x + np.asarray(background, np.float64)[None, None, :] * (1.0 - a)
    if post_processing == "linear-to-srgb":
        x = linear_to_srgb(x)
    return x


def psnr(x, y):
    mse = float(np.mean((np.asarray(x, np.float64) - np.asarray(y, np.float64)) ** 2))
    return float("inf") if mse == 0.0 else 10.0 * np.log10(1.0 / mse)


def ssim_map(x, y):
    """The SSIM map with the variances clamped at 0 (torchmetrics), float64, same-size; only the interior [5:-5, 5:-5] is meaningful."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    w = lo.gaussian_window()
    mu1, mu2 = lo._conv(x, w), lo._conv(y, w)
    s1 = np.maximum(lo._conv(x * x, w) - mu1 * mu1, 0.0)
    s2 = np.maximum(lo._conv(y * y, w) - mu2 * mu2, 0.0)
    s12 = lo._conv(x * y, w) - mu1 * mu2
    return (2 * mu1 * mu2 + lo.C1) * (2 * s12 + lo.C2) / ((mu1 * mu1 + mu2 * mu2 + lo.C1) * (s1 + s2 + lo.C2))


def ssim(x, y):
    H, W = np.shape(x)[:2]
    if H < 11 or W < 11:
        raise ValueError("SSIM needs at least 11 x 11 pixels")
    return float(ssim_map(x, y)[5:-5, 5:-5].mean())


def affine(x, y):
    """(a, b) per channel of color_correct_affine(x, y) in float64; b takes the slope before |a| < 1e-8 is replaced by 1."""
    xm, ym = np.asarray(x, np.float64).reshape(-1, 3), np.asarray(y, np.float64).reshape(-1, 3)
    ey, ex = ym.mean(0), xm.mean(0)
    exy, eyy = (ym * xm).mean(0), (ym * ym).mean(0)
    var = np.maximum(eyy - ey * ey, 1e-8)
    a = (exy - ey * ex) / var
    b = ex - a * ey
    a = np.where(np.abs(a) < 1e-8, 1.0, a)
    return a, b


def color_correct(x, y, a=None, b=None):
    """x_cc = clip((x - b) / a, 0, 1), computed as the kernel does: a, b rounded to float32, x in float32, IEEE float32 operations."""
    if a is None:
        a, b = affine(x, y)
    x32 = np.asarray(x, np.float32)
    return np.clip((x32 - np.float32(b)) / np.float32(a), np.float32(0), np.float32(1)).astype(np.float64)


def quantise(v):
    """uint8 bytes of torchvision.utils.save_image: mul(255), add(0.5), clamp(0, 255), cast (truncation), each step rounded to float32."""
    v = np.asarray(v, np.float32)
    s = np.clip((v * np.float32(255.0)).astype(np.float32) + np.float32(0.5), np.float32(0.0), np.float32(255.0))
    return s.astype(np.uint8)


def hit_stats(hits):
    h = np.asarray(hits, np.float64).ravel()
    return {"hits_mean": float(h.mean()), "hits_std": float(h.std(ddof=1)), "hits_min": float(h.min()), "hits_max": float(h.max())}


def frame_metrics(x, y, x32=None):
    """Every metric of one frame from x (the prediction the metrics see) and y, float64.  x32: x as the device holds it (float32), from
    which the colour-corrected image is made; defaults to x rounded to float32."""
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    a, b = affine(x, y)
    xcc = color_correct(x if x32 is None else x32, y, a, b)
    return {"psnr": psnr(x, y), "ssim": ssim(x, y), "cc_psnr": psnr(xcc, y), "cc_ssim": ssim(xcc, y), "l1": float(np.abs(x - y).mean()),
            "a": a, "b": b}

"""Image loss of the training step on the GPU (SURVEY.md section 8f row 3): lambda_l1 * L1 + lambda_ssim * (1 - SSIM) and its gradient
w.r.t. the rendered image in two launches (csrc/gut_loss.cu), replacing l1_loss + fused_ssim + their autograd
(threedgrut/model/losses.py:20-33, trainer.py:698-739).  The gradient comes out as [H,W,4] with a zero alpha gradient, i.e. directly the
`ray_radiance_density_grd` / d_rgba argument of SplatRaster.trace_bwd; image_loss_rgb takes and returns the 3DGRT layout (rgb [H,W,3]).

With `background=` and / or `mask=`, the loss is taken on the prediction composited onto the background and multiplied by the mask, as the
reference trainer does (model/background.py:80-93, trainer.py:691-694), in the same two launches (gutb200_image_loss_composited): the
gradient then has a live alpha part.  image_loss_rgb_alpha is that loss on the 3DGRT layout (rgb and alpha as separate tensors).
`Background` and `mask_hw` resolve the training steps' `background=` / `mask=` arguments.  No CPU fallback."""
from __future__ import annotations

import ctypes as C

import torch

import b200_native as native

_scratch = {}


def _check_image(t, what, ch):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.dim() == 3 and t.shape[2] == ch):
        raise RuntimeError(f"{what}: expected a contiguous float32 CUDA tensor [H,W,{ch}] (there is no CPU fallback)")


def _scratch_for(lib, dev, H, W):
    need = int(lib.gutb200_image_loss_scratch_bytes(H, W))
    key = (dev.index, H, W)
    if key not in _scratch or _scratch[key].numel() * 4 < need:
        _scratch[key] = torch.empty((need + 3) // 4, dtype=torch.float32, device=dev)
    return _scratch[key]


def _scalars(sums, H, W, lambda_l1, lambda_ssim):
    l1 = sums[0] / (3.0 * H * W)
    ssim = sums[1] / (3.0 * max(H - 10, 1) * max(W - 10, 1)) if (H > 10 and W > 10) else sums[1] * 0.0
    loss = lambda_l1 * l1 + lambda_ssim * (1.0 - ssim)
    return loss, l1, ssim


def _run(entry, pred, tgt, ch_pred, lambda_l1, lambda_ssim, d_pred, name):
    for t, w, ch in ((pred, name, ch_pred), (tgt, "target_rgb", 3)):
        _check_image(t, w, ch)
    H, W = int(pred.shape[0]), int(pred.shape[1])
    if tuple(tgt.shape[:2]) != (H, W):
        raise RuntimeError("prediction and target resolutions differ")
    dev = pred.device
    lib = native.load()
    scratch = _scratch_for(lib, dev, H, W)
    if d_pred is None:
        d_pred = torch.empty((H, W, ch_pred), dtype=torch.float32, device=dev)
    sums = torch.empty(2, dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        rc = getattr(lib, entry)(stream, H, W, pred.data_ptr(), tgt.data_ptr(), float(lambda_l1), float(lambda_ssim), scratch.data_ptr(),
                                 d_pred.data_ptr(), sums.data_ptr())
    if rc != 0:
        raise RuntimeError(f"{entry} failed ({rc})")
    return (*_scalars(sums, H, W, lambda_l1, lambda_ssim), d_pred)


def _run_composited(layout, pred, alpha, tgt, lambda_l1, lambda_ssim, background, mask, d_pred, d_alpha):
    """gutb200_image_loss_composited.  background: None (black), 3 floats, or a float32 CUDA image [H,W,3]; mask: None or [H,W]."""
    _check_image(pred, "pred_rgba" if layout == 4 else "pred_rgb", layout)
    _check_image(tgt, "target_rgb", 3)
    H, W = int(pred.shape[0]), int(pred.shape[1])
    if tuple(tgt.shape[:2]) != (H, W):
        raise RuntimeError("prediction and target resolutions differ")
    dev = pred.device
    bg_rgb, bg_img = None, None
    if isinstance(background, torch.Tensor):
        bg_img = background.reshape(background.shape[-3:]) if background.dim() == 4 else background
        _check_image(bg_img, "background", 3)
        if tuple(bg_img.shape[:2]) != (H, W) or bg_img.device != dev:
            raise RuntimeError("background image: expected [H,W,3] on the prediction's device")
    elif background is not None:
        rgb = [float(v) for v in background]
        if len(rgb) != 3:
            raise RuntimeError("background: expected three floats (r, g, b) or an [H,W,3] image")
        bg_rgb = (C.c_float * 3)(*rgb)
    if mask is not None:
        mask = mask_hw(mask, H, W)
        if mask.device != dev:
            raise RuntimeError("mask: expected a tensor on the prediction's device")
    lib = native.load()
    scratch = _scratch_for(lib, dev, H, W)
    if d_pred is None:
        d_pred = torch.empty((H, W, layout), dtype=torch.float32, device=dev)
    if layout == 3 and d_alpha is None:
        d_alpha = torch.empty((H, W, 1), dtype=torch.float32, device=dev)
    sums = torch.empty(2, dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    ptr = lambda t: None if t is None else t.data_ptr()  # noqa: E731
    with torch.cuda.device(dev):
        rc = lib.gutb200_image_loss_composited(stream, H, W, layout, pred.data_ptr(), ptr(alpha), tgt.data_ptr(), bg_rgb, ptr(bg_img), ptr(mask),
                                               float(lambda_l1), float(lambda_ssim), scratch.data_ptr(), d_pred.data_ptr(), ptr(d_alpha),
                                               sums.data_ptr())
    if rc != 0:
        raise RuntimeError(f"gutb200_image_loss_composited failed ({rc})")
    return (*_scalars(sums, H, W, lambda_l1, lambda_ssim), d_pred, d_alpha)


def image_loss(pred_rgba: torch.Tensor, target_rgb: torch.Tensor, lambda_l1: float = 0.8, lambda_ssim: float = 0.2, d_rgba: torch.Tensor | None = None,
               background=None, mask: torch.Tensor | None = None):
    """pred_rgba [H,W,4] (or [1,H,W,4]), target_rgb [H,W,3] float32 CUDA tensors.
    Returns (loss, l1, ssim, d_rgba): three device scalars and d loss / d pred_rgba [H,W,4].
    background: None (black), (r, g, b), or a float32 CUDA image [H,W,3]; mask: None or a float CUDA tensor [H,W] ([H,W,1], [1,H,W,1]).
    With either, the loss is taken on (rgb + background (1 - alpha)) * mask against target * mask and d_rgba carries the alpha gradient."""
    pred = pred_rgba.reshape(pred_rgba.shape[-3:])
    tgt = target_rgb.reshape(target_rgb.shape[-3:])
    if background is None and mask is None:
        return _run("gutb200_image_loss", pred, tgt, 4, lambda_l1, lambda_ssim, d_rgba, "pred_rgba")
    return _run_composited(4, pred, None, tgt, lambda_l1, lambda_ssim, background, mask, d_rgba, None)[:4]


def image_loss_rgb(pred_rgb: torch.Tensor, target_rgb: torch.Tensor, lambda_l1: float = 0.8, lambda_ssim: float = 0.2, d_rgb: torch.Tensor | None = None):
    """The same loss on the 3DGRT layout: pred_rgb [H,W,3] (or [1,H,W,3], the tracer's rgb output; its alpha takes no part), target_rgb
    [H,W,3].  Returns (loss, l1, ssim, d_rgb) with d_rgb [H,W,3] -- directly the rgb gradient of OptixTracer.trace_bwd.  Bit-identical to
    image_loss on cat([rgb, alpha], -1)."""
    pred = pred_rgb.reshape(pred_rgb.shape[-3:])
    tgt = target_rgb.reshape(target_rgb.shape[-3:])
    return _run("gutb200_image_loss_rgb", pred, tgt, 3, lambda_l1, lambda_ssim, d_rgb, "pred_rgb")


def image_loss_rgb_alpha(pred_rgb: torch.Tensor, pred_alpha: torch.Tensor, target_rgb: torch.Tensor, lambda_l1: float = 0.8,
                         lambda_ssim: float = 0.2, background=None, mask: torch.Tensor | None = None, d_rgb: torch.Tensor | None = None,
                         d_alpha: torch.Tensor | None = None):
    """The composited, masked loss on the 3DGRT layout: pred_rgb [H,W,3] and pred_alpha [H,W,1] (or [1,H,W,3] / [1,H,W,1], the tracer's
    outputs), target_rgb [H,W,3]; background / mask as in image_loss.  Returns (loss, l1, ssim, d_rgb [H,W,3], d_alpha [H,W,1]) -- directly
    the rgb and alpha gradients of OptixTracer.trace_bwd.  A black background with no mask gives d_rgb of image_loss_rgb and d_alpha = 0."""
    pred = pred_rgb.reshape(pred_rgb.shape[-3:])
    tgt = target_rgb.reshape(target_rgb.shape[-3:])
    H, W = int(pred.shape[0]), int(pred.shape[1])
    if not (isinstance(pred_alpha, torch.Tensor) and pred_alpha.is_cuda and pred_alpha.dtype == torch.float32 and pred_alpha.is_contiguous()
            and pred_alpha.numel() == H * W and pred_alpha.shape[-1] == 1):
        raise RuntimeError("pred_alpha: expected a contiguous float32 CUDA tensor [H,W,1] (there is no CPU fallback)")
    return _run_composited(3, pred, pred_alpha, tgt, lambda_l1, lambda_ssim, background, mask, d_rgb, d_alpha)


def mask_hw(mask: torch.Tensor, H: int, W: int) -> torch.Tensor:
    """A loss mask given as [H,W], [H,W,1] or [1,H,W,1] (a floating-point CUDA tensor) as a contiguous float32 [H,W] tensor."""
    if not isinstance(mask, torch.Tensor) or not mask.is_cuda or not mask.is_floating_point():
        raise RuntimeError("mask: expected a floating-point CUDA tensor (there is no CPU fallback)")
    if tuple(mask.shape) not in ((H, W), (H, W, 1), (1, H, W, 1)):
        raise RuntimeError(f"mask: expected shape [H,W], [H,W,1] or [1,H,W,1] with H, W = {H}, {W}; got {tuple(mask.shape)}")
    return mask.reshape(H, W).to(torch.float32).contiguous()


class Background:
    """The background a training step composites the render onto before the loss (model.background.color, configs/base_gs.yaml:125-127):
    "black" (nothing is composited), "white", "random" (a fresh U[0,1) colour per pixel and channel every step, background.py:83-91), or
    an (r, g, b) colour.  "random" draws from a generator of its own on `device`, seeded `seed`."""

    NAMES = ("black", "white", "random")

    def __init__(self, background="black", seed: int = 0, device=None):
        if isinstance(background, str):
            if background not in self.NAMES:
                raise ValueError(f"background: unknown name {background!r} (expected one of {', '.join(self.NAMES)} or an (r, g, b) colour)")
            self.color = {"black": (0.0, 0.0, 0.0), "white": (1.0, 1.0, 1.0), "random": None}[background]
        else:
            rgb = tuple(float(v) for v in background)
            if len(rgb) != 3:
                raise ValueError("background: expected a name or an (r, g, b) colour")
            self.color = rgb
        self.random = self.color is None
        self.black = self.color == (0.0, 0.0, 0.0)
        self.device = device
        self.generator = None
        self.image = None  # the latest random draw [H,W,3]
        if self.random:
            self.generator = torch.Generator(device=device)
            self.generator.manual_seed(int(seed))

    def draw(self, H: int, W: int):
        """None for black, the colour, or this step's random image [H,W,3] (drawn into a buffer that the next draw overwrites)."""
        if self.black:
            return None
        if not self.random:
            return self.color
        if self.image is None or tuple(self.image.shape) != (H, W, 3):
            self.image = torch.empty((H, W, 3), dtype=torch.float32, device=self.device)
        torch.rand((H, W, 3), generator=self.generator, out=self.image)
        return self.image

"""Image loss of the training step on the GPU (SURVEY.md section 8f row 3): lambda_l1 * L1 + lambda_ssim * (1 - SSIM) and its gradient
w.r.t. the rendered image in two launches of one C entry point (gutb200_image_loss, csrc/gut_loss.cu), replacing l1_loss + fused_ssim +
their autograd (threedgrut/model/losses.py:20-33, trainer.py:698-739).  The gradient comes out as [H,W,4] with a zero alpha gradient, i.e.
directly the `ray_radiance_density_grd` / d_rgba argument of SplatRaster.trace_bwd; image_loss_rgb takes and returns the 3DGRT layout (rgb
[H,W,3]).

With `background=` and / or `mask=`, the loss is taken on the prediction composited onto the background and multiplied by the mask, as the
reference trainer does (model/background.py:80-93, trainer.py:691-694), in the same two launches: the gradient then has a live alpha part.
image_loss_rgb_alpha is that loss on the 3DGRT layout (rgb and alpha as separate tensors).
`Background` and `mask_hw` resolve the training steps' `background=` / `mask=` arguments.

With `post_processing="linear-to-srgb"` (the reference's post_processing.method, configs/base_gs.yaml:188-197), the composited prediction is
encoded to sRGB before the mask and the loss (threedgrut/utils/post_processing_linear_to_srgb.py, trainer.py:1165-1172), still in the same
two launches: use it when the ground-truth images are display-referred sRGB and the renderer outputs linear radiance.  `linear_to_srgb` is
that encode for rendered images outside the loss.  No CPU fallback."""
from __future__ import annotations

import ctypes as C

import torch

import b200_native as native

_scratch = {}

POST_PROCESSING = {None: 0, "linear-to-srgb": 1}  # post_processing.method -> the post_processing code of gutb200_image_loss


def post_processing_code(method) -> int:
    """The device code of a post_processing.method: None -> 0, "linear-to-srgb" -> 1.  "ppisp" (a third-party package) and any other value
    raise NotImplementedError naming the key.  Pure config logic: needs no GPU."""
    if method is None or (isinstance(method, str) and method in POST_PROCESSING):
        return POST_PROCESSING[method]
    raise NotImplementedError(f"post_processing.method={method!r}: only null and 'linear-to-srgb' are built (PPISP is not)")


def linear_to_srgb(x: torch.Tensor) -> torch.Tensor:
    """Linear RGB -> sRGB, elementwise, as the reference Renderer applies post_processing.method linear-to-srgb to a rendered image
    (render.py:307, post_processing_linear_to_srgb.py:43-67): 1.055 max(x, 1e-8)^(1/2.4) - 0.055 where x > 0.0031308, else 12.92 x; no
    clamp, so values above 1 encode above 1.  Same shape, dtype and device as x."""
    return torch.where(x > 0.0031308, 1.055 * torch.pow(torch.clamp(x, min=1e-8), 1.0 / 2.4) - 0.055, 12.92 * x)


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


def _run(layout, pred, tgt, lambda_l1, lambda_ssim, d_pred, alpha=None, d_alpha=None, background=None, mask=None, post=0):
    """One call of gutb200_image_loss.  layout 4: pred [H,W,4]; layout 3: pred [H,W,3] and alpha [H,W,1] or None (image_loss_rgb: black and
    unmasked, the alpha is never read).  background: None (black), 3 floats, or a float32 CUDA image [H,W,3]; mask: None or as mask_hw.
    Returns (loss, l1, ssim, d_pred, d_alpha); layout 3 allocates d_alpha [H,W,1] when it is None and alpha is given (it is returned) or the
    post-processing writes it."""
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
        bg_img = bg_img.data_ptr()
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
    if layout == 3 and d_alpha is None and (alpha is not None or post):
        d_alpha = torch.empty((H, W, 1), dtype=torch.float32, device=dev)
    sums = torch.empty(2, dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        rc = lib.gutb200_image_loss(stream, H, W, layout, pred.data_ptr(), None if alpha is None else alpha.data_ptr(), tgt.data_ptr(), bg_rgb,
                                    bg_img, None if mask is None else mask.data_ptr(), float(lambda_l1), float(lambda_ssim), scratch.data_ptr(),
                                    d_pred.data_ptr(), None if d_alpha is None else d_alpha.data_ptr(), sums.data_ptr(), post)
    if rc != 0:
        raise RuntimeError(f"gutb200_image_loss failed ({rc}): {lib.gutb200_last_error(None).decode()}")
    return (*_scalars(sums, H, W, lambda_l1, lambda_ssim), d_pred, d_alpha)


def image_loss(pred_rgba: torch.Tensor, target_rgb: torch.Tensor, lambda_l1: float = 0.8, lambda_ssim: float = 0.2, d_rgba: torch.Tensor | None = None,
               background=None, mask: torch.Tensor | None = None, post_processing=None):
    """pred_rgba [H,W,4] (or [1,H,W,4]), target_rgb [H,W,3] float32 CUDA tensors.
    Returns (loss, l1, ssim, d_rgba): three device scalars and d loss / d pred_rgba [H,W,4].
    background: None (black), (r, g, b), or a float32 CUDA image [H,W,3]; mask: None or a float CUDA tensor [H,W] ([H,W,1], [1,H,W,1]).
    With either, the loss is taken on (rgb + background (1 - alpha)) * mask against target * mask and d_rgba carries the alpha gradient.
    post_processing: None or "linear-to-srgb" (the composite is encoded to sRGB before the mask; see linear_to_srgb)."""
    post = post_processing_code(post_processing)
    pred = pred_rgba.reshape(pred_rgba.shape[-3:])
    tgt = target_rgb.reshape(target_rgb.shape[-3:])
    return _run(4, pred, tgt, lambda_l1, lambda_ssim, d_rgba, background=background, mask=mask, post=post)[:4]


def image_loss_rgb(pred_rgb: torch.Tensor, target_rgb: torch.Tensor, lambda_l1: float = 0.8, lambda_ssim: float = 0.2, d_rgb: torch.Tensor | None = None,
                   post_processing=None):
    """The same loss on the 3DGRT layout: pred_rgb [H,W,3] (or [1,H,W,3], the tracer's rgb output; its alpha takes no part), target_rgb
    [H,W,3].  Returns (loss, l1, ssim, d_rgb) with d_rgb [H,W,3] -- directly the rgb gradient of OptixTracer.trace_bwd.  Bit-identical to
    image_loss on cat([rgb, alpha], -1).  post_processing as in image_loss."""
    post = post_processing_code(post_processing)
    pred = pred_rgb.reshape(pred_rgb.shape[-3:])
    tgt = target_rgb.reshape(target_rgb.shape[-3:])
    return _run(3, pred, tgt, lambda_l1, lambda_ssim, d_rgb, post=post)[:4]


def image_loss_rgb_alpha(pred_rgb: torch.Tensor, pred_alpha: torch.Tensor, target_rgb: torch.Tensor, lambda_l1: float = 0.8,
                         lambda_ssim: float = 0.2, background=None, mask: torch.Tensor | None = None, d_rgb: torch.Tensor | None = None,
                         d_alpha: torch.Tensor | None = None, post_processing=None):
    """The composited, masked loss on the 3DGRT layout: pred_rgb [H,W,3] and pred_alpha [H,W,1] (or [1,H,W,3] / [1,H,W,1], the tracer's
    outputs), target_rgb [H,W,3]; background / mask as in image_loss.  Returns (loss, l1, ssim, d_rgb [H,W,3], d_alpha [H,W,1]) -- directly
    the rgb and alpha gradients of OptixTracer.trace_bwd.  A black background with no mask gives d_rgb of image_loss_rgb and d_alpha = 0.
    post_processing as in image_loss."""
    post = post_processing_code(post_processing)
    pred = pred_rgb.reshape(pred_rgb.shape[-3:])
    tgt = target_rgb.reshape(target_rgb.shape[-3:])
    H, W = int(pred.shape[0]), int(pred.shape[1])
    if not (isinstance(pred_alpha, torch.Tensor) and pred_alpha.is_cuda and pred_alpha.dtype == torch.float32 and pred_alpha.is_contiguous()
            and pred_alpha.numel() == H * W and pred_alpha.shape[-1] == 1):
        raise RuntimeError("pred_alpha: expected a contiguous float32 CUDA tensor [H,W,1] (there is no CPU fallback)")
    return _run(3, pred, tgt, lambda_l1, lambda_ssim, d_rgb, alpha=pred_alpha, d_alpha=d_alpha, background=background, mask=mask, post=post)


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
        self.seed = int(seed)
        self.generator = None
        self.image = None  # the latest random draw [H,W,3]
        if self.random:
            self.generator = torch.Generator(device=device)
            self.generator.manual_seed(self.seed)

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

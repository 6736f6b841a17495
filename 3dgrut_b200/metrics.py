"""Test-set metrics of a rendered frame on the GPU: PSNR, SSIM, their colour-corrected twins, the mean L1, the hit statistics and the PNG
bytes, as the reference evaluator computes them (threedgrut/render.py:294-369, trainer.py:641-657) -- one C entry point,
gutb200_image_metrics (csrc/gut_metrics.cu), four launches and no host synchronisation.  The values land in a device float64 row of
FIELDS, so a pass over many frames fills one [F, K] tensor and copies it to the host once.  No CPU fallback."""
from __future__ import annotations

import ctypes as C

import torch

import b200_native as native
import losses

# the fields of one row of `out`, in the order of include/gut_b200.h's GUTB200_METRIC_* enum
FIELDS = ("psnr", "ssim", "cc_psnr", "cc_ssim", "l1", "hits_mean", "hits_std", "hits_min", "hits_max", "a_r", "a_g", "a_b", "b_r", "b_g", "b_b")
K = len(FIELDS)
MIN_SIZE = 11  # torchmetrics' SSIM reflect-pads and crops 5 pixels: no interior below 11 x 11

_scratch = {}


def _scratch_for(lib, dev, H, W):
    need = int(lib.gutb200_image_metrics_scratch_bytes(H, W))
    key = (dev.index, H, W)
    if key not in _scratch:
        _scratch[key] = torch.empty((need + 7) // 8, dtype=torch.float64, device=dev)
    return _scratch[key]


def background_rgb(background):
    """The constant colour evaluation composites onto: None / "black" / "random" -> None (nothing is composited: the reference's
    BackgroundColor.forward(train=False) adds no random colour), "white" -> (1, 1, 1), (r, g, b) -> itself; a losses.Background likewise."""
    if isinstance(background, losses.Background):
        return None if background.random or background.black else tuple(background.color)
    if background is None or (isinstance(background, str) and background in ("black", "random")):
        return None
    if isinstance(background, str):
        if background == "white":
            return (1.0, 1.0, 1.0)
        raise ValueError(f"background: unknown name {background!r} (expected black, white, random or an (r, g, b) colour)")
    rgb = tuple(float(v) for v in background)
    if len(rgb) != 3:
        raise ValueError("background: expected a name or three floats (r, g, b)")
    return None if rgb == (0.0, 0.0, 0.0) else rgb


def image_metrics(pred: torch.Tensor, target: torch.Tensor, alpha: torch.Tensor | None = None, background=None, post_processing=None,
                  hits: torch.Tensor | None = None, out: torch.Tensor | None = None, png: bool = False):
    """Metrics of one frame.  pred: float32 CUDA [H,W,4] rgba (the 3DGUT layout) or [H,W,3] rgb with alpha [H,W] / [H,W,1] (the 3DGRT
    layout; [1,H,W,C] is accepted); target: [H,W,3].  background: None / "black" / "random" (nothing composited), "white" or (r, g, b);
    post_processing: None or "linear-to-srgb", applied after the composite.  hits: the hit counts [H,W] (any shape of H*W elements, any
    dtype; rounded to int32) or None.  out: a contiguous float64 CUDA tensor of K elements (e.g. a row of [F, K]) or None (allocated).
    png: also return the quantised bytes of the prediction and the target as uint8 [H,W,3].
    Returns out (device, FIELDS order), or (out, pred_u8, target_u8) with png.  Raises ValueError below 11 x 11 pixels."""
    post = losses.post_processing_code(post_processing)
    pred = pred.reshape(pred.shape[-3:]) if pred.dim() == 4 else pred
    target = target.reshape(target.shape[-3:]) if target.dim() == 4 else target
    if pred.dim() != 3 or pred.shape[2] not in (3, 4):
        raise RuntimeError("pred: expected [H,W,4] rgba or [H,W,3] rgb")
    layout = int(pred.shape[2])
    losses._check_image(pred, "pred", layout)
    losses._check_image(target, "target_rgb", 3)
    H, W = int(pred.shape[0]), int(pred.shape[1])
    if tuple(target.shape[:2]) != (H, W) or target.device != pred.device:
        raise RuntimeError("prediction and target: expected the same resolution on the same device")
    if H < MIN_SIZE or W < MIN_SIZE:
        raise ValueError(f"image_metrics: {H}x{W} pixels; SSIM needs at least {MIN_SIZE}x{MIN_SIZE} (reflect pad and crop of 5)")
    dev = pred.device
    bg = background_rgb(background)
    if layout == 3 and bg is not None:
        if alpha is None:
            raise RuntimeError("alpha: the rgb layout needs the render's alpha to composite a background")
    if alpha is not None:
        if not (isinstance(alpha, torch.Tensor) and alpha.is_cuda and alpha.dtype == torch.float32 and alpha.is_contiguous()
                and alpha.numel() == H * W and alpha.device == dev):
            raise RuntimeError("alpha: expected a contiguous float32 CUDA tensor of H*W elements on the prediction's device")
    if hits is not None:
        if not (isinstance(hits, torch.Tensor) and hits.numel() == H * W and hits.device == dev):
            raise RuntimeError("hits: expected a CUDA tensor of H*W elements on the prediction's device")
        hits = hits.reshape(H, W).to(torch.int32).contiguous()
    if out is None:
        out = torch.empty(K, dtype=torch.float64, device=dev)
    elif not (out.is_cuda and out.dtype == torch.float64 and out.is_contiguous() and out.numel() == K and out.device == dev):
        raise RuntimeError(f"out: expected a contiguous float64 CUDA tensor of {K} elements on the prediction's device")
    pred_u8 = target_u8 = None
    if png:
        pred_u8 = torch.empty((H, W, 3), dtype=torch.uint8, device=dev)
        target_u8 = torch.empty((H, W, 3), dtype=torch.uint8, device=dev)
    lib = native.load()
    scratch = _scratch_for(lib, dev, H, W)
    bg_arg = None if bg is None else (C.c_float * 3)(*bg)
    stream = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        rc = lib.gutb200_image_metrics(stream, H, W, layout, pred.data_ptr(), None if alpha is None else alpha.data_ptr(), target.data_ptr(),
                                       bg_arg, post, None if hits is None else hits.data_ptr(), scratch.data_ptr(), out.data_ptr(),
                                       None if pred_u8 is None else pred_u8.data_ptr(), None if target_u8 is None else target_u8.data_ptr())
    if rc != 0:
        msg = f"gutb200_image_metrics failed ({rc}): {lib.gutb200_last_error(None).decode()}"
        raise ValueError(msg) if rc == 1 else RuntimeError(msg)
    return (out, pred_u8, target_u8) if png else out


def as_dict(row) -> dict:
    """A host row of FIELDS (numpy or a list) as {field: float}."""
    return {k: float(v) for k, v in zip(FIELDS, row)}

"""Image loss of the training step on the GPU (SURVEY.md section 8f row 3): lambda_l1 * L1 + lambda_ssim * (1 - SSIM) and its gradient
w.r.t. the rendered image in two launches (csrc/gut_loss.cu), replacing l1_loss + fused_ssim + their autograd
(threedgrut/model/losses.py:20-33, trainer.py:698-739).  The gradient comes out as [H,W,4] with a zero alpha gradient, i.e. directly the
`ray_radiance_density_grd` / d_rgba argument of SplatRaster.trace_bwd; image_loss_rgb takes and returns the 3DGRT layout (rgb [H,W,3]).
No CPU fallback."""
from __future__ import annotations

import ctypes as C

import torch

import b200_native as native

_scratch = {}


def _lib():
    lib = native.load()
    if not getattr(lib, "_loss_bound", False):
        vp, i32, f32 = C.c_void_p, C.c_int32, C.c_float
        lib.gutb200_image_loss_scratch_bytes.argtypes = [i32, i32]
        lib.gutb200_image_loss_scratch_bytes.restype = C.c_size_t
        lib.gutb200_image_loss.argtypes = [vp, i32, i32, vp, vp, f32, f32, vp, vp, vp]
        lib.gutb200_image_loss.restype = C.c_int
        lib.gutb200_image_loss_rgb.argtypes = [vp, i32, i32, vp, vp, f32, f32, vp, vp, vp]
        lib.gutb200_image_loss_rgb.restype = C.c_int
        lib._loss_bound = True
    return lib


def _run(entry, pred, tgt, ch_pred, lambda_l1, lambda_ssim, d_pred, name):
    for t, w, ch in ((pred, name, ch_pred), (tgt, "target_rgb", 3)):
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.dim() == 3 and t.shape[2] == ch):
            raise RuntimeError(f"{w}: expected a contiguous float32 CUDA tensor [H,W,{ch}] (there is no CPU fallback)")
    H, W = int(pred.shape[0]), int(pred.shape[1])
    if tuple(tgt.shape[:2]) != (H, W):
        raise RuntimeError("prediction and target resolutions differ")
    dev = pred.device
    lib = _lib()
    need = int(lib.gutb200_image_loss_scratch_bytes(H, W))
    key = (dev.index, H, W)
    if key not in _scratch or _scratch[key].numel() * 4 < need:
        _scratch[key] = torch.empty((need + 3) // 4, dtype=torch.float32, device=dev)
    if d_pred is None:
        d_pred = torch.empty((H, W, ch_pred), dtype=torch.float32, device=dev)
    sums = torch.empty(2, dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    with torch.cuda.device(dev):
        rc = getattr(lib, entry)(stream, H, W, pred.data_ptr(), tgt.data_ptr(), float(lambda_l1), float(lambda_ssim), _scratch[key].data_ptr(),
                                 d_pred.data_ptr(), sums.data_ptr())
    if rc != 0:
        raise RuntimeError(f"{entry} failed ({rc})")
    l1 = sums[0] / (3.0 * H * W)
    ssim = sums[1] / (3.0 * max(H - 10, 1) * max(W - 10, 1)) if (H > 10 and W > 10) else sums[1] * 0.0
    loss = lambda_l1 * l1 + lambda_ssim * (1.0 - ssim)
    return loss, l1, ssim, d_pred


def image_loss(pred_rgba: torch.Tensor, target_rgb: torch.Tensor, lambda_l1: float = 0.8, lambda_ssim: float = 0.2, d_rgba: torch.Tensor | None = None):
    """pred_rgba [H,W,4] (or [1,H,W,4]), target_rgb [H,W,3] float32 CUDA tensors.
    Returns (loss, l1, ssim, d_rgba): three device scalars and d loss / d pred_rgba [H,W,4]."""
    pred = pred_rgba.reshape(pred_rgba.shape[-3:])
    tgt = target_rgb.reshape(target_rgb.shape[-3:])
    return _run("gutb200_image_loss", pred, tgt, 4, lambda_l1, lambda_ssim, d_rgba, "pred_rgba")


def image_loss_rgb(pred_rgb: torch.Tensor, target_rgb: torch.Tensor, lambda_l1: float = 0.8, lambda_ssim: float = 0.2, d_rgb: torch.Tensor | None = None):
    """The same loss on the 3DGRT layout: pred_rgb [H,W,3] (or [1,H,W,3], the tracer's rgb output; its alpha takes no part), target_rgb
    [H,W,3].  Returns (loss, l1, ssim, d_rgb) with d_rgb [H,W,3] -- directly the rgb gradient of OptixTracer.trace_bwd.  Bit-identical to
    image_loss on cat([rgb, alpha], -1)."""
    pred = pred_rgb.reshape(pred_rgb.shape[-3:])
    tgt = target_rgb.reshape(target_rgb.shape[-3:])
    return _run("gutb200_image_loss_rgb", pred, tgt, 3, lambda_l1, lambda_ssim, d_rgb, "pred_rgb")

"""Evaluation of a trained scene as the reference reports it: render the held-out views, score each frame (PSNR, SSIM, colour-corrected
PSNR and SSIM, optionally LPIPS) and write the renders, the ground truth and `metrics.json` (threedgrut/render.py:233-420), or run the
training's validation pass (trainer.py:1325-1384) without its writer.

A view is `(render_args, target_rgb)`: render_args is the tuple the step's `render()` takes, target_rgb the float32 CUDA [H,W,3] image.
Each frame is one forward (`metrics_inputs`, the step's render before background and post-processing) and one gutb200_image_metrics
pass (metrics.image_metrics: composite, post-processing, metrics and PNG bytes in four launches) into a row of a device [F, K] tensor.
Nothing is read back per frame: the pass synchronises once, after the last frame.  NHT steps are scored with the decoder's EMA shadow
applied and their live weights restored afterwards (render.py:197-201, trainer.py:1331-1332,1381-1382).  The step's training state --
frame, BVH cadence, generators, parameters, decoder weights -- is left as it was.

LPIPS needs network weights that are not part of this project; pass `lpips=` a callable (x, y) -> scalar tensor, called as render.py
calls its metric: NCHW, clip(x, 0, 1) against y, and clip(x_cc) against y.  Without it the LPIPS keys are absent."""
from __future__ import annotations

import contextlib
import json
import os
import struct
import zlib
from collections.abc import Sequence
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

import losses
import metrics as M


@contextlib.contextmanager
def ema_weights(step):
    """The NHT decoder's EMA shadow in place of its live weights for the duration (a no-op for SH steps and for a decoder without EMA)."""
    dec = getattr(step, "decoder", None)
    if dec is None:
        yield
        return
    dec.apply_ema_shadow()
    try:
        yield
    finally:
        dec.restore_ema()


def write_png(path: str, rgb_u8: np.ndarray) -> None:
    """An 8-bit RGB PNG of rgb_u8 [H,W,3] (the pixels of torchvision.utils.save_image's file for the same bytes)."""
    h, w, _ = rgb_u8.shape
    raw = np.concatenate([np.zeros((h, 1), np.uint8), np.ascontiguousarray(rgb_u8, np.uint8).reshape(h, w * 3)], axis=1).tobytes()

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)

    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)) + chunk(b"IDAT", zlib.compress(raw, 6))
                + chunk(b"IEND", b""))


def _x_of(inputs, background, post_processing):
    """The prediction the metrics see, in torch (for the LPIPS callable only): composited, post-processed, [H,W,3]."""
    pred = inputs["pred"]
    rgb = pred[..., :3]
    alpha = pred[..., 3:] if inputs["alpha"] is None else inputs["alpha"].reshape(rgb.shape[0], rgb.shape[1], 1)
    bg = M.background_rgb(background)
    x = rgb if bg is None else rgb + torch.tensor(bg, dtype=rgb.dtype, device=rgb.device) * (1.0 - alpha)
    return x if post_processing is None else losses.linear_to_srgb(x)


def _pass(step, views, png: bool, lpips):
    """Score every view; returns (rows [F,K] numpy, render times ms [F], png bytes [(pred, target)] numpy, lpips [(v, v_cc)])."""
    views = views if isinstance(views, Sequence) else list(views)  # a Sequence makes its items as they are read
    if not len(views):
        raise ValueError("views: nothing to evaluate")
    dev = step.device
    rows = torch.empty((len(views), M.K), dtype=torch.float64, device=dev)
    events, images, scores = [], [], []
    with ema_weights(step):
        for i, (args, target) in enumerate(views):
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            inputs = step.metrics_inputs(*args)
            end.record()
            events.append((start, end))
            tgt = target.reshape(target.shape[-3:]).contiguous()
            res = M.image_metrics(inputs["pred"], tgt, alpha=inputs["alpha"], background=step.background, post_processing=step.post_processing,
                                  hits=inputs["hits"], out=rows[i], png=png)
            if png:
                images.append(res[1:])
            if lpips is not None:
                x = _x_of(inputs, step.background, step.post_processing)
                a, b = rows[i, 9:12].float(), rows[i, 12:15].float()
                xcc = ((x - b) / a).clip(0, 1)
                nchw = lambda t: t.permute(2, 0, 1)[None]  # noqa: E731
                scores.append((lpips(nchw(x.clip(0, 1)), nchw(tgt)), lpips(nchw(xcc), nchw(tgt))))
    torch.cuda.synchronize(dev)  # the pass's one wait
    times = np.array([s.elapsed_time(e) for s, e in events], np.float64)
    host_images = [(p.cpu().numpy(), t.cpu().numpy()) for p, t in images]
    host_scores = [(float(v), float(c)) for v, c in scores]
    return rows.cpu().numpy(), times, host_images, host_scores


def evaluate(step, views, out_dir: str | None = None, global_step: int | None = None, save_gt: bool = True, lpips=None) -> dict:
    """render_all of the reference Renderer on `step`.  views: iterable of (render_args, target_rgb).  out_dir: where to write
    ours_{global_step}/renders/{i:05d}.png, ours_{global_step}/gt/{i:05d}.png (save_gt) and metrics.json; None writes nothing.
    global_step: defaults to the step's frame.  lpips: None or a callable (see the module).
    Returns {"psnr", "ssim", "cc_psnr", "cc_ssim", "l1", "inference_time_ms" (per-frame numpy arrays), ["lpips", "cc_lpips"],
    "metrics": the metrics.json dict, "mean_psnr", "std_psnr" (population), "mean_inference_time"}."""
    gs = int(step.frame if global_step is None else global_step)
    rows, times, images, scores = _pass(step, views, out_dir is not None, lpips)
    out = summarise(rows, times, scores if lpips is not None else None)
    if out_dir is not None:
        write_outputs(out_dir, gs, images, out["metrics"], save_gt)
    return out


def summarise(rows: np.ndarray, times, scores=None) -> dict:
    """evaluate's result from the host rows [F, K] of the pass, the render times (ms) and the LPIPS pairs (None: no LPIPS): per-frame
    arrays, the metrics.json table (render.py's keys and order; the LPIPS keys only with scores) and render_all's (mean_psnr, std_psnr,
    mean_inference_time), std the population np.std.  Pure host logic."""
    rows = np.asarray(rows, np.float64).reshape(-1, M.K)
    out = {k: rows[:, M.FIELDS.index(k)].copy() for k in ("psnr", "ssim", "cc_psnr", "cc_ssim", "l1")}
    out["inference_time_ms"] = np.asarray(times, np.float64)
    table = {"mean_psnr": float(np.mean(out["psnr"])), "mean_ssim": float(np.mean(out["ssim"]))}
    if scores is not None:
        out["lpips"] = np.array([v for v, _ in scores], np.float64)
        out["cc_lpips"] = np.array([c for _, c in scores], np.float64)
        table["mean_lpips"] = float(np.mean(out["lpips"]))
    table["mean_cc_psnr"] = float(np.mean(out["cc_psnr"]))
    table["mean_cc_ssim"] = float(np.mean(out["cc_ssim"]))
    if scores is not None:
        table["mean_cc_lpips"] = float(np.mean(out["cc_lpips"]))
    table["mean_inference_time_ms"] = float(np.mean(out["inference_time_ms"]))
    out.update(metrics=table, mean_psnr=table["mean_psnr"], std_psnr=float(np.std(out["psnr"])), mean_inference_time=table["mean_inference_time_ms"])
    return out


def write_outputs(out_dir: str, global_step: int, images, table: dict, save_gt: bool = True) -> None:
    """ours_{global_step}/renders/{i:05d}.png (and gt/{i:05d}.png) from the host bytes [(pred_u8, target_u8)], and metrics.json."""
    renders = os.path.join(out_dir, f"ours_{int(global_step)}", "renders")
    gt = os.path.join(out_dir, f"ours_{int(global_step)}", "gt")
    os.makedirs(renders, exist_ok=True)
    if save_gt:
        os.makedirs(gt, exist_ok=True)
    jobs = [(os.path.join(renders, f"{i:05d}.png"), p) for i, (p, _) in enumerate(images)]
    if save_gt:
        jobs += [(os.path.join(gt, f"{i:05d}.png"), t) for i, (_, t) in enumerate(images)]
    with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 1) or 1) as pool:  # zlib releases the GIL
        list(pool.map(lambda job: write_png(*job), jobs))
    with open(os.path.join(out_dir, "metrics.json"), "w") as f:
        json.dump(table, f, indent=2)


def validate(step, views, lpips=None) -> dict:
    """The validation pass of the reference trainer (run_validation_pass) without its writer: per view and mean "psnr", "ssim",
    "hits_mean", "hits_std", "hits_min", "hits_max" (and "lpips" of clip(x) against y with a callable), as {"per_view": {key: numpy
    [F]}, "mean": {key: float}}."""
    rows, _, _, scores = _pass(step, views, False, lpips)
    keys = ("psnr", "ssim", "hits_mean", "hits_std", "hits_min", "hits_max")
    per_view = {k: rows[:, M.FIELDS.index(k)].copy() for k in keys}
    if lpips is not None:
        per_view["lpips"] = np.array([v for v, _ in scores])
    return {"per_view": per_view, "mean": {k: float(np.mean(v)) for k, v in per_view.items()}}


# ---- checkpoints --------------------------------------------------------------------------------------------------------------------

GRT_OVERRIDES = {"particle_kernel_density_clamping": True, "min_transmittance": 0.03}  # render.py:109-111


def eval_config(conf) -> dict:
    """The checkpoint's config as evaluation reads it: a plain dict, with render.py's 3DGRT overrides applied (render.method 3dgrt:
    particle_kernel_density_clamping true, min_transmittance 0.03).  post_processing.method ppisp raises NotImplementedError.  Pure
    host logic."""
    conf = _plain(conf)
    method = str(_get(conf, "render.method", "3dgut")).lower()
    if method not in ("3dgut", "3dgrt"):
        raise NotImplementedError(f"render.method={method!r}: evaluation builds 3dgut and 3dgrt steps")
    losses.post_processing_code(_get(conf, "post_processing.method", None))
    if method == "3dgrt":
        conf.setdefault("render", {}).update(GRT_OVERRIDES)
    return conf


def _plain(conf):
    if conf is None:
        return {}
    try:
        from omegaconf import OmegaConf

        if OmegaConf.is_config(conf):
            return OmegaConf.to_container(conf, resolve=True)
    except ImportError:
        pass
    if isinstance(conf, dict):
        return {k: _plain(v) if isinstance(v, dict) else v for k, v in conf.items()}
    return conf


def _get(conf, path, default):
    from b200_native import cfg_get

    return cfg_get(conf, path, default)


def from_checkpoint(path: str, conf=None, device="cuda"):
    """A training step holding the scene of the `ckpt_*.pt` at `path` (written by checkpoint.save or by the reference trainer), built
    from its `config` (or `conf`) as evaluation renders it: render.method 3dgut or 3dgrt (with eval_config's overrides), SH or NHT
    features, the model's background colour and post-processing.  Returns the step; score it with evaluate / validate."""
    import checkpoint
    import step_config

    device = torch.device(device)
    ckpt = torch.load(path, map_location=device, weights_only=False)
    conf = eval_config(conf if conf is not None else ckpt.get("config"))
    ft = str(_get(conf, "model.feature_type", "sh")).lower()
    state = checkpoint.from_reference_layout(ckpt, feature_type=ft)
    settings = state.get("settings") or {}
    bg = settings.get("background", _get(conf, "model.background.color", "black"))
    params = {k: v.detach().to(device=device, dtype=torch.float32).contiguous() for k, v in state["params"].items()}
    lrs = {k: float(v) for k, v in state["lrs"].items()}
    if ft == "nht":
        dec = state["decoder"]
        decoder = step_config.make_decoder(conf, device, arch=dec["arch"])
        step = step_config.build_step(conf, params, 1.0, lrs=lrs, decoder=decoder, background=bg, train=False)
        decoder.network.params.data.copy_(dec["params"])
        if dec["ema"]:
            decoder.load_ema_state_dict({k: v.to(device) for k, v in dec["ema"].items()})
    else:
        sph = int(state.get("sph_degree") if state.get("sph_degree") is not None else 3)
        step = step_config.build_step(conf, params, 1.0, lrs=lrs, sph_degree=sph, background=bg, train=False)
    step.frame = int(state["frame"])
    return step

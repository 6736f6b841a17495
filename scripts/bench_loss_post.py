"""Device time of the image loss with and without the linear-to-sRGB post-processing (post_processing.method: linear-to-srgb), alternating
in one process, at 800x800 and 1237x822 (0.8 L1 + 0.2 (1 - SSIM), white background + a 0/1 mask), per layout:

    rgba    gutb200_image_loss, layout 4, post_processing 0   vs  post_processing 1 (linear-to-sRGB)
    split   gutb200_image_loss, layout 3, post_processing 0   vs  post_processing 1 (linear-to-sRGB)    (d_rgb + d_alpha)

    python scripts/bench_loss_post.py [--reps 200] [--rounds 5]

Each variant is timed with CUDA events around `--reps` back-to-back calls (the two launches and the host wrapper), in `--rounds` rounds
that alternate the variants; the median per-call time is printed with the device time of the kernels alone (torch.profiler), the card
(benchkit.card)."""
from __future__ import annotations

import argparse

import numpy as np

import benchkit

SIZES = ((800, 800), (822, 1237))  # (H, W)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--reps", type=int, default=200, help="calls per timed round")
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds per variant (median is reported)")
    args = ap.parse_args()

    import torch
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    import losses

    dev = benchkit.cuda_device("bench_loss_post.py")
    print(f"device: {benchkit.card(dev)}")
    white = (1.0, 1.0, 1.0)
    variants = {}
    for H, W in SIZES:
        gen = torch.Generator(device=dev).manual_seed(0)
        tgt = torch.rand((H, W, 3), device=dev, generator=gen)
        rgb = (tgt ** 2.2 + 0.05 * torch.randn((H, W, 3), device=dev, generator=gen)).clamp(0, 1.2).contiguous()
        alpha = torch.rand((H, W, 1), device=dev, generator=gen)
        rgba = torch.cat([rgb, alpha], -1).contiguous()
        mask = (torch.rand((H, W), device=dev, generator=gen) > 0.2).float()
        d4, d3, da = torch.empty((H, W, 4), device=dev), torch.empty((H, W, 3), device=dev), torch.empty((H, W, 1), device=dev)
        for post in (None, "linear-to-srgb"):
            tag = "composited" if post is None else "linear-to-sRGB"
            variants[f"{W}x{H} rgba  {tag}"] = (lambda rgba=rgba, tgt=tgt, mask=mask, d4=d4, post=post:
                                                losses.image_loss(rgba, tgt, 0.8, 0.2, d_rgba=d4, background=white, mask=mask, post_processing=post))
            variants[f"{W}x{H} split {tag}"] = (lambda rgb=rgb, alpha=alpha, tgt=tgt, mask=mask, d3=d3, da=da, post=post:
                                                losses.image_loss_rgb_alpha(rgb, alpha, tgt, 0.8, 0.2, background=white, mask=mask, d_rgb=d3,
                                                                            d_alpha=da, post_processing=post))
    for fn in variants.values():  # warm-up: binding, scratch allocation, first launches of every shape
        for _ in range(10):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in variants}
    for _ in range(args.rounds):
        for name, fn in variants.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.reps):
                fn()
            b.record()
            b.synchronize()
            times[name].append(a.elapsed_time(b) * 1000.0 / args.reps)
    kernel_us = {}
    for name, fn in variants.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                fn()
            torch.cuda.synchronize()
        total = sum(getattr(e, "self_device_time_total", 0.0) for e in prof.key_averages() if e.device_type == DeviceType.CUDA)
        kernel_us[name] = total / args.reps
    print(f"0.8 L1 + 0.2 (1 - SSIM), white background + mask; per call: median over {args.rounds} alternating rounds of {args.reps} "
          f"back-to-back calls (CUDA events, host wrapper included) and the device time of the kernels alone (torch.profiler)")
    for name, ts in times.items():
        print(f"  {name:<32s} {np.median(ts):8.1f} us/call  {kernel_us[name]:8.1f} us kernels  (rounds: {' '.join(f'{t:.1f}' for t in ts)})")


if __name__ == "__main__":
    main()

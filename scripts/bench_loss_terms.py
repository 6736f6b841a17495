"""Device time of the per-step launches the rest of the reference loss adds, against the launches they replace, alternating in one process:

  - image loss at 800x800 (0.8 L1 + 0.2 (1 - SSIM)), per layout:
      rgba    gutb200_image_loss, layout 4, plain   vs  composited: white background + a 0/1 mask
      split   gutb200_image_loss, layout 3, plain   vs  composited: white background + a 0/1 mask (d_rgb + d_alpha)
              and, for the random background, the composited loss on a [H,W,3] background image
  - fused Adam at 300k Gaussians: gutb200_gaussian_adam_step vs gutb200_gaussian_adam_step_reg (lambda_opacity = lambda_scale = 0.01)

    python scripts/bench_loss_terms.py [--reps 200] [--rounds 5]

Each variant is timed with CUDA events around `--reps` back-to-back launches, in `--rounds` rounds that alternate the variants; the
median per-launch time over the rounds is printed with the card (benchkit.card)."""
from __future__ import annotations

import argparse

import numpy as np

import benchkit

LRS = dict(positions=1.6e-4, density=0.05, rotation=1e-3, scale=5e-3, features_albedo=2.5e-3, features_specular=1.25e-4)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--reps", type=int, default=200, help="launches per timed round")
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds per variant (median is reported)")
    ap.add_argument("--size", type=int, default=800, help="image side")
    ap.add_argument("--n", type=int, default=300_000, help="Gaussians of the Adam step")
    args = ap.parse_args()

    import torch

    import losses
    import optimizers

    dev = benchkit.cuda_device("bench_loss_terms.py")
    print(f"device: {benchkit.card(dev)}")
    H = W = args.size
    gen = torch.Generator(device=dev).manual_seed(0)
    tgt = torch.rand((H, W, 3), device=dev, generator=gen)
    rgb = (tgt + 0.1 * torch.randn((H, W, 3), device=dev, generator=gen)).clamp(0, 1.2).contiguous()
    alpha = torch.rand((H, W, 1), device=dev, generator=gen)
    rgba = torch.cat([rgb, alpha], -1).contiguous()
    mask = (torch.rand((H, W), device=dev, generator=gen) > 0.2).float()
    bg_img = torch.rand((H, W, 3), device=dev, generator=gen)
    d4 = torch.empty((H, W, 4), device=dev)
    d3 = torch.empty((H, W, 3), device=dev)
    da = torch.empty((H, W, 1), device=dev)
    white = (1.0, 1.0, 1.0)

    n = args.n
    rng = np.random.default_rng(1)
    params = {k: torch.from_numpy(rng.normal(size=(n, w)).astype(np.float32) * 0.1).to(dev) for k, w in zip(optimizers.GROUPS, optimizers.WIDTHS)}
    opt = optimizers.FusedGaussianAdam(params, LRS)
    dp = torch.from_numpy(rng.normal(size=(n, 12)).astype(np.float32) * 1e-4).to(dev)
    ds = torch.from_numpy(rng.normal(size=(n, 48)).astype(np.float32) * 1e-4).to(dev)

    variants = {
        "loss rgba  plain (gutb200_image_loss, layout 4)": lambda: losses.image_loss(rgba, tgt, 0.8, 0.2, d_rgba=d4),
        "loss rgba  white + mask (composited)": lambda: losses.image_loss(rgba, tgt, 0.8, 0.2, d_rgba=d4, background=white, mask=mask),
        "loss split plain (gutb200_image_loss, layout 3)": lambda: losses.image_loss_rgb(rgb, tgt, 0.8, 0.2, d_rgb=d3),
        "loss split white + mask (composited)": lambda: losses.image_loss_rgb_alpha(rgb, alpha, tgt, 0.8, 0.2, background=white, mask=mask,
                                                                                   d_rgb=d3, d_alpha=da),
        "loss split random image + mask (composited)": lambda: losses.image_loss_rgb_alpha(rgb, alpha, tgt, 0.8, 0.2, background=bg_img,
                                                                                          mask=mask, d_rgb=d3, d_alpha=da),
        f"adam {n // 1000}k plain (gutb200_gaussian_adam_step)": lambda: opt.step(dp, ds),
        f"adam {n // 1000}k regularised (gutb200_gaussian_adam_step_reg)": lambda: opt.step(dp, ds, lambda_opacity=0.01, lambda_scale=0.01),
    }
    for fn in variants.values():  # warm-up: binding, scratch allocation, first launches
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
    # kernel time alone (the event-timed loop above includes the host wrapper when the launches are short): torch.profiler's device
    # activity, summed over the kernels of `reps` calls
    kernel_us = {}
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile

    for name, fn in variants.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                fn()
            torch.cuda.synchronize()
        total = sum(getattr(e, "self_device_time_total", 0.0) for e in prof.key_averages() if e.device_type == DeviceType.CUDA)
        kernel_us[name] = total / args.reps
    print(f"{H}x{W} image, {n} Gaussians; per call: median over {args.rounds} alternating rounds of {args.reps} back-to-back calls (CUDA events, "
          f"host wrapper included) and the device time of the kernels alone (torch.profiler)")
    for name, ts in times.items():
        print(f"  {name:<62s} {np.median(ts):8.1f} us/call  {kernel_us[name]:8.1f} us kernels  (rounds: {' '.join(f'{t:.1f}' for t in ts)})")


if __name__ == "__main__":
    main()

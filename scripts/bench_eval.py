"""Device time of the test-set metrics of one frame, and of one evaluation frame end to end.

    python scripts/bench_eval.py [--reps 200] [--frames 20]

  metrics    metrics.image_metrics (gutb200_image_metrics: PSNR, SSIM, colour correction, cc PSNR, cc SSIM, L1 -- four launches) at
             800x800 and 1237x822, against a torch restatement of the reference's chain in the same call: PSNR, SSIM as torchmetrics
             computes it (reflect pad, one 15-channel grouped conv2d, crop, variance clamp), color_correct_affine, cc PSNR, cc SSIM, with
             the reference's .item() after every metric (render.py:326-369).  CUDA events around --reps calls after a warm-up.
  eval frame evaluate.evaluate on C2 (300k Gaussians, 800x800, 3DGUT) over --frames views, per frame: render + metrics, with and without
             writing the PNG files (to a temporary directory).

Prints the card (benchkit.card) first."""
from __future__ import annotations

import argparse
import tempfile
import time

import benchkit

SIZES = ((800, 800), (822, 1237))  # (H, W)


def _reference_chain(x, y, win):
    """The reference's per-frame metrics in torch (x, y: [H,W,3]); returns five floats, synchronising after each as .item() does."""
    import torch
    import torch.nn.functional as F

    def psnr(a, b):
        return (10.0 * torch.log10(1.0 / torch.mean((a - b) ** 2))).item()

    def ssim(a, b):
        p, t = a.permute(2, 0, 1)[None], b.permute(2, 0, 1)[None]
        p, t = F.pad(p, (5, 5, 5, 5), mode="reflect"), F.pad(t, (5, 5, 5, 5), mode="reflect")
        out = F.conv2d(torch.cat([p, t, p * p, t * t, p * t]), win, groups=3)
        mu_p, mu_t, e_pp, e_tt, e_pt = out.split(1)
        s_p, s_t = torch.clamp(e_pp - mu_p ** 2, min=0.0), torch.clamp(e_tt - mu_t ** 2, min=0.0)
        m = (2 * mu_p * mu_t + 1e-4) * (2 * (e_pt - mu_p * mu_t) + 9e-4) / ((mu_p ** 2 + mu_t ** 2 + 1e-4) * (s_p + s_t + 9e-4))
        return m[..., 5:-5, 5:-5].mean().item()

    def color_correct(img, ref):
        im, rm = img.reshape(-1, 3), ref.reshape(-1, 3)
        r_mean, i_mean = rm.mean(0), im.mean(0)
        ri, rr = (rm * im).mean(0), (rm * rm).mean(0)
        var = torch.clamp(rr - r_mean * r_mean, min=1e-8)
        a = (ri - r_mean * i_mean) / var
        b = i_mean - a * r_mean
        a = torch.where(a.abs() < 1e-8, torch.ones_like(a), a)
        return torch.clip((im - b) / a, 0, 1).reshape(img.shape)

    out = [psnr(x, y), ssim(x, y)]
    xcc = color_correct(x, y)
    return out + [psnr(xcc, y), ssim(xcc, y), (x - y).abs().mean().item()]


def _time(fn, reps, torch):
    fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / reps


def bench_metrics(reps, torch):
    import metrics as M
    from oracle import loss_oracle as lo

    dev = torch.device("cuda", 0)
    g = torch.as_tensor(lo.gaussian_window(), dtype=torch.float32, device=dev)
    win = (g[:, None] * g[None, :]).expand(15, 1, 11, 11).contiguous()
    for H, W in SIZES:
        gen = torch.Generator(device=dev).manual_seed(0)
        tgt = torch.rand((H, W, 3), device=dev, generator=gen)
        rgba = torch.cat([(tgt + 0.05 * torch.randn((H, W, 3), device=dev, generator=gen)), torch.ones((H, W, 1), device=dev)], -1).contiguous()
        out = torch.empty(M.K, dtype=torch.float64, device=dev)
        ours = _time(lambda: M.image_metrics(rgba, tgt, out=out), reps, torch)
        ref = _time(lambda: _reference_chain(rgba[..., :3], tgt, win), reps, torch)
        got = M.as_dict(out.cpu().numpy())
        chain = _reference_chain(rgba[..., :3], tgt, win)
        print(f"metrics {W}x{H}: image_metrics {ours * 1e3:.1f} us/frame, reference chain {ref * 1e3:.1f} us/frame ({ref / ours:.1f}x);  "
              f"psnr {got['psnr']:.5f} vs {chain[0]:.5f}, ssim {got['ssim']:.6f} vs {chain[1]:.6f}, cc_psnr {got['cc_psnr']:.5f} vs "
              f"{chain[2]:.5f}, cc_ssim {got['cc_ssim']:.6f} vs {chain[3]:.6f}")


def bench_eval_frame(frames, torch):
    import evaluate
    import scenes
    import train_step

    dev = torch.device("cuda", 0)
    sc = scenes.scene_c2()
    raw = train_step.raw_params(torch.from_numpy(sc.particles).to(dev), torch.from_numpy(sc.sph).to(dev))
    lrs = dict(positions=1e-4, density=0.05, rotation=1e-3, scale=5e-3, features_albedo=1e-2, features_specular=5e-4)
    st = train_step.GaussianTrainStep(raw, lrs, background="white")
    ro, rd = sc.rays()
    rays_o, rays_d = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)

    poses = [scenes.pose7_from_c2w(sc.camera(i, frames)) for i in range(frames)]
    sensor = sc.pinhole_sensor()
    gen = torch.Generator(device=dev).manual_seed(0)
    targets = []
    for p in poses:  # the render on the white background, with noise
        rgba = st.render(rays_o, rays_d, sensor, p)[0]
        noise = 0.02 * torch.randn((sc.height, sc.width, 3), device=dev, generator=gen)
        targets.append((rgba[..., :3] + (1.0 - rgba[..., 3:]) + noise).clamp(0, 1).contiguous())
    views = [((rays_o, rays_d, sensor, p), t) for p, t in zip(poses, targets)]
    evaluate.evaluate(st, views[:2])  # warm-up
    for png in (False, True):
        with tempfile.TemporaryDirectory() as tmp:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = evaluate.evaluate(st, views, out_dir=tmp if png else None)
            dt = (time.perf_counter() - t0) / frames
        print(f"eval frame C2 800x800 ({sc.n} Gaussians, 3DGUT){' + PNG writing' if png else ''}: {dt * 1e3:.2f} ms/frame wall, "
              f"render {out['mean_inference_time']:.2f} ms/frame (events), mean psnr {out['mean_psnr']:.3f}")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--reps", type=int, default=200, help="timed calls per variant")
    ap.add_argument("--frames", type=int, default=20, help="views of the end-to-end evaluation")
    args = ap.parse_args()

    import torch

    print(f"device: {benchkit.card(benchkit.cuda_device('bench_eval.py'))}")
    bench_metrics(args.reps, torch)
    bench_eval_frame(args.frames, torch)


if __name__ == "__main__":
    main()

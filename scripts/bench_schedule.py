"""C2 (300k Gaussians at 800x800) through train_step.GaussianTrainStep with and without a training schedule (schedule.TrainingSchedule of
configs/base_gs.yaml with the MCMC perturbation: exp position decay, progressive SH), alternating step by step in one process.

    python scripts/bench_schedule.py [--steps 60] [--warmup 5] [--n 300000]

Per variant it prints
  - device-timed steps/s (CUDA events around the step, inputs already on the device), median and range,
  - end-to-end steps/s with host inputs (target image copied from pinned host memory each step, wall clock to a synchronise),
and the card (benchkit.card).  Both variants render at SH degree 3 (the scheduled one starts at init_n_features 3), so the two
do the same device work: what differs is the schedule's host update after Adam.  The loss is 0.8 L1 + 0.2 (1 - SSIM)."""
from __future__ import annotations

import argparse
import time

import numpy as np

import benchkit

# configs/base_gs.yaml's schedule (the keys the schedule reads), starting at SH degree 3
CONF = {
    "model": {"feature_type": "sh", "progressive_training": {"init_n_features": 3, "max_n_features": 3, "increase_frequency": 1000,
                                                             "increase_step": 1}},
    "optimizer": {"params": {"positions": {"lr": 0.00016}, "density": {"lr": 0.05}, "features_albedo": {"lr": 0.0025},
                             "features_specular": {"lr": 0.000125}, "rotation": {"lr": 0.001}, "scale": {"lr": 0.005}}},
    "scheduler": {"positions": {"type": "exp", "lr_init": 0.00016, "lr_final": 0.0000016, "max_steps": 30000}, "density": {"type": "skip"}},
    "render": {"particle_radiance_sph_degree": 3},
}
SCENE_EXTENT = 3.0


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=60, help="timed steps per variant and loop")
    ap.add_argument("--warmup", type=int, default=5, help="untimed steps per variant")
    ap.add_argument("--n", type=int, default=300_000, help="Gaussians of the C2 scene")
    args = ap.parse_args()

    import torch

    import densify
    import scenes
    import schedule
    import train_step

    dev = benchkit.cuda_device("bench_schedule.py")
    print(f"device: {benchkit.card(dev)}")

    sc = scenes.scene_c2(n=args.n)
    H, W = sc.height, sc.width
    sensor = sc.pinhole_sensor()
    ro, rd = sc.rays()
    rays_o, rays_d = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)
    P, S = torch.from_numpy(sc.particles).to(dev), torch.from_numpy(sc.sph).to(dev)
    n_views = 10
    poses = [scenes.pose7_from_c2w(sc.camera(i, n_views)) for i in range(n_views)]

    sched = schedule.TrainingSchedule.from_config(CONF, scene_extent=SCENE_EXTENT)
    truth = train_step.GaussianTrainStep(train_step.raw_params(P, S), sched.initial_lrs())
    targets = [truth.render(rays_o, rays_d, sensor, p)[0][..., :3].clone() for p in poses]
    del truth
    host_targets = [t.cpu().pin_memory() for t in targets]
    gen = torch.Generator(device=dev).manual_seed(0)
    P2 = P.clone()
    P2[:, 0:3] += 0.005 * torch.randn((sc.n, 3), device=dev, generator=gen)
    P2[:, 8:11] *= torch.exp(0.1 * torch.randn((sc.n, 3), device=dev, generator=gen))
    # the MCMC perturbation every step (it reads the position rate); no relocation or growth, so N stays the same in both variants
    mcmc = densify.MCMCConfig(relocate_start=10 ** 9, add_start=10 ** 9, perturb_start=0, perturb_end=-1, seed=1)
    weights = dict(lambda_l1=0.8, lambda_ssim=0.2)
    steps = {"schedule=None": train_step.GaussianTrainStep(train_step.raw_params(P2, S), sched.initial_lrs(), densify_conf=mcmc,
                                                           scene_extent=SCENE_EXTENT, **weights),
             "schedule": train_step.GaussianTrainStep(train_step.raw_params(P2, S), None, schedule=sched, densify_conf=mcmc,
                                                      scene_extent=SCENE_EXTENT, **weights)}
    counters = {k: 0 for k in steps}

    def one(name, host=False):
        st = steps[name]
        v = counters[name] % n_views
        counters[name] += 1
        tgt = host_targets[v].to(dev, non_blocking=True) if host else targets[v]
        return st.step(rays_o, rays_d, sensor, poses[v], tgt)

    order = list(steps)
    for _ in range(args.warmup):
        for name in order:
            one(name)
    torch.cuda.synchronize(dev)

    full = {k: [] for k in steps}
    for i in range(args.steps):
        for name in (order if i % 2 == 0 else order[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            one(name)
            b.record()
            b.synchronize()
            full[name].append(a.elapsed_time(b))

    e2e = {k: [] for k in steps}
    block = max(1, args.steps // 3)
    for rep in range(6):
        for name in (order if rep % 2 == 0 else order[::-1]):
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            for _ in range(block):
                one(name, host=True)
            torch.cuda.synchronize(dev)
            e2e[name].append(block / (time.perf_counter() - t0))

    print(f"C2: {sc.n} Gaussians, {W}x{H}, 0.8 L1 + 0.2 SSIM, MCMC perturbation every step, {args.steps} timed steps per variant after "
          f"{args.warmup} warm-up steps, variants alternating")
    for name in order:
        f = np.array(full[name])
        e = np.array(e2e[name])
        print(f"{name:<14} device-timed {np.median(f):7.3f} ms/step ({f.min():.3f}-{f.max():.3f}) -> {1000.0 / np.median(f):6.1f} steps/s;  "
              f"end to end {np.median(e):6.1f} steps/s (blocks of {block}: {' '.join(f'{x:.1f}' for x in e)})")
    st = steps["schedule"]
    print(f"schedule after {counters['schedule']} steps: positions lr {st.optimizer.lrs['positions']:.6g} (start "
          f"{steps['schedule=None'].optimizer.lrs['positions']:.6g}), SH degree {st.sph_degree}")


if __name__ == "__main__":
    main()

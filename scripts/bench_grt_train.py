"""C4 (the C2 scene, 300k Gaussians at 800x800, through 3DGRT) as a training step: train_step_grt.GaussianTrainStepGRT with the
`instances` proxies (density clamping on, a BVH rebuild every step) and the 3DGRT paper config (icosahedron proxies, degree-2 kernel,
clamping off, update cadence 15), alternating step by step in one process.

    python scripts/bench_grt_train.py [--steps 30] [--warmup 5] [--n 300000] [--ssim]
    torchrun --nproc-per-node N scripts/bench_grt_train.py ...

Per config it prints
  - device-timed steps/s of the full step (CUDA events around the step, inputs already on the device),
  - the per-phase breakdown (build = activations + BVH build, trace, loss, backward, exchange, adam; CUDA events between the phases,
    in a separate timed loop),
  - end-to-end steps/s with host inputs (target image and pose copied from pinned host memory each step, wall clock to a synchronise).
With more than one rank every rank traces its own view (view-parallel) and rank 0 also prints views/s over all ranks and the bytes each
rank moves per step in the gradient exchange.  The loss is L1 (--ssim: 0.8 L1 + 0.2 (1 - SSIM)); the start is the scene with its positions
and scales perturbed, the targets are the scene rendered from 10 orbit views."""
from __future__ import annotations

import argparse
import time

import numpy as np

import benchkit

CONFIGS = {
    "instances": {"render": {"min_transmittance": 0.001}},
    "icosahedron": {"render": {"min_transmittance": 0.001, "primitive_type": "icosahedron", "particle_kernel_degree": 2,
                               "particle_kernel_density_clamping": False, "max_consecutive_bvh_update": 15}},
}
PHASES = ("build", "trace", "loss", "backward", "exchange", "adam")
LRS = dict(positions=1.6e-4, density=0.05, rotation=1e-3, scale=5e-3, features_albedo=2.5e-3, features_specular=1.25e-4)


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=30, help="timed steps per config and loop")
    ap.add_argument("--warmup", type=int, default=5, help="untimed steps per config")
    ap.add_argument("--n", type=int, default=300_000, help="Gaussians of the C2 scene")
    ap.add_argument("--ssim", action="store_true", help="0.8 L1 + 0.2 (1 - SSIM) instead of L1")
    args = ap.parse_args()

    import torch
    import torch.distributed as dist

    import scenes
    import train_step
    import train_step_grt
    import view_parallel as vp

    dev = benchkit.cuda_device("bench_grt_train.py")
    rank, world, log = benchkit.ranks(dev)
    log(f"device: {benchkit.card(dev)}, ranks {world}")

    sc = scenes.scene_c2(n=args.n)
    H, W = sc.height, sc.width
    ro, rd = sc.rays()
    rays_o, rays_d = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)
    P, S = torch.from_numpy(sc.particles).to(dev), torch.from_numpy(sc.sph).to(dev)
    n_views = 10
    poses = [torch.from_numpy(np.asarray(sc.camera(i, n_views), np.float32))[None] for i in range(n_views)]

    weights = dict(lambda_l1=0.8, lambda_ssim=0.2) if args.ssim else dict(lambda_l1=1.0, lambda_ssim=0.0)
    gen = torch.Generator(device=dev).manual_seed(0)
    P2 = P.clone()
    P2[:, 0:3] += 0.005 * torch.randn((sc.n, 3), device=dev, generator=gen)
    P2[:, 8:11] *= torch.exp(0.1 * torch.randn((sc.n, 3), device=dev, generator=gen))
    steps, targets = {}, {}
    for name, conf in CONFIGS.items():
        truth = train_step_grt.GaussianTrainStepGRT(train_step.raw_params(P, S), LRS, conf=conf)
        targets[name] = [truth.render(rays_o, rays_d, p)[0][0].clone() for p in poses]
        del truth
        steps[name] = train_step_grt.GaussianTrainStepGRT(train_step.raw_params(P2, S), LRS, conf=conf, **weights)
    host_targets = {k: [t.cpu().pin_memory() for t in v] for k, v in targets.items()}

    counters = {k: 0 for k in CONFIGS}

    def one(name, host=False):
        st = steps[name]
        i = counters[name]
        counters[name] += 1
        views = [vp.views_for_rank(i, r, world, n_views)[0] for r in range(world)]
        positions = np.stack([st.sensor_position(poses[v]) for v in views])
        v = views[rank]
        tgt = host_targets[name][v].to(dev, non_blocking=True) if host else targets[name][v]
        return st.step(rays_o, rays_d, poses[v], tgt, all_sensor_positions=positions)

    order = list(CONFIGS)
    for _ in range(args.warmup):
        for name in order:
            one(name)
    torch.cuda.synchronize(dev)

    # 1. device-timed full steps, configs alternating (the order flips every step so that drift hits both alike)
    full = {k: [] for k in CONFIGS}
    for i in range(args.steps):
        for name in (order if i % 2 == 0 else order[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            one(name)
            b.record()
            b.synchronize()
            full[name].append(a.elapsed_time(b))

    # 2. per-phase breakdown (events between the phases)
    phases = {k: {p: [] for p in PHASES} for k in CONFIGS}
    for i in range(args.steps):
        for name in (order if i % 2 == 0 else order[::-1]):
            st = steps[name]
            st.phase_events = []
            a = torch.cuda.Event(enable_timing=True)
            a.record()
            one(name)
            torch.cuda.synchronize(dev)
            prev = a
            for ph, ev in st.phase_events:
                if ph in phases[name]:
                    phases[name][ph].append(prev.elapsed_time(ev))
                prev = ev
            st.phase_events = None

    # 3. end to end with host inputs (wall clock over blocks of steps, ended by a synchronise)
    e2e = {k: [] for k in CONFIGS}
    block = max(1, args.steps // 3)
    for rep in range(3):
        for name in (order if rep % 2 == 0 else order[::-1]):
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            for _ in range(block):
                one(name, host=True)
            torch.cuda.synchronize(dev)
            e2e[name].append(block / (time.perf_counter() - t0))

    log(f"C4: {sc.n} Gaussians, {W}x{H}, loss {'0.8 L1 + 0.2 SSIM' if args.ssim else 'L1'}, {args.steps} timed steps per config and loop "
        f"after {args.warmup} warm-up steps; median ms (min-max)")
    for name in order:
        f = np.array(full[name])
        log(f"{name:<12} full step {np.median(f):7.3f} ms ({f.min():.3f}-{f.max():.3f}) -> {1000.0 / np.median(f):6.1f} steps/s device-timed")
        log(f"{'':<12} " + "  ".join(f"{p} {np.median(phases[name][p]):.3f}" for p in PHASES))
        log(f"{'':<12} end-to-end with host inputs: " + ", ".join(f"{v:.1f}" for v in e2e[name]) + " steps/s (three blocks of "
            f"{block} steps)  N {steps[name].n}  BVH updates counted {steps[name].num_update_bvh}")
        if world > 1:
            log(f"{'':<12} {world} ranks: {world * 1000.0 / np.median(f):.1f} views/s; exchange {steps[name].bytes_on_wire() / 1e6:.1f} MB "
                f"per rank and step (one all-reduce of 240 B x N)")
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()

"""C5 (the 3DGRUT hybrid: a garden-like scene of 5M Gaussians at 1237x822, primary rays through 3DGUT, their reflections off the
z = -1.2 mirror through 3DGRT) as a training step: train_step_hybrid.GaussianTrainStepHybrid.

    python scripts/bench_hybrid_train.py --workload c5 [--steps 20] [--warmup 5] [--n 5000000] [--ssim]
    torchrun --nproc-per-node N scripts/bench_hybrid_train.py --workload c5 ...

Prints one JSON line with
  - device-timed steps/s of the full step (CUDA events around the step, inputs on the device) and the median ms of every phase of
    train_step_hybrid.PHASES (events between the phases, in a separate loop),
  - fwd+bwd frames/s: mirror rays, primary forward, BVH build, secondary forward, composite and the backward of both passes into the
    exchange buffer, with a fixed image gradient (no loss, no exchange, no Adam),
  - the fraction of pixels whose ray meets the mirror, over the timed views,
  - the 3DGRT work counters of one secondary trace next to those of the C4 primary trace (300k Gaussians at 800x800, the C2 scene),
  - the peak device memory and the card (benchkit.card), read in the same run.
With more than one rank every rank trains its own view and rank 0 also reports views/s over all ranks.  The start is the scene with its
positions and scales perturbed; the targets are the hybrid renders of the scene from 6 orbit views.  Writes no file."""
from __future__ import annotations

import argparse
import json

import numpy as np

import benchkit

LRS = dict(positions=1.6e-4, density=0.05, rotation=1e-3, scale=5e-3, features_albedo=2.5e-3, features_specular=1.25e-4)
N_VIEWS = 6


def _median(v):
    return float(np.median(v)) if len(v) else float("nan")


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--workload", choices=["c5"], default="c5")
    ap.add_argument("--steps", type=int, default=20, help="timed steps per loop")
    ap.add_argument("--warmup", type=int, default=5, help="untimed steps")
    ap.add_argument("--n", type=int, default=5_000_000, help="Gaussians of the C5 scene")
    ap.add_argument("--ssim", action="store_true", help="0.8 L1 + 0.2 (1 - SSIM) instead of L1")
    args = ap.parse_args()

    import torch
    import torch.distributed as dist

    import scenes
    import threedgrt_tracer
    import train_step
    import train_step_hybrid as th
    import view_parallel as vp

    dev = benchkit.cuda_device("bench_hybrid_train.py")
    rank, world, _ = benchkit.ranks(dev)
    card = benchkit.card(dev)

    sc = scenes.scene_c5(n=args.n)
    H, W = sc.height, sc.width
    sensor = sc.pinhole_sensor()
    ro, rd = sc.rays()
    rays_o, rays_d = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)
    P, S = torch.from_numpy(sc.particles).to(dev), torch.from_numpy(sc.sph).to(dev)
    poses = [torch.from_numpy(np.asarray(sc.camera(i, N_VIEWS), np.float32))[None] for i in range(N_VIEWS)]

    weights = dict(lambda_l1=0.8, lambda_ssim=0.2) if args.ssim else dict(lambda_l1=1.0, lambda_ssim=0.0)
    truth = th.GaussianTrainStepHybrid(train_step.raw_params(P, S), LRS, mirror=scenes.C5_MIRROR)
    targets = [truth.render(rays_o, rays_d, sensor, p)[0].clone() for p in poses]
    del truth
    gen = torch.Generator(device=dev).manual_seed(0)
    P2 = P.clone()
    P2[:, 0:3] += 0.005 * torch.randn((sc.n, 3), device=dev, generator=gen)
    P2[:, 8:11] *= torch.exp(0.1 * torch.randn((sc.n, 3), device=dev, generator=gen))
    st = th.GaussianTrainStepHybrid(train_step.raw_params(P2, S), LRS, mirror=scenes.C5_MIRROR, **weights)
    del P2
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats(dev)
    counter = [0]

    def views_now():
        i = counter[0]
        counter[0] += 1
        return [vp.views_for_rank(i, r, world, N_VIEWS)[0] for r in range(world)]

    def one():
        views = views_now()
        positions = np.stack([np.asarray(poses[v][0, :3, 3], np.float32) for v in views])
        v = views[rank]
        return st.step(rays_o, rays_d, sensor, poses[v], targets[v], all_sensor_positions=positions)

    for _ in range(args.warmup):
        one()
    torch.cuda.synchronize(dev)

    # 1. device-timed full steps
    full = []
    for _ in range(args.steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        one()
        b.record()
        b.synchronize()
        full.append(a.elapsed_time(b))

    # 2. per-phase split
    phases = {p: [] for p in th.PHASES}
    for _ in range(args.steps):
        st.phase_events = []
        a = torch.cuda.Event(enable_timing=True)
        a.record()
        one()
        torch.cuda.synchronize(dev)
        prev = a
        for ph, ev in st.phase_events:
            phases[ph].append(prev.elapsed_time(ev))
            prev = ev
        st.phase_events = None

    # 3. fwd+bwd only: both passes forward and backward into the exchange buffer, a fixed image gradient, no loss / exchange / Adam
    d_img = (torch.randn((H, W, 3), device=dev, generator=gen) * 1e-6).contiguous()
    ot = st.tracer.tracer_wrapper
    hits = []

    def fwd_bwd(v):
        with torch.no_grad():
            frame = st._forward((rays_o, rays_d, sensor, poses[v]), *st.activated(), train=True)
            st._backward(frame, d_img, None)
            *_, (_, _, hit) = frame.saved  # the secondary rays and their mirror hit mask
            return hit

    for i in range(2):
        fwd_bwd(i % N_VIEWS)
    fb = []
    for i in range(args.steps):
        v = i % N_VIEWS
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        hit = fwd_bwd(v)
        b.record()
        b.synchronize()
        fb.append(a.elapsed_time(b))
        if i < N_VIEWS:
            hits.append(float(hit.mean()))
    peak = torch.cuda.max_memory_allocated(dev)

    # 4. work counters: one C5 secondary trace, one C4 primary trace
    with torch.no_grad():
        particles, sph = st.activated()
        m = th.mirror_settings(scenes.C5_MIRROR)
        so, sd, _ = th.hybrid_rays(rays_o, rays_d, poses[0], m["plane_point"], m["plane_normal"])
        ot.build_bvh_packed(particles)
        sec_counters = ot.trace_counters(st._identity, so, sd, particles, sph, st.sph_degree, st.min_transmittance)
    del st, particles, sph
    torch.cuda.empty_cache()
    c4 = scenes.scene_c2(n=300_000)
    ro4, rd4 = c4.rays()
    P4, S4 = torch.from_numpy(c4.particles).to(dev), torch.from_numpy(c4.sph).to(dev)
    t4 = threedgrt_tracer.Tracer({"render": {"min_transmittance": 0.001}}).tracer_wrapper
    t4.build_bvh_packed(P4)
    c4_counters = t4.trace_counters(torch.from_numpy(np.asarray(c4.camera(0, 10), np.float32))[None], torch.from_numpy(ro4).to(dev),
                                    torch.from_numpy(rd4).to(dev), P4, S4, 3, 0.001)

    f = np.array(full)
    result = {
        "workload": "c5", "scene": sc.name, "gaussians": sc.n, "width": W, "height": H, "ranks": world,
        "loss": "0.8 L1 + 0.2 SSIM" if args.ssim else "L1", "steps": args.steps, "warmup": args.warmup,
        "step_ms_median": float(np.median(f)), "step_ms_min": float(f.min()), "step_ms_max": float(f.max()),
        "steps_per_s": 1000.0 / float(np.median(f)),
        "phase_ms_median": {p: _median(phases[p]) for p in th.PHASES},
        "fwd_bwd_ms_median": _median(fb), "fwd_bwd_frames_per_s": 1000.0 / _median(fb),
        "hit_fraction": float(np.mean(hits)), "hit_fraction_per_view": hits,
        "secondary_trace_counters": sec_counters, "c4_primary_trace_counters": c4_counters,
        "peak_memory_gb": peak / 1e9, "device": card,
    }
    if world > 1:
        result["views_per_s_all_ranks"] = world * 1000.0 / float(np.median(f))
    if rank == 0:
        print(json.dumps(result))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()

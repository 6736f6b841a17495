"""Cost of the 3DGRT normals (render.enable_normals): C4 traced with and without normals in one process.

    python scripts/bench_grt_normals.py [--steps 30] [--warmup 5] [--n 300000]

C4 is the C2 scene (300k Gaussians, 800x800) through 3DGRT, on the default `instances` config and on the icosahedron paper config
(degree-2 kernel, no density clamping).  The BVH is built once per config; each timed step is one forward trace of an orbit view, with
normals (grtb200_trace_normals) and without (grtb200_trace) alternately, each timed with CUDA events.  The hit-list recording for the
backward is off, as in an inference render (Tracer.render without gradients), where the normals view is used.  Prints the card
(benchkit.card) and the median trace times.
"""
from __future__ import annotations

import argparse

import numpy as np

import benchkit

CONFIGS = {
    "instances": {"min_transmittance": 0.001},
    "icosahedron paper": {"min_transmittance": 0.001, "primitive_type": "icosahedron", "particle_kernel_degree": 2,
                          "particle_kernel_density_clamping": False},
}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=30, help="timed traces per config and mode")
    ap.add_argument("--warmup", type=int, default=5, help="untimed traces per config and mode")
    ap.add_argument("--n", type=int, default=300_000, help="Gaussians of the C2 scene")
    args = ap.parse_args()

    import torch

    import scenes
    import threedgrt_tracer

    dev = benchkit.cuda_device("bench_grt_normals.py")
    print(f"device: {benchkit.card(dev)}")
    sc = scenes.scene_c2(n=args.n)
    H, W = sc.height, sc.width
    particles = torch.from_numpy(sc.particles).to(dev)
    sph = torch.from_numpy(sc.sph).to(dev)
    ro_np, rd_np = sc.rays()
    rays_o, rays_d = torch.from_numpy(ro_np).to(dev), torch.from_numpy(rd_np).to(dev)
    n_views = 100
    c2ws = [torch.from_numpy(np.asarray(sc.camera(i, n_views), np.float32))[None] for i in range(n_views)]
    modes = ("plain", "normals")

    print(f"C4: {sc.n} Gaussians, {W}x{H}, {args.steps} timed traces per mode after {args.warmup} warm-up traces (median ms)")
    print(f"{'config':<18} {'plain':>9} {'normals':>9} {'overhead':>9}")
    for label, render in CONFIGS.items():
        ot = threedgrt_tracer.Tracer({"render": dict(render, enable_normals=True)}).tracer_wrapper
        ot.build_bvh_packed(particles)
        ot.set_replay(False, dev)
        times = {m: [] for m in modes}

        def trace(mode, i, timed):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            out = ot.trace(i, c2ws[i % n_views], rays_o, rays_d, particles, sph, 0, sc.sph_degree, 0.001, normals=mode == "normals")
            ev[1].record()
            torch.cuda.synchronize(dev)
            if timed:
                times[mode].append(ev[0].elapsed_time(ev[1]))
            return out

        for i in range(args.warmup):
            for m in modes:
                trace(m, i, False)
        for i in range(args.steps):
            for m in (modes if i % 2 == 0 else modes[::-1]):
                trace(m, args.warmup + i, True)
        a, b = trace("plain", 3, False), trace("normals", 3, False)
        same = all(torch.equal(x, y) for k, (x, y) in enumerate(zip(a, b)) if k != 3)
        med = {m: float(np.median(times[m])) for m in modes}
        print(f"{label:<18} {med['plain']:9.3f} {med['normals']:9.3f} {100.0 * (med['normals'] / med['plain'] - 1.0):8.1f}%"
              f"   other outputs identical: {same}, rays with a normal: {float((b[3].abs().sum(-1) > 0).float().mean()):.3f}")


if __name__ == "__main__":
    main()

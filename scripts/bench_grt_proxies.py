"""C4 (the C2 scene through 3DGRT) with both proxy primitives in one process: build / trace / trace_bwd times and work counters.

    python scripts/bench_grt_proxies.py [--steps 20] [--warmup 5] [--n 300000]

A step is the step of bench.py's c4 line (full BVH build + trace + trace_bwd of one orbit view).  The primitives alternate step by step
so that clock drift hits both alike; every stage is timed with CUDA events.  Both use the 3DGRT default kernel (degree 4, density
clamping), so only the proxy differs.  Prints the card and its power limit, median stage times, and the work counters of one forward
per ray (grtb200_debug_trace_counters): k-nearest queries, node visits, proxy tests, candidate and accepted hits.
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "3dgrut_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

PRIMITIVES = ("instances", "icosahedron")


def _power_limit(index: int) -> str:
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30)
        return out.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=20, help="timed steps per primitive")
    ap.add_argument("--warmup", type=int, default=5, help="untimed steps per primitive")
    ap.add_argument("--n", type=int, default=300_000, help="Gaussians of the C2 scene")
    args = ap.parse_args()

    import torch

    import scenes
    import threedgrt_tracer

    dev = torch.device("cuda", 0)
    print(f"device: {torch.cuda.get_device_name(dev)}, power limit {_power_limit(0)}")
    sc = scenes.scene_c2(n=args.n)
    H, W = sc.height, sc.width
    tracers = {p: threedgrt_tracer.Tracer({"render": {"min_transmittance": 0.001, "primitive_type": p}}).tracer_wrapper for p in PRIMITIVES}
    particles = torch.from_numpy(sc.particles).to(dev)
    sph = torch.from_numpy(sc.sph).to(dev)
    pos, dns, rot, scl = (particles[:, 0:3].contiguous(), particles[:, 3:4].contiguous(), particles[:, 4:8].contiguous(),
                          particles[:, 8:11].contiguous())
    ro_np, rd_np = sc.rays()
    rays_o, rays_d = torch.from_numpy(ro_np).to(dev), torch.from_numpy(rd_np).to(dev)
    n_views = 100
    c2ws = [torch.from_numpy(np.asarray(sc.camera(i, n_views), np.float32))[None] for i in range(n_views)]
    gen = torch.Generator(device=dev).manual_seed(1234)
    d_rgb = torch.randn((1, H, W, 3), device=dev, generator=gen)
    d_alpha = torch.randn((1, H, W, 1), device=dev, generator=gen)
    d_dist = 0.05 * torch.randn((1, H, W, 1), device=dev, generator=gen)
    d_nrm = torch.zeros((1, H, W, 3), device=dev)
    stages = ("build_bvh", "trace", "trace_bwd")
    times = {p: {k: [] for k in stages} for p in PRIMITIVES}
    hits = {}

    def step(prim, i, timed):
        ot = tracers[prim]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        ot.build_bvh(pos, rot, scl, dns, True, False)
        ev[1].record()
        c2w = c2ws[i % n_views]
        feat, alpha, hit, nrm, nh, vis = ot.trace(i, c2w, rays_o, rays_d, particles, sph, 0, sc.sph_degree, 0.001)
        ev[2].record()
        ot.trace_bwd(i, c2w, rays_o, rays_d, feat, alpha, hit, nrm, particles, sph, d_rgb, d_alpha, d_dist, d_nrm, 0, sc.sph_degree, 0.001)
        ev[3].record()
        torch.cuda.synchronize(dev)
        if timed:
            for k, a, b in zip(stages, ev[:-1], ev[1:]):
                times[prim][k].append(a.elapsed_time(b))
        hits[prim] = float(nh.sum())

    for i in range(args.warmup):
        for prim in PRIMITIVES:
            step(prim, i, False)
    for i in range(args.steps):
        for prim in (PRIMITIVES if i % 2 == 0 else PRIMITIVES[::-1]):
            step(prim, args.warmup + i, True)

    print(f"C4: {sc.n} Gaussians, {W}x{H}, {args.steps} timed steps per primitive after {args.warmup} warm-up steps (median ms)")
    print(f"{'primitive':<12} " + " ".join(f"{k:>10}" for k in stages) + f" {'step':>10} {'frames/s':>9}")
    for prim in PRIMITIVES:
        med = [float(np.median(times[prim][k])) for k in stages]
        tot = float(np.median(np.sum([times[prim][k] for k in stages], 0)))
        print(f"{prim:<12} " + " ".join(f"{v:10.3f}" for v in med) + f" {tot:10.3f} {1000.0 / tot:9.1f}")

    print("work per ray of one forward (view 2): queries, node visits, proxy tests, candidate hits, accepted hits")
    for prim in PRIMITIVES:
        ot = tracers[prim]
        ot.build_bvh(pos, rot, scl, dns, True, False)
        c = ot.trace_counters(c2ws[2], rays_o, rays_d, particles, sph, sc.sph_degree, 0.001)
        r = max(c["rays"], 1)
        print(f"{prim:<12} " + " ".join(f"{k}={c[k] / r:.2f}" for k in ("queries", "node_visits", "proxy_tests", "candidate_hits", "accepted_hits"))
              + f"  packet rays {c['packet_rays'] / r:.3f}, hits (last timed frame) {hits[prim] / (H * W):.2f}")


if __name__ == "__main__":
    main()

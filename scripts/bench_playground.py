"""Cost of the playground render (playground.Engine, grtb200_trace_playground) at C4 scale, against the plain 3DGRT trace.

    python scripts/bench_playground.py [--steps 30] [--warmup 5] [--n 300000]

C4 is the C2 scene (300k Gaussians, 800x800) through 3DGRT on the default `instances` config.  Cases, each timed with CUDA events per
render over an orbit of views, alternating with the plain trace (grtb200_trace, hit-list recording off as in an inference render):
  no mesh         the playground with no mesh inserted
  mirror quad     a mirror quad between the camera and the Gaussians, facing the camera, covering half of the view
  glass sphere    a glass sphere (ior 1.5) of 19,800 triangles between the camera and the Gaussians
  diffuse cube    a diffuse cube between the camera and the Gaussians
The meshes follow the orbiting camera: the mesh BVH is rebuilt for every view, outside the timed window.  "mesh px" is the fraction of
pixels whose colour differs from the plain trace.  Prints the card (benchkit.card) beside the median render times.
"""
from __future__ import annotations

import argparse

import numpy as np

import benchkit


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=30, help="timed renders per case and mode")
    ap.add_argument("--warmup", type=int, default=5, help="untimed renders per case and mode")
    ap.add_argument("--n", type=int, default=300_000, help="Gaussians of the C2 scene")
    args = ap.parse_args()

    import torch

    import playground as pg
    import scenes

    dev = benchkit.cuda_device("bench_playground.py")
    card = benchkit.card(dev)
    sc = scenes.scene_c2(n=args.n)
    H, W = sc.height, sc.width
    ro_np, rd_np = sc.rays()
    rays_o, rays_d = torch.from_numpy(ro_np).to(dev), torch.from_numpy(rd_np).to(dev)
    n_views = 100
    c2ws = [np.asarray(sc.camera(i, n_views), np.float32) for i in range(n_views)]
    eng = pg.Engine.from_gaussians(torch.from_numpy(sc.particles), torch.from_numpy(sc.sph), sc.sph_degree, device=dev)
    plain = eng.tracer.tracer_wrapper
    particles, sph = eng.particles, eng.sph

    def frame(c2w, ahead):
        """A 4x4 transform `ahead` x the camera distance in front of the camera, z towards it, and the camera distance."""
        eye, fwd = c2w[:3, 3].astype(np.float64), c2w[:3, 2].astype(np.float64)
        z = -fwd / np.linalg.norm(fwd)
        x = np.cross([0.0, 1.0, 0.0], z)
        x /= np.linalg.norm(x)
        m = np.eye(4)
        m[:3, :3] = np.stack([x, np.cross(z, x), z], 1)
        dist = float(np.linalg.norm(eye))
        m[:3, 3] = eye - z * ahead * dist
        return m, x, dist

    def mirror_quad(c2w):
        # between the camera and the Gaussians (a mesh behind opaque Gaussians changes nothing); its edge on the optical axis, so it
        # covers one half of the image
        m, x, dist = frame(c2w, 0.4)
        m[:3, 3] += x * dist
        return pg.Mesh.quad(2.0 * dist, material="mirror", transform=m)

    def scaled(c2w, size):
        m, _, dist = frame(c2w, 0.5)
        m[:3, :3] *= size * dist
        return m

    # the meshes follow the orbiting camera, so each view rebuilds the mesh BVH (outside the timed window)
    cases = {
        "no mesh": lambda c2w: {},
        "mirror quad": lambda c2w: {"quad": mirror_quad(c2w)},
        "glass sphere": lambda c2w: {"ball": pg.Mesh.sphere(1.0, stacks=100, slices=100, material="glass", ior=1.5, transform=scaled(c2w, 0.12))},
        "diffuse cube": lambda c2w: {"cube": pg.Mesh.cube(1.0, material="diffuse", color=(0.8, 0.3, 0.2), transform=scaled(c2w, 0.15))},
    }
    print(f"device: {card}")
    print(f"C4: {sc.n} Gaussians, {W}x{H}, {args.steps} timed renders per mode after {args.warmup} warm-up renders (median ms)")
    print(f"{'case':<14} {'triangles':>9} {'plain':>9} {'playground':>11} {'ratio':>7} {'mesh px':>8}")
    for label, make in cases.items():
        times = {"plain": [], "playground": []}
        ntri, covered = 0, 0.0
        for i in range(args.warmup + args.steps):
            v = i % n_views
            for name in list(eng.meshes):
                eng.remove_mesh(name)
            for name, m in make(c2ws[v]).items():
                eng.add_mesh(name, m)
                ntri = m.faces.shape[0]
            batch = {"rays_ori": rays_o, "rays_dir": rays_d, "T_to_world": torch.from_numpy(c2ws[v])[None]}
            if eng._dirty:
                with torch.cuda.device(dev):
                    eng._build_meshes()
            torch.cuda.synchronize(dev)
            for mode in (("plain", "playground") if i % 2 == 0 else ("playground", "plain")):
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
                ev[0].record()
                if mode == "plain":
                    plain.trace(i, batch["T_to_world"], rays_o, rays_d, particles, sph, 0, sc.sph_degree, eng.min_transmittance, normals=False)
                else:
                    out = eng.render(batch)
                ev[1].record()
                torch.cuda.synchronize(dev)
                if i >= args.warmup:
                    times[mode].append(ev[0].elapsed_time(ev[1]))
            if i == args.warmup:
                ref = plain.trace(i, batch["T_to_world"], rays_o, rays_d, particles, sph, 0, sc.sph_degree, eng.min_transmittance, normals=False)
                covered = float(((out["rgb"] - ref[0].clamp(0, 1)).abs().amax(-1) > 0).float().mean())
        med = {m: float(np.median(t)) for m, t in times.items()}
        print(f"{label:<14} {ntri:9d} {med['plain']:9.3f} {med['playground']:11.3f} {med['playground'] / med['plain']:7.2f} {covered:8.3f}"
              f"   [{card}]")


if __name__ == "__main__":
    main()

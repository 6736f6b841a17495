"""NHT training steps on one GPU: C2 (300k Gaussians at 800x800) through 3DGUT (train_step_nht.GaussianTrainStepNHT) and C4 (the same
scene through 3DGRT, GaussianTrainStepGRTNHT), with the shipped decoder (3 hidden layers of 128, SH degree 3, sh_scale 3, sigmoid) and
random NHT features, then the fused NHT Adam launch against what the reference runs instead.

    python scripts/bench_nht_train.py [--steps 20] [--warmup 5] [--n 300000]

Prints, with the card (benchkit.card):
  - device-timed steps/s of each step (CUDA events around the step; the two renderers alternate step by step),
  - the per-phase split (CUDA events between the phases, `phase_events`, in a separate loop): render, decode (the [H,W,25] slice copies
    that feed the decoder included), loss, decode_backward, render_backward, exchange, adam, densify; 3DGRT adds the BVH build,
  - one gutb200_nht_adam_step launch against torch.optim.Adam(fused=True) over the five Gaussian tensors plus a second fused Adam for the
    decoder (trainer.py:573-577), with the raw gradients already in place, alternating in the same process."""
from __future__ import annotations

import argparse
import json
import math

import numpy as np

import benchkit

LRS = dict(positions=1.6e-4, density=0.05, rotation=1e-3, scale=5e-3, features=2.5e-3, decoder=6.8e-4)
CONF = {"model": {"feature_type": "nht", "nht_features": {"dim": 48, "activation": {"type": "sincos", "num_frequencies": 1},
                                                           "interpolation_type": "barycentric"}},
        "render": {"min_transmittance": 0.001, "pipeline_type": "referenceSlang", "backward_pipeline_type": "referenceSlangBwd"}}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, default=20, help="timed steps per workload and loop")
    ap.add_argument("--warmup", type=int, default=5, help="untimed steps per workload")
    ap.add_argument("--n", type=int, default=300_000, help="Gaussians of the C2 scene")
    args = ap.parse_args()

    import torch

    import feature_decoder as fdm
    import optimizers
    import scenes
    import train_step
    import train_step_nht as tsn

    dev = benchkit.cuda_device("bench_nht_train.py")
    card = benchkit.card(dev)
    print(f"device: {card}")

    sc = scenes.scene_c2(n=args.n)
    H, W = sc.height, sc.width
    ro, rd = sc.rays()
    rays_o, rays_d = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)
    P = torch.from_numpy(sc.particles).to(dev)
    feats = torch.from_numpy(np.random.default_rng(1).uniform(-math.pi / 2, math.pi / 2, (sc.n, 48)).astype(np.float32)).to(dev)
    n_views = 10
    c2w = [np.asarray(sc.camera(i, n_views), np.float32) for i in range(n_views)]
    T = [torch.from_numpy(m)[None] for m in c2w]
    pose7 = [scenes.pose7_from_c2w(m) for m in c2w]
    sensor = sc.pinhole_sensor()

    def decoder():
        torch.manual_seed(0)
        return fdm.FeatureDecoder(24, hidden_dim=128, num_layers=3, sh_scale=3.0).to(dev)

    steps = {"C2 3DGUT": tsn.GaussianTrainStepNHT(train_step.raw_params(P, features=feats), LRS, decoder(), CONF),
             "C4 3DGRT": tsn.GaussianTrainStepGRTNHT(train_step.raw_params(P, features=feats), LRS, decoder(), CONF)}
    targets = [(0.5 + 0.3 * torch.rand((H, W, 3), device=dev, generator=torch.Generator(device=dev).manual_seed(i))).contiguous()
               for i in range(n_views)]
    counters = {k: 0 for k in steps}

    def one(name):
        st, i = steps[name], counters[name] % n_views
        counters[name] += 1
        if name.endswith("3DGUT"):
            return st.step(rays_o, rays_d, sensor, pose7[i], targets[i])
        return st.step(rays_o, rays_d, T[i], targets[i])

    for name in steps:
        for _ in range(args.warmup):
            one(name)
    torch.cuda.synchronize()

    times = {k: [] for k in steps}
    for _ in range(args.steps):
        for name in steps:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            one(name)
            b.record()
            times[name].append((a, b))
    torch.cuda.synchronize()
    result = {"card": card, "n": sc.n, "resolution": [W, H], "workloads": {}}
    for name, evs in times.items():
        ms = [a.elapsed_time(b) for a, b in evs]
        result["workloads"][name] = {"steps_per_s": 1000.0 / float(np.mean(ms)), "ms_median": float(np.median(ms))}
        print(f"{name}: {1000.0 / np.mean(ms):.2f} steps/s (median {np.median(ms):.2f} ms/step)  [{card}]")

    for name, st in steps.items():
        split = {}
        for _ in range(args.steps):
            st.phase_events = []
            start = torch.cuda.Event(enable_timing=True)
            start.record()
            one(name)
            torch.cuda.synchronize()
            prev = start
            for phase, ev in st.phase_events:
                split[phase] = split.get(phase, 0.0) + prev.elapsed_time(ev) / args.steps
                prev = ev
            st.phase_events = None
        result["workloads"][name]["phases_ms"] = split
        print(f"{name} phases (ms): " + ", ".join(f"{k} {v:.3f}" for k, v in split.items()) + f"  [{card}]")

    # one fused NHT Adam launch against torch.optim.Adam(fused=True) x 2 (Gaussians + decoder) on the same tensors
    st = steps["C2 3DGUT"]
    n_dec = st.decoder.network.params.numel()
    g = torch.Generator(device=dev).manual_seed(3)
    dp, df, dd = (torch.randn(s, device=dev, generator=g) for s in ((st.n, 12), (st.n, 48), (n_dec,)))
    opt = optimizers.FusedNHTAdam({k: v.clone() for k, v in st.params.items()}, st.decoder.network.params.detach().clone(), LRS)
    leaves = [torch.nn.Parameter(v.detach().clone()) for v in st.params.values()]
    dparam = torch.nn.Parameter(st.decoder.network.params.detach().clone())
    for p in leaves:
        p.grad = torch.randn(p.shape, device=dev, generator=g)
    dparam.grad = dd.clone()
    ref_g = torch.optim.Adam([{"params": [p], "lr": LRS[k]} for p, k in zip(leaves, optimizers.NHT_GROUPS)], eps=1e-15, fused=True)
    ref_d = torch.optim.Adam([dparam], lr=LRS["decoder"], eps=1e-8, fused=True)
    ours_ms, ref_ms = [], []
    reps = 50
    for it in range(reps + 5):
        for which in ("ours", "ref"):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            if which == "ours":
                opt.step(dp, df, dd)
            else:
                ref_g.step()
                ref_d.step()
            b.record()
            if it >= 5:
                (ours_ms if which == "ours" else ref_ms).append((a, b))
    torch.cuda.synchronize()
    o = float(np.median([a.elapsed_time(b) for a, b in ours_ms]))
    r = float(np.median([a.elapsed_time(b) for a, b in ref_ms]))
    result["adam_ms"] = {"fused_nht_adam": o, "torch_adam_fused_x2": r}
    print(f"Adam over {st.n} Gaussians + {n_dec} decoder params: gutb200_nht_adam_step {o * 1e3:.1f} us, torch.optim.Adam(fused=True) x 2 "
          f"{r * 1e3:.1f} us (median of {reps})  [{card}]")
    print(json.dumps(result))


if __name__ == "__main__":
    main()

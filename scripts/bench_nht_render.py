"""Device time of an NHT frame through 3DGUT on scene C2 (300k Gaussians, 800x800), split by stage, with the SH frame of the same scene.

Stages (CUDA events, L2 flushed before every timed call, warmup first): NHT render forward (gutb200_forward_nht), NHT render backward
(gutb200_backward_nht), decoder forward, decoder forward + backward, and the whole NHT training frame (render -> decode -> L1 gradient ->
decode backward -> render backward).  The SH forward + backward (gutb200_forward / gutb200_backward) runs in the same process, alternating
with the NHT runs.  Features are drawn from U(-pi/2, pi/2), the init range of configs/base_gs.yaml.  Prints the card name and power limit
and one JSON line.  A CUDA device is required.

  python scripts/bench_nht_render.py [--iters 20] [--warmup 5] [--half]
"""
from __future__ import annotations

import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "3dgrut_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"{torch.cuda.get_device_name()} (power limit unavailable: {e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--half", action="store_true", help="fp16 particle features (render.particle_feature_half)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nht_render: a CUDA device is required")
    import b200_native as nat
    import feature_decoder as fdm
    import scenes

    sc = scenes.scene_c2()
    c2w = sc.camera(0, 100)
    pose = scenes.pose7_from_c2w(c2w)
    ctx = nat.Context(nat.default_config(), 0)
    cam = nat.Camera()
    cam.width, cam.height = sc.width, sc.height
    cam.principal[:] = [sc.cx, sc.cy]
    cam.focal[:] = [sc.fx, sc.fy]
    cam.pose_start[:] = [float(v) for v in pose]
    cam.pose_end[:] = [float(v) for v in pose]
    ro, rd = (torch.from_numpy(np.ascontiguousarray(t)).cuda() for t in sc.rays())
    n, h, w = sc.n, sc.height, sc.width
    p = torch.from_numpy(sc.particles).cuda()
    sph = torch.from_numpy(sc.sph).cuda()
    g = torch.Generator().manual_seed(0)
    feats = (torch.rand((n, 48), generator=g) * math.pi - math.pi / 2).cuda()
    feats = feats.half().contiguous() if a.half else feats
    half = int(a.half)
    dec = fdm.FeatureDecoder(24).cuda()
    rd4 = rd.reshape(1, h, w, 3)
    target = torch.rand((1, h, w, 3), device="cuda")
    out = torch.empty((h, w, 25), device="cuda")
    rgba = torch.empty((h, w, 4), device="cuda")
    dist, hits, vis = torch.empty((h, w, 1), device="cuda"), torch.empty((h, w, 1), device="cuda"), torch.empty((n, 1), device="cuda")
    d_out, d_rgba = torch.randn((h, w, 25), device="cuda"), torch.randn((h, w, 4), device="cuda")
    d_dist = torch.zeros((h, w, 1), device="cuda")
    dp, df, ds = torch.empty((n, 12), device="cuda"), torch.empty((n, 48), device="cuda"), torch.empty((n, 48), device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")  # > the 50 MB L2

    def nht_fwd():
        ctx.forward_nht(s, cam, n, p.data_ptr(), feats.data_ptr(), 48, half, ro.data_ptr(), rd.data_ptr(), out.data_ptr(), dist.data_ptr(),
                        hits.data_ptr(), vis.data_ptr())

    def nht_bwd(grad=None):
        ctx.backward_nht(s, cam, n, p.data_ptr(), feats.data_ptr(), 48, half, ro.data_ptr(), rd.data_ptr(), out.data_ptr(),
                         (d_out if grad is None else grad).data_ptr(), dist.data_ptr(), d_dist.data_ptr(), dp.data_ptr(), df.data_ptr())

    def sh_fwd():
        ctx.forward(s, cam, n, p.data_ptr(), sph.data_ptr(), 3, ro.data_ptr(), rd.data_ptr(), rgba.data_ptr(), dist.data_ptr(), hits.data_ptr(),
                    vis.data_ptr())

    def sh_bwd():
        ctx.backward(s, cam, n, p.data_ptr(), sph.data_ptr(), 3, ro.data_ptr(), rd.data_ptr(), rgba.data_ptr(), d_rgba.data_ptr(),
                     dist.data_ptr(), d_dist.data_ptr(), dp.data_ptr(), ds.data_ptr())

    feat_in = torch.randn((1, h, w, 24), device="cuda")

    def dec_fwd():
        with torch.no_grad():
            dec(feat_in, rd4)

    def dec_fwd_bwd():
        x = feat_in.detach().requires_grad_(True)
        dec(x, rd4).sum().backward()

    def nht_frame():
        nht_fwd()
        x = out[..., :24].unsqueeze(0).detach().requires_grad_(True)
        loss = (dec(x, rd4) - target).abs().mean()
        loss.backward()
        grad = torch.cat([x.grad[0], torch.zeros((h, w, 1), device="cuda")], -1).contiguous()
        nht_bwd(grad)

    # the backward stages replay the forward before them: time them after an untimed forward of the same kind
    stages = {
        "nht_forward": (None, nht_fwd), "nht_backward": (nht_fwd, nht_bwd), "decoder_forward": (None, dec_fwd),
        "decoder_forward_backward": (None, dec_fwd_bwd), "nht_frame": (None, nht_frame),
        "sh_forward": (None, sh_fwd), "sh_backward": (sh_fwd, sh_bwd),
    }
    times = {k: [] for k in stages}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for it in range(a.warmup + a.iters):
        for name, (pre, fn) in stages.items():  # NHT and SH stages alternate within every iteration
            if pre is not None:
                pre()
            flush.zero_()
            ev0.record()
            fn()
            ev1.record()
            torch.cuda.synchronize()
            if it >= a.warmup:
                times[name].append(ev0.elapsed_time(ev1))
    med = {k: float(np.median(v)) for k, v in times.items()}
    med["sh_frame"] = med["sh_forward"] + med["sh_backward"]
    info = card()
    print(f"card: {info}")
    for k, v in med.items():
        print(f"{k:>26}: {v:.3f} ms (min {min(times[k]) if k in times else v:.3f})")
    print(json.dumps({"scene": "C2 300k 800x800", "features": "fp16" if a.half else "fp32", "card": info, "median_ms": med}))


if __name__ == "__main__":
    main()

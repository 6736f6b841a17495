"""Device time of the 3DGRT trace with NHT features on scene C4 (the C2 scene through 3DGRT: 300k Gaussians, 800x800), next to the SH
trace of the same scene.

Stages (CUDA events, L2 flushed before every timed call, warmup first): NHT forward (grtb200_trace_nht), NHT backward
(grtb200_trace_bwd_nht, replaying the forward's hit lists), SH forward (grtb200_trace) and SH backward (grtb200_trace_bwd), alternating
in one process; each backward follows an untimed forward of its kind.  Both feature precisions are timed (fp32 and fp16 rows) unless
--only fp32|fp16.  The NHT configs' max_alpha 0.999 is used for both kinds; features are drawn from U(-pi/2, pi/2), the init range of
configs/base_gs.yaml.  Prints the card (benchkit.card) and one JSON line.  A CUDA device is required.

  python scripts/bench_grt_nht.py [--iters 20] [--warmup 5] [--only fp32|fp16]
"""
from __future__ import annotations

import argparse
import json
import math

import numpy as np
import torch

import benchkit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", choices=("fp32", "fp16"), default=None)
    a = ap.parse_args()
    info = benchkit.card(benchkit.cuda_device("bench_grt_nht.py"))
    print(f"device: {info}")
    import b200_native as nat
    import scenes

    sc = scenes.scene_c2()
    c2w = np.asarray(sc.camera(0, 100), np.float32)
    r2w = np.ascontiguousarray(c2w[:3, :4])
    cfg = nat.grt_default_config()
    cfg.max_alpha = 0.999
    ctx = nat.GrtContext(cfg, 0)
    ro, rd = (torch.from_numpy(np.ascontiguousarray(t)).cuda() for t in sc.rays())
    n, h, w = sc.n, sc.height, sc.width
    R = h * w
    p = torch.from_numpy(sc.particles).cuda()
    sph = torch.from_numpy(sc.sph).cuda()
    g = torch.Generator().manual_seed(0)
    f32 = (torch.rand((n, 48), generator=g) * math.pi - math.pi / 2).cuda().contiguous()
    feats = {"fp32": f32, "fp16": f32.half().contiguous()}
    kinds = [a.only] if a.only else ["fp32", "fp16"]
    s = torch.cuda.current_stream().cuda_stream
    ctx.build_bvh_packed(s, n, p.data_ptr())
    feat, rgb = torch.empty((R, 24), device="cuda"), torch.empty((R, 3), device="cuda")
    alpha, dist, hits, vis = torch.empty(R, device="cuda"), torch.empty((R, 2), device="cuda"), torch.empty(R, device="cuda"), torch.empty(n, device="cuda")
    d_feat, d_rgb = torch.randn((R, 24), device="cuda"), torch.randn((R, 3), device="cuda")
    d_alpha, d_dist = torch.randn(R, device="cuda"), torch.zeros(R, device="cuda")
    dp, df, ds = torch.empty((n, 12), device="cuda"), torch.empty((n, 48), device="cuda"), torch.empty((n, 48), device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")  # > the 50 MB L2
    args = (1, h, w, ro.data_ptr(), rd.data_ptr(), r2w.ctypes.data)

    def nht_fwd(k):
        return lambda: ctx.trace_nht(s, n, p.data_ptr(), feats[k].data_ptr(), 48, int(k == "fp16"), 0.001, *args, feat.data_ptr(),
                                     alpha.data_ptr(), dist.data_ptr(), hits.data_ptr(), vis.data_ptr())

    def nht_bwd(k):
        return lambda: ctx.trace_bwd_nht(s, n, p.data_ptr(), feats[k].data_ptr(), 48, int(k == "fp16"), 0.001, *args, feat.data_ptr(),
                                         alpha.data_ptr(), dist.data_ptr(), d_feat.data_ptr(), d_alpha.data_ptr(), d_dist.data_ptr(),
                                         dp.data_ptr(), df.data_ptr())

    def sh_fwd():
        ctx.trace(s, n, p.data_ptr(), sph.data_ptr(), 3, 0.001, *args, rgb.data_ptr(), alpha.data_ptr(), dist.data_ptr(), hits.data_ptr(),
                  vis.data_ptr())

    def sh_bwd():
        ctx.trace_bwd(s, n, p.data_ptr(), sph.data_ptr(), 3, 0.001, *args, rgb.data_ptr(), alpha.data_ptr(), dist.data_ptr(), d_rgb.data_ptr(),
                      d_alpha.data_ptr(), d_dist.data_ptr(), dp.data_ptr(), ds.data_ptr())

    stages = {}
    for k in kinds:
        stages[f"nht_{k}_forward"] = (None, nht_fwd(k))
        stages[f"nht_{k}_backward"] = (nht_fwd(k), nht_bwd(k))
        stages[f"sh_forward_{k}_pass"] = (None, sh_fwd)  # SH stages alternate with each NHT precision
        stages[f"sh_backward_{k}_pass"] = (sh_fwd, sh_bwd)
    times = {k: [] for k in stages}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for it in range(a.warmup + a.iters):
        for name, (pre, fn) in stages.items():
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
    med["sh_forward"] = float(np.median(sum((times[k] for k in times if k.startswith("sh_forward")), [])))
    med["sh_backward"] = float(np.median(sum((times[k] for k in times if k.startswith("sh_backward")), [])))
    for k, v in med.items():
        print(f"{k:>26}: {v:.3f} ms")
    print(json.dumps({"scene": "C4 300k 800x800 (3DGRT)", "max_alpha": 0.999, "card": info, "median_ms": med}))
    ctx.close()


if __name__ == "__main__":
    main()

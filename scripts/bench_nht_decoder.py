"""Device time of the NHT feature decoder (default net: 24 features, SH degree 3, 3 hidden layers of 128, Sigmoid) at 800x800 and
1237x822 rows: this project's forward and backward, tiny-cuda-nn's (oracle/_ref/libtcnn_ref.so, when built) and a torch fp16 nn.Linear
chain (cuBLAS), timed alternately in one process with CUDA events after warm-up.  Prints achieved TFLOP/s and bytes/s computed from shapes
and the share of the binding bound (989 TFLOP/s dense fp16, 3.35 TB/s HBM3; NVIDIA H100 SXM data sheet), with the card's name and power
limit read in the same run.  Usage: python scripts/bench_nht_decoder.py [--iters 20] [--warmup 5]"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "3dgrut_b200")]

import b200_native as nat  # noqa: E402
import feature_decoder as fd  # noqa: E402
from oracle import nht_tcnn_ref  # noqa: E402

F, DEGREE, LAYERS, SH_SCALE = 24, 3, 3, 3.0
PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12


def shapes_cost(n: int, cfg):
    """(forward FLOP, backward FLOP, forward bytes, backward bytes) the algorithm needs: 2 FLOP per MAC; the backward is the input
    gradient and the weight gradient (2x the forward).  Bytes: fp32 inputs and outputs only (features, directions, rgb, d_rgb, d_features)."""
    macs = sum(o * i for o, i in fd.matrix_shapes(cfg)) * n
    fwd_b = n * (F + 3 + 3) * 4
    bwd_b = n * (F + 3 + 3 + F) * 4
    return 2 * macs, 4 * macs, fwd_b, bwd_b


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1e3  # us


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nht_decoder.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(f"card: {torch.cuda.get_device_name(0)}; nvidia-smi: {smi}")
    cfg = fd.decoder_config(F, 128, LAYERS, "SphericalHarmonics", DEGREE, SH_SCALE, "Sigmoid")
    lib = nat.nht_lib()
    params = fd.initial_params(cfg, torch.Generator().manual_seed(0)).to(dev)
    results = []
    for w, h in ((800, 800), (1237, 822)):
        n = w * h
        g = torch.Generator(device=dev).manual_seed(1)
        feat = torch.randn(n, F, device=dev, generator=g) * 0.5
        dirs = torch.nn.functional.normalize(torch.randn(n, 3, device=dev, generator=g), dim=1)
        d_out = torch.randn(n, 3, device=dev, generator=g) / n
        out = torch.empty(n, 3, device=dev)
        d_feat = torch.empty(n, F, device=dev)
        d_params = torch.empty_like(params)
        ws = torch.empty(lib.nhtb200_backward_workspace_bytes(C.byref(cfg), n), device=dev, dtype=torch.uint8)
        s = torch.cuda.current_stream().cuda_stream

        def ours_fwd():
            nat.nht_check(lib.nhtb200_forward(C.byref(cfg), s, n, feat.data_ptr(), dirs.data_ptr(), params.data_ptr(), out.data_ptr()), "fwd")

        def ours_bwd():
            nat.nht_check(lib.nhtb200_backward(C.byref(cfg), s, n, feat.data_ptr(), dirs.data_ptr(), params.data_ptr(), d_out.data_ptr(),
                                               d_feat.data_ptr(), d_params.data_ptr(), ws.data_ptr()), "bwd")

        # torch fp16 Linear chain (cuBLAS) on the encoded input: the dense-library baseline
        k0 = fd.matrix_shapes(cfg)[0][1]
        x16 = torch.randn(n, k0, device=dev, dtype=torch.float16, requires_grad=True)
        lins = [torch.nn.Linear(i, o, bias=False, device=dev, dtype=torch.float16) for o, i in fd.matrix_shapes(cfg)]
        g16 = torch.randn(n, 16, device=dev, dtype=torch.float16)

        def torch_fwd():
            with torch.no_grad():
                a = x16
                for j, l in enumerate(lins):
                    a = l(a)
                    a = torch.relu(a) if j + 1 < len(lins) else torch.sigmoid(a)

        def torch_fwd_bwd():
            a = x16
            for j, l in enumerate(lins):
                a = l(a)
                a = torch.relu(a) if j + 1 < len(lins) else torch.sigmoid(a)
            a.backward(g16)

        cases = {"ours_fwd": ours_fwd, "ours_fwd_bwd": lambda: (ours_fwd(), ours_bwd()), "torch_fp16_fwd": torch_fwd,
                 "torch_fp16_fwd_bwd": torch_fwd_bwd}
        tc = None
        if nht_tcnn_ref.available():
            tc = nht_tcnn_ref.TcnnDecoder(F, DEGREE, LAYERS)
            tc.set_params(params)
            inputs = torch.cat([feat, (dirs * SH_SCALE + 1.0) * 0.5], dim=1).contiguous()
            t_out = torch.empty(n, 3, device=dev)
            d_in = torch.empty_like(inputs)
            t_dp = torch.empty_like(params)
            cases["tcnn_fwd_inference"] = lambda: tc.forward(inputs, t_out, training=False)
            cases["tcnn_fwd_bwd"] = lambda: (tc.forward(inputs, t_out), tc.backward(n, d_out, d_in, t_dp))
        times = {k: [] for k in cases}
        for _rep in range(3):  # alternate the implementations
            for k, fn in cases.items():
                times[k].append(timed(fn, args.iters, args.warmup))
        if tc is not None:
            tc.close()
        ff, bf, fb, bb = shapes_cost(n, cfg)
        for k, ts in times.items():
            us = min(ts)
            flop = ff + (bf if "bwd" in k else 0)
            byts = fb + (bb if "bwd" in k else 0)
            bound_us = max(flop / PEAK_FLOPS, byts / PEAK_BYTES) * 1e6
            r = dict(rows=n, image=f"{w}x{h}", case=k, us=round(us, 1), us_all=[round(t, 1) for t in ts], tflops=round(flop / us / 1e6, 1),
                     gbytes_s=round(byts / us / 1e3, 1), share_of_bound=round(bound_us / us, 3),
                     bound="compute" if flop / PEAK_FLOPS > byts / PEAK_BYTES else "memory")
            results.append(r)
            print(json.dumps(r))
        if "tcnn_fwd_bwd" in times:
            print(f"{w}x{h}: forward+backward speed-up over tcnn {min(times['tcnn_fwd_bwd']) / min(times['ours_fwd_bwd']):.2f}x")
        del ws


if __name__ == "__main__":
    main()

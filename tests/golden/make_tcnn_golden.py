"""Writes tests/golden/nht_decoder_tcnn.npz: tiny-cuda-nn's own forward and backward of the NHT decoder (the reference's default
FeatureDecoder config: 24 features, SH degree 3, sh_scale 3, 3 hidden layers of 128, Sigmoid) on seeded inputs, through
oracle/_ref/libtcnn_ref.so.  Run once on an H100 from the repository root: python tests/golden/make_tcnn_golden.py [out.npz]"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import nht_decoder_oracle as ndo  # noqa: E402
from oracle.nht_tcnn_ref import TcnnDecoder  # noqa: E402

F, DEGREE, LAYERS, SH_SCALE, N = 24, 3, 3, 3.0, 3001  # N is not a multiple of 128


def main(path: str):
    rng = np.random.default_rng(20261015)
    features = rng.normal(0.0, 0.5, size=(N, F)).astype(np.float32)
    d = rng.normal(size=(N, 3))
    dirs = (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)
    params = np.concatenate([rng.uniform(-1, 1, o * i) * np.sqrt(6.0 / (o + i)) for o, i in ndo.matrix_shapes(F, DEGREE, LAYERS)])
    params = params.astype(np.float32)
    d_out = (rng.normal(size=(N, 3)) / N).astype(np.float32)

    dev = torch.device("cuda", 0)
    net = TcnnDecoder(F, DEGREE, LAYERS)
    assert net.n_params == params.size, (net.n_params, params.size)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    inputs = torch.cat([t(features), (t(dirs) * SH_SCALE + 1.0) * 0.5], dim=1).contiguous()
    out = torch.empty((N, 3), device=dev)
    d_in = torch.empty_like(inputs)
    d_params = torch.empty(params.size, device=dev)
    net.set_params(t(params))
    net.forward(inputs, out)
    net.backward(N, t(d_out), d_in, d_params)
    torch.cuda.synchronize()
    res = dict(features=features, dirs=dirs, params=params, d_out=d_out, out=out.cpu().numpy(),
               d_features=d_in[:, :F].cpu().numpy(), d_params=d_params.cpu().numpy(),
               config=np.array([F, DEGREE, LAYERS, 128], np.int32), sh_scale=np.float32(SH_SCALE),
               padded_input_width=np.int32(net.padded_input_width))
    net.close()
    # tcnn's parameter count for every SH degree and layer count the decoder builds (F = 24, and F + d^2 = 128 at degree 4)
    table = []
    for f in (24, 112):
        for degree in (1, 2, 3, 4):
            for layers in (1, 2, 3, 4):
                t_net = TcnnDecoder(f, degree, layers)
                table.append((f, degree, layers, t_net.n_params, t_net.padded_input_width))
                t_net.close()
    res["n_params_table"] = np.array(table, np.int64)
    np.savez_compressed(path, **res)

    # tcnn against float64 on its own fp16-rounded parameters: the yardstick the tests size their bounds from
    p16 = params.astype(np.float16).astype(np.float64)
    o64, df64, dp64 = ndo.forward_backward(features.astype(np.float16), dirs, p16, d_out, DEGREE, LAYERS, SH_SCALE)
    rel = lambda a, b: float(np.linalg.norm(a - b) / np.linalg.norm(b))  # noqa: E731
    print(f"wrote {path}: max|out-f64| {np.abs(res['out'] - o64).max():.3e}  rel-L2 d_features {rel(res['d_features'], df64):.3e}"
          f"  d_params {rel(res['d_params'], dp64):.3e}")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "nht_decoder_tcnn.npz"))

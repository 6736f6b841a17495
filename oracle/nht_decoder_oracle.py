"""Float64 restatement of the NHT feature decoder (TEST INFRASTRUCTURE ONLY; the product never imports it).

tiny-cuda-nn's NetworkWithInputEncoding as the reference's FeatureDecoder configures it (threedgrut/model/feature_decoder.py:69-97):
  encoding  Composite[Identity(F), SphericalHarmonics(degree d)] of [features, (dir * sh_scale + 1) / 2].  Row layout
            [features (F), ones (P), SH (d^2)]: the Composite pads its last nested encoding up to the network's 16-alignment
            (encodings/composite.h set_padded_output_width), and the SH encoding writes its padding lanes first, with value 1
            (encodings/spherical_harmonics.h kernel_sh).  The SH polynomials are tcnn's (common_device.h sh_enc), evaluated at u * 2 - 1
            of the unit-cube input u, i.e. at dir * sh_scale.
  MLP       bias-free FullyFusedMLP: W_0 [128][K0], n_hidden_layers - 1 x [128][128], W_out [16][128], row-major [out][in], concatenated
            in that order (src/fully_fused_mlp.cu constructor); ReLU on hidden layers, output activation on the 16 padded outputs, the
            first 3 returned.
The backward is float64 torch autograd of the same expressions.
"""
from __future__ import annotations

import numpy as np
import torch

WIDTH = 128
OUT_PAD = 16


def padded_input_width(n_features: int, sh_degree: int) -> int:
    return (n_features + sh_degree * sh_degree + 15) // 16 * 16


def matrix_shapes(n_features: int, sh_degree: int, n_hidden_layers: int) -> list[tuple[int, int]]:
    k0 = padded_input_width(n_features, sh_degree)
    return [(WIDTH, k0)] + [(WIDTH, WIDTH)] * (n_hidden_layers - 1) + [(OUT_PAD, WIDTH)]


def n_params(n_features: int, sh_degree: int, n_hidden_layers: int) -> int:
    return sum(o * i for o, i in matrix_shapes(n_features, sh_degree, n_hidden_layers))


def sh_basis(degree: int, x, y, z):
    """tcnn sh_enc up to degree 4 (d^2 = 16 coefficients), as a list of tensors."""
    xy, xz, yz, x2, y2, z2 = x * y, x * z, y * z, x * x, y * y, z * z
    out = [torch.full_like(x, 0.28209479177387814)]
    if degree > 1:
        out += [-0.48860251190291987 * y, 0.48860251190291987 * z, -0.48860251190291987 * x]
    if degree > 2:
        out += [1.0925484305920792 * xy, -1.0925484305920792 * yz, 0.94617469575755997 * z2 - 0.31539156525251999,
                -1.0925484305920792 * xz, 0.54627421529603959 * x2 - 0.54627421529603959 * y2]
    if degree > 3:
        out += [0.59004358992664352 * y * (-3.0 * x2 + y2), 2.8906114426405538 * xy * z, 0.45704579946446572 * y * (1.0 - 5.0 * z2),
                0.3731763325901154 * z * (5.0 * z2 - 3.0), 0.45704579946446572 * x * (1.0 - 5.0 * z2), 1.4453057213202769 * z * (x2 - y2),
                0.59004358992664352 * x * (-x2 + 3.0 * y2)]
    return out


def encode(features: torch.Tensor, dirs: torch.Tensor, sh_degree: int, sh_scale: float) -> torch.Tensor:
    """[n, K0] encoded rows.  The direction enters as tcnn receives it, u = (dir * sh_scale + 1) / 2, and is mapped back by u * 2 - 1."""
    n, f = features.shape
    u = (dirs * sh_scale + 1.0) * 0.5
    c = u * 2.0 - 1.0
    sh = torch.stack(sh_basis(sh_degree, c[:, 0], c[:, 1], c[:, 2]), dim=1)
    pad = padded_input_width(f, sh_degree) - f - sh_degree * sh_degree
    return torch.cat([features, torch.ones((n, pad), dtype=features.dtype, device=features.device), sh], dim=1)


def activate(name: str, x: torch.Tensor) -> torch.Tensor:
    return {"Sigmoid": torch.sigmoid, "ReLU": torch.relu, "None": lambda v: v}[name](x)


def _fp16_storage(a: torch.Tensor) -> torch.Tensor:
    """a rounded to fp16 in value, with the identity as its derivative (the gradient flows to the stored activation unchanged)."""
    return a + (a.to(torch.float16).to(a.dtype) - a).detach()


def forward(features, dirs, params, sh_degree: int, n_hidden_layers: int, sh_scale: float, output_activation: str = "Sigmoid",
            fp16_activations: bool = False):
    """rgb [n, 3] in float64 (torch tensors in, differentiable in features and params).  fp16_activations rounds the encoded input and
    every hidden activation to fp16, as a network with fp16 operands stores them; everything else stays float64."""
    f = features.shape[1]
    a = encode(features, dirs, sh_degree, sh_scale)
    off = 0
    shapes = matrix_shapes(f, sh_degree, n_hidden_layers)
    for m, (o, i) in enumerate(shapes):
        if fp16_activations:
            a = _fp16_storage(a)
        w = params[off:off + o * i].reshape(o, i)
        off += o * i
        a = a @ w.T
        if m + 1 < len(shapes):
            a = torch.relu(a)
    return activate(output_activation, a)[:, :3]


def forward_backward(features, dirs, params, d_out, sh_degree, n_hidden_layers, sh_scale, output_activation="Sigmoid",
                     fp16_activations=False):
    """numpy in, float64 numpy (out [n,3], d_features [n,F], d_params [n_params]) out."""
    feat = torch.tensor(np.asarray(features, np.float64), requires_grad=True)
    prm = torch.tensor(np.asarray(params, np.float64), requires_grad=True)
    out = forward(feat, torch.tensor(np.asarray(dirs, np.float64)), prm, sh_degree, n_hidden_layers, sh_scale, output_activation,
                  fp16_activations)
    out.backward(torch.tensor(np.asarray(d_out, np.float64)))
    return out.detach().numpy(), feat.grad.numpy(), prm.grad.numpy()

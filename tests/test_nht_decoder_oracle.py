"""The float64 NHT decoder oracle (oracle/nht_decoder_oracle.py) against tiny-cuda-nn's own outputs (tests/golden/nht_decoder_tcnn.npz,
made by tests/golden/make_tcnn_golden.py on an H100) and against central differences.  No GPU needed."""
import os

import numpy as np
import pytest
import torch

from oracle import nht_decoder_oracle as ndo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "nht_decoder_tcnn.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - b) / np.linalg.norm(b))


def _oracle(z, **kw):
    f, degree, layers, _ = (int(v) for v in z["config"])
    return ndo.forward_backward(z["features"].astype(np.float16), z["dirs"], z["params"].astype(np.float16), z["d_out"], degree, layers,
                                float(z["sh_scale"]), **kw)


# tiny-cuda-nn runs fp16 operands with fp16 accumulation in its hidden layers and stores fp16 activations and outputs, so it sits at a
# distance from float64 that is a property of tcnn, measured on this golden (H100, FullyFusedMLP): max |out| error 4.7e-4, rel-L2
# 2.2e-2 for d_features and 2.5e-2 for d_params.  The bounds are those figures with headroom; a wrong padding value or order, SH
# polynomial, sh_scale or params layout moves every figure by orders of magnitude (test_golden_pins_the_layout).
OUT_BOUND, GRAD_BOUND = 2e-3, 6e-2


def test_oracle_reproduces_tcnn_golden(golden):
    z = golden
    out, df, dp = _oracle(z)
    errs = (np.abs(z["out"] - out).max(), _rel(z["d_features"], df), _rel(z["d_params"], dp))
    print(f"tcnn vs float64 oracle: max|out| {errs[0]:.2e}  d_features {errs[1]:.2e}  d_params {errs[2]:.2e}")
    assert errs[0] <= OUT_BOUND and errs[1] <= GRAD_BOUND and errs[2] <= GRAD_BOUND, errs
    assert int(z["padded_input_width"]) == ndo.padded_input_width(24, 3) == 48


def test_golden_pins_the_layout(golden, monkeypatch):
    """The alternative readings of tcnn's encoding are far from the golden: ones after the SH block, or sh_scale ignored."""
    z = golden
    good = np.abs(_oracle(z)[0] - z["out"]).max()

    def pad_last(features, dirs, sh_degree, sh_scale):
        n, f = features.shape
        c = (dirs * sh_scale + 1.0) * 0.5 * 2.0 - 1.0
        sh = torch.stack(ndo.sh_basis(sh_degree, c[:, 0], c[:, 1], c[:, 2]), dim=1)
        pad = ndo.padded_input_width(f, sh_degree) - f - sh_degree * sh_degree
        return torch.cat([features, sh, torch.ones((n, pad), dtype=features.dtype)], dim=1)

    with monkeypatch.context() as m:
        m.setattr(ndo, "encode", pad_last)
        assert np.abs(_oracle(z)[0] - z["out"]).max() > 20 * good
    f, degree, layers, _ = (int(v) for v in z["config"])
    unscaled = ndo.forward_backward(z["features"].astype(np.float16), z["dirs"], z["params"].astype(np.float16), z["d_out"], degree, layers,
                                    1.0)[0]
    assert np.abs(unscaled - z["out"]).max() > 20 * good


def test_n_params_matches_tcnn(golden):
    import ctypes as C

    import feature_decoder as fd
    import b200_native as nat

    for f, degree, layers, n_params, k0 in golden["n_params_table"]:
        assert ndo.n_params(int(f), int(degree), int(layers)) == n_params
        assert ndo.padded_input_width(int(f), int(degree)) == k0
        cfg = fd.decoder_config(int(f), 128, int(layers), "SphericalHarmonics", int(degree), 3.0, "Sigmoid")
        assert nat.nht_lib().nhtb200_n_params(C.byref(cfg)) == n_params


@pytest.mark.parametrize("act", ["Sigmoid", "ReLU", "None"])
def test_oracle_autograd_matches_central_differences(act):
    rng = np.random.default_rng(3)
    f, degree, layers, n = 5, 2, 2, 7
    feat = rng.normal(size=(n, f))
    d = rng.normal(size=(n, 3))
    dirs = d / np.linalg.norm(d, axis=1, keepdims=True)
    params = np.concatenate([rng.uniform(-1, 1, o * i) * np.sqrt(6.0 / (o + i)) for o, i in ndo.matrix_shapes(f, degree, layers)])
    d_out = rng.normal(size=(n, 3))
    _, df, dp = ndo.forward_backward(feat, dirs, params, d_out, degree, layers, 3.0, act)

    def loss(fe, pa):
        out = ndo.forward(torch.tensor(fe), torch.tensor(dirs), torch.tensor(pa), degree, layers, 3.0, act)
        return float((out.numpy() * d_out).sum())

    h = 1e-6
    for _ in range(12):
        i, j = rng.integers(n), rng.integers(f)
        e = np.zeros_like(feat)
        e[i, j] = h
        num = (loss(feat + e, params) - loss(feat - e, params)) / (2 * h)
        assert abs(num - df[i, j]) <= 1e-6 * max(1.0, abs(num)), (num, df[i, j])
    for k in rng.choice(params.size, 24, replace=False):
        e = np.zeros_like(params)
        e[k] = h
        num = (loss(feat, params + e) - loss(feat, params - e)) / (2 * h)
        assert abs(num - dp[k]) <= 1e-6 * max(1.0, abs(num)), (num, dp[k])

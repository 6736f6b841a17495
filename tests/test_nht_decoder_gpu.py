"""The NHT feature decoder (include/nht_b200.h, feature_decoder.FeatureDecoder) on the GPU, against the float64 oracle, tiny-cuda-nn's own
golden outputs and, where oracle/_ref/libtcnn_ref.so was built, tiny-cuda-nn live."""
import os

import numpy as np
import pytest
import torch

from oracle import nht_decoder_oracle as ndo
from oracle import nht_tcnn_ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "nht_decoder_tcnn.npz")
F, DEGREE, LAYERS, SH_SCALE = 24, 3, 3, 3.0
DEV = torch.device("cuda", 0)


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - b) / max(np.linalg.norm(b), 1e-300))


def _inputs(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    feat = torch.randn(n, F, generator=g) * 0.5
    d = torch.randn(n, 3, generator=g)
    dirs = d / d.norm(dim=1, keepdim=True)
    return feat, dirs


def _cfg(act="Sigmoid", degree=DEGREE, layers=LAYERS, f=F):
    import feature_decoder as fd

    return fd.decoder_config(f, 128, layers, "SphericalHarmonics", degree, SH_SCALE, act)


def _params(cfg, seed=1):
    import feature_decoder as fd

    return fd.initial_params(cfg, torch.Generator().manual_seed(seed))


def _run(cfg, feat, dirs, params, d_out=None):
    import feature_decoder as fd

    f = feat.to(DEV).requires_grad_(d_out is not None)
    p = params.to(DEV).requires_grad_(d_out is not None)
    out = fd.decode(f, dirs.to(DEV), p, cfg)
    if d_out is None:
        return out.detach().cpu().numpy()
    out.backward(d_out.to(DEV))
    return out.detach().cpu().numpy(), f.grad.cpu().numpy(), p.grad.cpu().numpy()


def _oracle(cfg, feat, dirs, params, d_out, act="Sigmoid", fp16_activations=False):
    # the oracle sees the operands as the tensor cores do: fp16 features and params
    f16 = feat.numpy().astype(np.float16).astype(np.float64)
    p16 = params.numpy().astype(np.float16).astype(np.float64)
    return ndo.forward_backward(f16, dirs.numpy(), p16, d_out.numpy(), cfg.sh_degree, cfg.n_hidden_layers, SH_SCALE, act, fp16_activations)


# Forward bound: fp16 operands with fp32 accumulation.  Each hidden activation is rounded to fp16 (relative 2^-11) before the next layer;
# through 4 matrices the rounding of ~128-term sums of unit-size terms leaves |error| of a few 1e-4 on the pre-activation, and the
# sigmoid's slope (<= 1/4) scales it down.  2e-3 is ~4x the largest error measured at 1,000,003 rows.
FWD_BOUND = 2e-3


@pytest.mark.parametrize("n", [1, 127, 1_000_003, 640_000])
def test_forward_against_float64(n):
    cfg = _cfg()
    feat, dirs = _inputs(n)
    params = _params(cfg)
    out = _run(cfg, feat, dirs, params)
    m = min(n, 20000)  # the float64 oracle on a prefix (all rows for the small cases, tails included)
    ref, _, _ = _oracle(cfg, feat[:m], dirs[:m], params, torch.zeros(m, 3))
    err = np.abs(out[:m] - ref).max()
    tail = np.abs(out[-min(n, 127):] - _oracle(cfg, feat[-min(n, 127):], dirs[-min(n, 127):], params, torch.zeros(min(n, 127), 3))[0]).max()
    print(f"n={n}: max |out - f64| {err:.3e}, last rows {tail:.3e} (bound {FWD_BOUND})")
    assert np.isfinite(out).all() and err <= FWD_BOUND and tail <= FWD_BOUND


@pytest.mark.parametrize("act", ["Sigmoid", "ReLU", "None"])
@pytest.mark.parametrize("degree,layers,f", [(3, 3, 24), (1, 1, 8), (2, 2, 13), (4, 4, 32), (4, 2, 112)])
def test_backward_against_float64(act, degree, layers, f):
    cfg = _cfg(act, degree, layers, f)
    n = 4099
    g = torch.Generator().manual_seed(7)
    feat = torch.randn(n, f, generator=g) * 0.5
    d = torch.randn(n, 3, generator=g)
    dirs = d / d.norm(dim=1, keepdim=True)
    params = _params(cfg)
    d_out = torch.randn(n, 3, generator=g) / n
    out, df, dp = _run(cfg, feat, dirs, params, d_out)
    # Against plain float64 the gradients sit at ~2e-2 rel-L2 (tiny-cuda-nn: ~3e-2): fp16 storage of the activations moves pre-activations
    # by ~1e-4, which flips the ReLU mask of about 1e-4 of the units, and rel-L2 grows as the square root of that share.  So the backward
    # is held to 1e-3 against the float64 oracle that stores its activations in fp16 as the network does (fp16_activations); the
    # distance from plain float64 is pinned by the tiny-cuda-nn comparisons below.  With 4 hidden layers that oracle stops being a
    # twin: fp32-vs-fp64 accumulation flips the fp16 rounding of ~4e-4 of the activations, each flip moves the next layer by an ulp,
    # and two layers later the two nets round independently; measured 9e-3 there, so 4 hidden layers are held to 2e-2 (below tcnn's
    # own 2.5e-2 from float64 on the default net).
    bound = 1e-3 if layers <= 3 else 2e-2
    ro, rdf, rdp = _oracle(cfg, feat, dirs, params, d_out, act, fp16_activations=True)
    errs = {"out": float(np.abs(out - ro).max()), "d_features": _rel(df, rdf)}
    off = 0
    for m, (o, i) in enumerate(ndo.matrix_shapes(f, degree, layers)):
        blk = slice(off, off + o * i)
        errs[f"W{m}"] = _rel(dp[blk], rdp[blk]) if np.linalg.norm(rdp[blk]) > 0 else float(np.abs(dp[blk]).max())
        off += o * i
    print(act, degree, layers, f, {k: f"{v:.2e}" for k, v in errs.items()})
    assert errs["out"] <= FWD_BOUND
    assert all(v <= bound for k, v in errs.items() if k != "out"), errs


def test_backward_is_deterministic_and_zero_rows():
    cfg = _cfg()
    feat, dirs = _inputs(5000, seed=3)
    params = _params(cfg)
    d_out = torch.randn(5000, 3) / 5000
    a = _run(cfg, feat, dirs, params, d_out)
    b = _run(cfg, feat, dirs, params, d_out)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    _, df, dp = _run(cfg, feat, dirs, params, torch.zeros(5000, 3))
    assert not df.any() and not dp.any()
    _, _, dp0 = _run(cfg, feat[:0], dirs[:0], params, torch.zeros(0, 3))
    assert not dp0.any()


def test_against_tcnn_golden():
    """No further from float64 than tiny-cuda-nn itself is, on tcnn's golden inputs."""
    z = np.load(GOLDEN)
    cfg = _cfg()
    feat, dirs, params, d_out = (torch.from_numpy(z[k]) for k in ("features", "dirs", "params", "d_out"))
    out, df, dp = _run(cfg, feat, dirs, params, d_out)
    ro, rdf, rdp = _oracle(cfg, feat, dirs, params, d_out)
    ours = (np.abs(out - ro).max(), _rel(df, rdf), _rel(dp, rdp))
    tcnn = (np.abs(z["out"] - ro).max(), _rel(z["d_features"], rdf), _rel(z["d_params"], rdp))
    print(f"vs float64: ours {ours}, tcnn {tcnn}")
    assert all(o <= t for o, t in zip(ours, tcnn)), (ours, tcnn)
    assert np.abs(out - z["out"]).max() <= 2 * tcnn[0] + FWD_BOUND


@pytest.mark.skipif(not nht_tcnn_ref.available(), reason="oracle/_ref/libtcnn_ref.so was not built (needs the reference's sources)")
def test_against_tcnn_live_640k():
    n = 640_000
    cfg = _cfg()
    feat, dirs = _inputs(n, seed=5)
    params = _params(cfg)
    d_out = torch.randn(n, 3, generator=torch.Generator().manual_seed(6)) / n
    out, df, dp = _run(cfg, feat, dirs, params, d_out)
    net = nht_tcnn_ref.TcnnDecoder(F, DEGREE, LAYERS)
    inputs = torch.cat([feat, (dirs * SH_SCALE + 1.0) * 0.5], dim=1).to(DEV).contiguous()
    t_out = torch.empty(n, 3, device=DEV)
    d_in = torch.empty_like(inputs)
    t_dp = torch.empty(net.n_params, device=DEV)
    net.set_params(params.to(DEV))
    net.forward(inputs, t_out)
    net.backward(n, d_out.to(DEV), d_in, t_dp)
    torch.cuda.synchronize()
    net.close()
    m = 20000
    ro, rdf, _ = _oracle(cfg, feat[:m], dirs[:m], params, d_out[:m])
    ours = (np.abs(out[:m] - ro).max(), _rel(df[:m], rdf))
    tc = (np.abs(t_out.cpu().numpy()[:m] - ro).max(), _rel(d_in[:m, :F].cpu().numpy(), rdf))
    dp_dist = _rel(dp, t_dp.cpu().numpy().astype(np.float64))
    print(f"640k vs float64 (first {m} rows): ours {ours}, tcnn {tc}; d_params ours vs tcnn rel-L2 {dp_dist:.2e}")
    assert all(o <= t for o, t in zip(ours, tc)), (ours, tc)
    assert dp_dist <= 5e-2


def test_feature_decoder_module():
    import feature_decoder as fd

    torch.manual_seed(0)
    dec = fd.FeatureDecoder(F, 128, LAYERS, "SphericalHarmonics", DEGREE, SH_SCALE, "Sigmoid", ema_decay=0.9,
                            unpremultiply_alpha=True).to(DEV)
    assert [k for k in dec.state_dict()] == ["network.params"] and dec.network.params.dtype == torch.float32
    feat, dirs = _inputs(2 * 5 * 7)
    feat, dirs = feat.to(DEV), dirs.to(DEV)
    flat = dec(feat, dirs)
    four = dec(feat.reshape(2, 5, 7, F), dirs.reshape(2, 5, 7, 3))
    assert flat.shape == (70, 3) and four.shape == (2, 5, 7, 3) and torch.equal(four.reshape(70, 3), flat)
    alpha = torch.rand(70, 1, device=DEV) * 0.9 + 0.05
    un = dec(feat, dirs, alpha)
    assert torch.allclose(un, fd.decode(feat / alpha, dirs, dec.network.params, dec.config) * alpha)
    # EMA round trip
    p0 = dec.network.params.detach().clone()
    with torch.no_grad():
        dec.network.params.add_(1.0)
    dec.ema_update(0)
    dec.apply_ema_shadow()
    assert torch.allclose(dec.network.params, p0 + 0.1, atol=1e-6)
    dec.restore_ema()
    assert torch.equal(dec.network.params, p0 + 1.0)
    # state dict saved and loaded
    sd = {k: v.clone() for k, v in dec.state_dict().items()}
    dec2 = fd.FeatureDecoder(F, 128, LAYERS, "SphericalHarmonics", DEGREE, SH_SCALE, "Sigmoid").to(DEV)
    dec2.load_state_dict(sd)
    assert torch.equal(dec2(feat, dirs), dec(feat, dirs))
    assert "hidden_dim=128" in repr(dec) and dec.regularization_loss().item() > 0


def test_fit_matches_a_float32_torch_mlp():
    """300 Adam steps (lr 6.8e-4) onto a smooth target: the loss falls as a float32 torch MLP's from the same initial params."""
    import feature_decoder as fd

    n = 8192
    feat, dirs = _inputs(n, seed=11)
    feat, dirs = feat.to(DEV), dirs.to(DEV)
    target = torch.sigmoid(torch.stack([feat[:, 0] + dirs[:, 0], feat[:, 1] * feat[:, 2] - dirs[:, 1], torch.sin(2 * feat[:, 3]) + dirs[:, 2]], 1))
    dec = fd.FeatureDecoder(F, 128, LAYERS, "SphericalHarmonics", DEGREE, SH_SCALE, "Sigmoid").to(DEV)
    ref = dec.network.params.detach().clone().requires_grad_(True)
    opt = torch.optim.Adam(dec.parameters(), lr=6.8e-4)
    opt_ref = torch.optim.Adam([ref], lr=6.8e-4)
    losses = []
    for _ in range(300):
        opt.zero_grad()
        loss = ((dec(feat, dirs) - target) ** 2).mean()
        loss.backward()
        opt.step()
        opt_ref.zero_grad()
        loss_ref = ((_torch_mlp(feat, dirs, ref) - target) ** 2).mean()
        loss_ref.backward()
        opt_ref.step()
        losses.append((loss.item(), loss_ref.item()))
    (l0, r0), (l1, r1) = losses[0], losses[-1]
    print(f"fit: ours {l0:.4e} -> {l1:.4e}, float torch {r0:.4e} -> {r1:.4e}")
    assert l1 < 0.5 * l0 and abs(l1 - r1) <= 0.1 * r1


def _torch_mlp(feat, dirs, params):
    """The oracle's network in torch on the GPU (float32), the yardstick of the fit."""
    a = ndo.encode(feat, dirs, DEGREE, SH_SCALE)
    off = 0
    shapes = ndo.matrix_shapes(F, DEGREE, LAYERS)
    p = params
    for m, (o, i) in enumerate(shapes):
        a = a @ p[off:off + o * i].reshape(o, i).T
        off += o * i
        if m + 1 < len(shapes):
            a = torch.relu(a)
    return torch.sigmoid(a)[:, :3]

"""Pins tests/loss_terms_oracle.py -- background compositing, the image mask and the opacity / scale regularisers of the reference loss --
against torch autograd of the reference's formulas (model/background.py:80-93, trainer.py:691-736) and torch.optim.Adam on the CPU."""
import numpy as np
import pytest

torch = pytest.importorskip("torch")

import loss_terms_oracle as lto  # noqa: E402
from oracle import adam_oracle as ao  # noqa: E402
from test_adam_oracle import LRS, _state  # noqa: E402
from test_loss_oracle import _torch_loss  # noqa: E402


def _inputs(h=37, w=45, seed=0):
    rng = np.random.default_rng(seed)
    y = rng.uniform(0, 1, (h, w, 3))
    rgb = np.clip(0.7 * y + 0.1 * rng.normal(size=(h, w, 3)), 0, 1.2)
    alpha = rng.uniform(0.05, 1.0, (h, w, 1))
    return rng, rgb, alpha, y


BACKGROUNDS = {"black": None, "white": (1.0, 1.0, 1.0), "colour": (0.2, 0.5, 0.9), "random": "image"}
MASKS = ("none", "random", "zeros", "ones")


@pytest.mark.parametrize("background", list(BACKGROUNDS))
@pytest.mark.parametrize("mask", MASKS)
def test_composited_masked_loss_matches_autograd(background, mask):
    rng, rgb, alpha, y = _inputs(seed=len(background) * 7 + len(mask))
    h, w = y.shape[:2]
    bg = BACKGROUNDS[background]
    if bg == "image":
        bg = rng.uniform(0, 1, (h, w, 3))
    m = {"none": None, "random": (rng.uniform(size=(h, w)) > 0.3).astype(np.float64), "zeros": np.zeros((h, w)), "ones": np.ones((h, w))}[mask]
    # the reference's formulas, fp64 autograd
    t_rgb = torch.tensor(rgb, requires_grad=True)
    t_alpha = torch.tensor(alpha, requires_grad=True)
    t_y = torch.tensor(y)
    x = t_rgb
    if bg is not None:
        x = x + torch.tensor(np.broadcast_to(bg, rgb.shape).copy()) * (1.0 - t_alpha)   # background.py:91 / 93
    if m is not None:
        tm = torch.tensor(m)[..., None]
        x, t_y = x * tm, t_y * tm                                                          # trainer.py:693-694
    loss_t, ssim_t = _torch_loss(x, t_y, 0.8, 0.2)
    loss_t.backward()
    loss, l1, ssim, d_rgb, d_alpha = lto.composited_loss_and_gradients(rgb, alpha, y, 0.8, 0.2, background=bg, mask=m)
    assert abs(loss - float(loss_t.detach())) <= 1e-10 and abs(ssim - float(ssim_t.detach())) <= 1e-10
    assert np.abs(d_rgb - t_rgb.grad.numpy()).max() <= 1e-10
    want_alpha = t_alpha.grad.numpy() if t_alpha.grad is not None else np.zeros_like(alpha)
    assert np.abs(d_alpha - want_alpha).max() <= 1e-10
    if bg is None:
        assert not d_alpha.any()
    if mask == "zeros":
        assert not d_rgb.any() and not d_alpha.any()


def _torch_regularised_adam(params, seq, steps, lo, ls, visibility=None, update=True):
    """torch autograd through sigmoid / exp / normalize + lo mean|sigmoid| + ls mean|exp|, then torch.optim.Adam, or with `visibility`
    the selective rule restated from optimizers.cu:66-80 on the visible rows.  Returns (parameters, per-step raw gradients)."""
    leaves = {k: torch.tensor(v, requires_grad=True) for k, v in params.items()}
    opt = torch.optim.Adam([{"params": [leaves[k]], "lr": LRS[k]} for k in ao.GROUPS], lr=0.0, eps=1e-15)
    mom = {k: (torch.zeros_like(v), torch.zeros_like(v)) for k, v in leaves.items()}
    grads = []
    for dp, ds in seq[:steps]:
        opt.zero_grad()
        dns, scl = torch.sigmoid(leaves["density"]), torch.exp(leaves["scale"])
        act = torch.cat([leaves["positions"], dns, torch.nn.functional.normalize(leaves["rotation"]), scl, torch.zeros_like(leaves["density"])], 1)
        feat = torch.cat([leaves["features_albedo"], leaves["features_specular"]], 1)
        loss = (act * torch.tensor(dp)).sum() + (feat * torch.tensor(ds)).sum() + lo * dns.abs().mean() + ls * scl.abs().mean()
        loss.backward()
        grads.append({k: v.grad.detach().clone().numpy() for k, v in leaves.items()})
        if not update:
            continue
        if visibility is None:
            opt.step()
            continue
        vis = torch.tensor(visibility)
        b1, b2, eps = torch.tensor(0.9, dtype=torch.float32), torch.tensor(0.999, dtype=torch.float32), 1e-15
        with torch.no_grad():
            for k, leaf in leaves.items():
                m, v = mom[k]
                g = leaf.grad
                m_new = b1 * m + (1 - b1) * g
                v_new = b2 * v + (1 - b2) * g * g
                p_new = leaf - LRS[k] * m_new / (torch.sqrt(v_new) + eps)
                leaf[vis] = p_new[vis]
                m[vis] = m_new[vis]
                v[vis] = v_new[vis]
    return {k: v.detach().numpy() for k, v in leaves.items()}, grads


def test_regularised_chain_rule_matches_autograd():
    params, dp, ds = _state()
    _, grads = _torch_regularised_adam(params, [(dp, ds)], 1, 0.01, 0.01, update=False)
    got = lto.raw_gradients(params, dp, ds, 0.01, 0.01)
    for k in ao.GROUPS:
        assert np.allclose(got[k], grads[0][k], rtol=2e-6, atol=1e-7), k
    # the regularisers' part alone
    zp, zs = np.zeros_like(dp), np.zeros_like(ds)
    _, g0 = _torch_regularised_adam(params, [(zp, zs)], 1, 0.05, 0.02, update=False)
    got0 = lto.raw_gradients(params, zp, zs, 0.05, 0.02)
    for k in ("density", "scale"):
        assert np.abs(got0[k]).max() > 0 and np.allclose(got0[k], g0[0][k], rtol=2e-6, atol=1e-12), k
    want = 0.05 * (1 / (1 + np.exp(-params["density"].astype(np.float64)))).mean() + 0.02 * np.exp(params["scale"].astype(np.float64)).mean()
    assert abs(lto.regulariser_loss(params, 0.05, 0.02) - want) <= 1e-12


@pytest.mark.parametrize("selective", [False, True])
def test_three_regularised_adam_steps_match_torch(selective):
    params, _, _ = _state()
    rng = np.random.default_rng(5)
    seq = [(rng.normal(size=(257, 12)).astype(np.float32), rng.normal(size=(257, 48)).astype(np.float32)) for _ in range(3)]
    vis = (rng.uniform(size=257) > 0.4) if selective else None
    want, _ = _torch_regularised_adam(params, seq, 3, 0.3, 0.2, visibility=vis)
    p = {k: v.copy() for k, v in params.items()}
    m = {k: np.zeros_like(v) for k, v in params.items()}
    v = {k: np.zeros_like(vv) for k, vv in params.items()}
    for t, (dp, ds) in enumerate(seq, 1):
        p, m, v = lto.gaussian_adam_step(p, m, v, LRS, dp, ds, eps=1e-15, step=t, selective=selective, visibility=vis, lambda_opacity=0.3,
                                         lambda_scale=0.2)
    for k in ao.GROUPS:
        assert np.allclose(p[k], want[k], rtol=1e-5, atol=1e-6), k
    if selective:
        # the regulariser gradient is non-zero on every row, yet the invisible rows do not move (SelectiveAdam)
        assert np.abs(lto.raw_gradients(params, np.zeros((257, 12), np.float32), np.zeros((257, 48), np.float32), 0.3, 0.2)["density"]).min() > 0
        for k in ao.GROUPS:
            assert np.array_equal(p[k][~vis], params[k][~vis]) and not np.array_equal(p[k][vis], params[k][vis]), k

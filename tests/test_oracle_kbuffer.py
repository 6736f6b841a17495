"""The oracle of the sorted (k-buffer) 3DGUT variant (SURVEY.md 8f row 4; renderers/gutKBufferRenderer.cuh:62-112,274-352) against its
defining properties.  Its CUDA twin (gut_render_kbuffer.cu) is compared with it in test_kbuffer_gpu.py, test_kbuffer_host_emul.py and the
k = 16 cases of test_gut_off_default_gpu.py."""
import numpy as np

import scenes
from helpers import oracle_camera
from oracle import gut_oracle as go


def _frame(k, cam_index=2, scale=1.0):
    sc = scenes.scene_c1(n=400, width=64, height=48)
    if scale != 1.0:
        sc.particles[:, 8:11] *= scale
    cfg = go.default_config()
    cam, _ = oracle_camera(sc, sc.camera(cam_index, 5))
    ro, rd = sc.rays()
    pr = go.project(cfg, cam, sc.particles, sc.sph, 3)
    bn = go.bin_tiles(cfg, cam, pr)
    base = go.render_forward(cfg, cam, ro, rd, sc.particles, pr, bn)
    kb = go.render_forward_kbuffer(cfg, cam, k, ro, rd, sc.particles, pr, bn) if k else None
    return sc, cfg, cam, ro, rd, pr, bn, base, kb


def test_large_buffer_composites_in_exact_hit_distance_order():
    """With K >= the number of hits of a ray nothing is flushed early: the ray is composited strictly by hit distance.  Restated in
    numpy from the per-hit oracle (hit_forward) on a few rays."""
    sc, cfg, cam, ro, rd, pr, bn, base, kb = _frame(64, scale=2.5)
    rgba_k, dist_k, hits_k = kb
    inv = go.sensor_matrices(cam)[1]
    Rm, t = inv[:3].T, inv[3]
    gx = (sc.width + 15) // 16
    rng = np.random.default_rng(0)
    checked = 0
    for _ in range(200):
        py, px = int(rng.integers(0, sc.height)), int(rng.integers(0, sc.width))
        if hits_k[py, px, 0] < 3 or hits_k[py, px, 0] > 60:
            continue
        tile = (py // 16) * gx + px // 16
        b, e = bn.ranges.reshape(-1, 2)[tile]
        o = (Rm @ ro.reshape(sc.height, sc.width, 3)[py, px] + t).astype(np.float32)
        d = (Rm @ rd.reshape(sc.height, sc.width, 3)[py, px]).astype(np.float32)
        found = []
        for idx in bn.sorted_values[b:e]:
            acc, alpha, tt = go.hit_forward(cfg, o, d, sc.particles[idx])
            if acc:
                found.append((tt, alpha, idx))
        found.sort(key=lambda h: h[0])
        T, c = 1.0, np.zeros(3)
        for tt, alpha, idx in found:
            c += alpha * T * np.maximum(pr.rgb[idx], 0)
            T *= 1 - alpha
            if T < cfg.min_transmittance:
                break
        assert np.allclose(rgba_k[py, px, :3], c, atol=2e-5) and abs(rgba_k[py, px, 3] - (1 - T)) <= 2e-5
        checked += 1
    assert checked >= 10


def test_kbuffer_equals_unsorted_when_list_order_is_hit_order_and_differs_otherwise():
    sc, cfg, cam, ro, rd, pr, bn, base, kb = _frame(16, scale=2.5)
    # the per-particle depth order of the lists is not the per-ray hit order for large overlapping Gaussians: some pixels must change
    assert np.abs(kb[0] - base[0]).max() > 1e-4
    # opacity is order-independent as long as no early termination differs: compare where the ray did not saturate (small Gaussians)
    _, _, _, _, _, _, _, base1, kb1 = _frame(16, scale=1.0)
    unsat = (base1[0][..., 3] < 0.99) & (kb1[0][..., 3] < 0.99)
    assert unsat.sum() > 100 and np.allclose(kb1[0][..., 3][unsat], base1[0][..., 3][unsat], atol=1e-5)
    # K = 1 still reorders at most adjacent hits; K = 64 is the fully sorted limit: the images converge as K grows
    e = []
    full = _frame(64, scale=2.5)[8][0]
    for k in (1, 4, 16):
        e.append(float(np.abs(_frame(k, scale=2.5)[8][0] - full).mean()))
    assert e[0] >= e[1] >= e[2]


def test_kbuffer_backward_equals_autograd():
    """The oracle's k-buffer adjoint against torch autograd (float64) of the same forward: per pixel the hit quantities are differentiable
    torch expressions, the processing ORDER (and the early termination) is replayed from a numpy emulation of the buffer on the detached
    values -- the order is piecewise constant, so this is the exact gradient the adjoint must produce."""
    import pytest

    torch = pytest.importorskip("torch")
    from test_oracle_autograd import _rot_rows, _sh

    K = 4
    sc = scenes.scene_c1(n=60, seed=31, width=32, height=24)
    sc.particles[:, 8:11] *= 2.0
    sc.particles[:, 3] = np.minimum(sc.particles[:, 3], 0.6)  # keep alpha below the 0.99 clamp the hand adjoint does not mask
    cfg = go.default_config()
    cam, _ = oracle_camera(sc, sc.camera(1, 5))
    ro, rd = sc.rays()
    pr = go.project(cfg, cam, sc.particles, sc.sph, 3)
    bn = go.bin_tiles(cfg, cam, pr)
    rgba, dist, hits = go.render_forward_kbuffer(cfg, cam, K, ro, rd, sc.particles, pr, bn)
    assert hits.max() > K  # the buffer does flush early on some rays
    rng = np.random.default_rng(4)
    d_rgba = rng.normal(size=rgba.shape).astype(np.float32)
    d_dist = (0.2 * rng.normal(size=dist.shape)).astype(np.float32)
    dp, ds = go.render_backward_kbuffer(cfg, cam, K, ro, rd, sc.particles, sc.sph, 3, pr, bn, rgba, dist, d_rgba, d_dist)

    f64 = torch.float64
    P = torch.tensor(sc.particles, dtype=f64)
    pos = P[:, 0:3].clone().requires_grad_(True)
    dns = P[:, 3].clone().requires_grad_(True)
    quat = P[:, 4:8].clone().requires_grad_(True)
    scl = P[:, 8:11].clone().requires_grad_(True)
    sph = torch.tensor(sc.sph, dtype=f64).reshape(-1, 16, 3).clone().requires_grad_(True)
    _, inv, campos = go.sensor_matrices(cam)
    inv_t, campos_t = torch.tensor(inv, dtype=f64), torch.tensor(campos, dtype=f64)
    W, H = sc.width, sc.height
    gx = (W + 15) // 16
    o_w = torch.tensor(ro.reshape(-1, 3), dtype=f64) @ inv_t[:3] + inv_t[3]
    d_w = torch.tensor(rd.reshape(-1, 3), dtype=f64) @ inv_t[:3]
    g_rgba = torch.tensor(d_rgba.reshape(-1, 4), dtype=f64)
    g_dist = torch.tensor(d_dist.reshape(-1), dtype=f64)
    rgb_p = {}
    for i in np.nonzero(pr.tiles_count > 0)[0]:
        v = pos[i] - campos_t
        rgb_p[int(i)] = torch.clamp(_sh(sph[i], v / v.norm()), min=0.0)
    R_all = {int(i): _rot_rows(quat[i]) for i in np.nonzero(pr.tiles_count > 0)[0]}
    loss = torch.zeros((), dtype=f64)
    for py in range(H):
        for px in range(W):
            pix = py * W + px
            b, e = bn.ranges[(py // 16) * gx + px // 16]
            ids = [int(v) for v in bn.sorted_values[b:e]]
            if not ids:
                continue
            o, d = o_w[pix], d_w[pix]
            al, tt = [], []
            for i in ids:
                R = R_all[i]
                gro = (R @ (o - pos[i])) / scl[i]
                grdu = (R @ d) / scl[i]
                grd = grdu / grdu.norm()
                gray = torch.linalg.cross(grd, gro).pow(2).sum()
                gres = torch.exp(-0.5 * gray)
                alpha = torch.clamp(gres * dns[i], max=0.99)
                t = (scl[i] * grd * (-(grd * gro).sum())).norm()
                ok = bool(gres > 0.0113) and bool(alpha > 1.0 / 255.0) and bool(t > 0)
                al.append(alpha if ok else None)
                tt.append(t)
            # replay of gutKBufferRenderer.cuh:62-112,274-352 on the detached values -> processing order
            order, buf, T = [], [], 1.0
            alive = True
            for j, a in enumerate(al):
                if not alive:
                    break
                if a is None:
                    continue
                if len(buf) == K:
                    buf.sort(key=lambda q: float(tt[q]))
                    j0 = buf.pop(0)
                    order.append(j0)
                    T *= 1 - float(al[j0])
                    if T < 1e-4:
                        alive = False
                buf.append(j)
            buf.sort(key=lambda q: float(tt[q]))
            for j0 in buf:
                if not alive:
                    break
                order.append(j0)
                T *= 1 - float(al[j0])
                if T < 1e-4:
                    alive = False
            Tt = torch.ones((), dtype=f64)
            C, D = torch.zeros(3, dtype=f64), torch.zeros((), dtype=f64)
            for j0 in order:
                w = al[j0] * Tt
                C = C + w * rgb_p[ids[j0]]
                D = D + w * tt[j0]
                Tt = Tt * (1 - al[j0])
            loss = loss + (C * g_rgba[pix, :3]).sum() + (1 - Tt) * g_rgba[pix, 3] + D * g_dist[pix]
    loss.backward()
    from helpers import rel_l2

    assert rel_l2(pos.grad.numpy(), dp[:, 0:3]) < 5e-4
    assert rel_l2(dns.grad.numpy(), dp[:, 3]) < 5e-4
    assert rel_l2(quat.grad.numpy(), dp[:, 4:8]) < 5e-4
    assert rel_l2(scl.grad.numpy(), dp[:, 8:11]) < 5e-4
    assert rel_l2(sph.grad.numpy().reshape(-1, 48), ds) < 5e-4

"""Float64 torch restatement of the 3DGUT forward with Neural Harmonic Texture (NHT) features; autograd gives its adjoint.

It composites over the C oracle's projection and sorted tile lists (oracle.gut_oracle: project / bin_tiles), so the set of (pixel,
particle) pairs it tests is the CUDA path's.  Restated from the reference (not copied):
  threedgut_tracer/include/3dgut/kernels/slang/models/gaussianParticles.slang
    :96-110, :181-190   canonical ray (gro, grd) and hit point P = gro + grd dot(grd, -gro)
    :231                alpha = min(MaxParticleAlpha, response density); bwd_diff differentiates the min
  .../slang/models/neuralHarmonicFeaturesParticle.slang
    :46-66              canonical tetrahedron (inradius 1) and its Cramer terms
    :123-134            barycentric weights, w0 = 1 - w1 - w2 - w3, not clamped
    :152-170            base[n] = sum_k w_k f[k*12 + n]
    :180-189            sincos: out[2n] = sin(base[n]), out[2n+1] = cos(base[n])
    :199-212            integrate out * alpha T when alpha T > 0 (no max(., 0))
Test infrastructure only.
"""
from __future__ import annotations

import math

import numpy as np
import torch

F64 = torch.float64
NHT_DIM, NHT_BASE, NHT_OUT = 48, 12, 24

_S = math.sqrt(24.0)  # tetrahedron edge
TETRA = np.array([[0.5 * _S, -math.sqrt(2.0), -1.0], [-0.5 * _S, -math.sqrt(2.0), -1.0], [0.0, _S * math.sqrt(3.0) / 2 - math.sqrt(2.0), -1.0],
                  [0.0, 0.0, 3.0]])


def barycentric(P: torch.Tensor) -> torch.Tensor:
    """[..., 3] canonical points -> [..., 4] weights (Cramer's rule against vertex 0, as the slang writes it)."""
    v = torch.as_tensor(TETRA, dtype=P.dtype, device=P.device)
    e1, e2, e3 = v[1] - v[0], v[2] - v[0], v[3] - v[0]
    inv_det = 1.0 / torch.dot(e1, torch.linalg.cross(e2, e3))
    d = P - v[0]
    w1 = (d * torch.linalg.cross(e2, e3)).sum(-1) * inv_det
    w2 = (e1 * torch.linalg.cross(d, e3.expand_as(d))).sum(-1) * inv_det
    w3 = (e1 * torch.linalg.cross(e2.expand_as(d), d)).sum(-1) * inv_det
    return torch.stack([1.0 - w1 - w2 - w3, w1, w2, w3], -1)


def features_at(P: torch.Tensor, f: torch.Tensor) -> torch.Tensor:
    """Ray features of a particle with feature row f [48] (or [..., 48]) hit at canonical point(s) P [..., 3]: [..., 24]."""
    w = barycentric(P)
    base = (w[..., :, None] * f.reshape(*f.shape[:-1], 4, NHT_BASE)).sum(-2)
    return torch.stack([torch.sin(base), torch.cos(base)], -1).reshape(*base.shape[:-1], NHT_OUT)


def rot_rows(q):
    """[..., 4] quaternions (wxyz) -> [..., 3, 3] rotation rows."""
    r, x, y, z = q.unbind(-1)
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y)], -1),
        torch.stack([2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x)], -1),
        torch.stack([2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def _pairs(cfg, o, d, pos, R, scl, dns):
    """Exact test of (ray, particle) pairs, broadcast over the leading dimensions: o, d, pos, scl [..., 3], R [..., 3, 3], dns [...].
    Returns (canonical origin gro, direction grd, pd = -grd . gro, alpha (clamped at max_alpha), hit distance t, accepted, clamped:
    response x density above max_alpha)."""
    gro = ((o - pos)[..., None, :] * R).sum(-1) / scl
    grdu = (d[..., None, :] * R).sum(-1) / scl
    grd = grdu / grdu.norm(dim=-1, keepdim=True)
    gray = torch.linalg.cross(grd, gro).pow(2).sum(-1)
    gres = torch.exp(-0.0555555555556 * gray * gray) if int(cfg.kernel_degree) == 4 else torch.exp(-0.5 * gray)
    raw = gres * dns
    alpha = torch.clamp(raw, max=float(cfg.max_alpha))
    pd = -(grd * gro).sum(-1, keepdim=True)
    t = (scl * grd * pd).norm(dim=-1)
    acc = (gres > float(cfg.min_kernel_density)) & (alpha > float(cfg.min_alpha)) & (t > 0)
    return gro, grd, pd, alpha, t, acc, raw > float(cfg.max_alpha)


def tile_pixels(tile, width, height):
    """Flat indices of the pixels of 16x16 tile `tile` (row-major tiles, partial on the right and bottom edges)."""
    gx = (width + 15) // 16
    tx, ty = tile % gx, tile // gx
    ys, xs = np.meshgrid(np.arange(ty * 16, min(height, ty * 16 + 16)), np.arange(tx * 16, min(width, tx * 16 + 16)), indexing="ij")
    return (ys * width + xs).reshape(-1)


def accepted_pairs(cfg, o, d, pos, quat, scl, dns, entries, max_pairs=1 << 18):
    """Without gradients: which entries of one tile's list each pixel composites.  o, d [m,3] world rays; entries [L] particle indices in
    list order.  The walk of every pixel accepts a pair when response > min_kernel_density, alpha > min_alpha and t > 0, and stops
    once its transmittance is below min_transmittance.  Entries are tested in chunks of at most max_pairs (pixel, entry) pairs; the
    transmittance carries from chunk to chunk.  Returns ([m, K] list positions of the composited entries, front to back, padded with
    0; [m, K] validity), K = the largest count of the tile."""
    m, L = o.shape[0], entries.shape[0]
    dev = o.device
    chunk = max(1, max_pairs // max(m, 1))
    T = torch.ones(m, dtype=o.dtype, device=dev)
    taken = []
    with torch.no_grad():
        for c in range(0, L, chunk):
            i = entries[c:c + chunk]
            _, _, _, alpha, _, acc, _ = _pairs(cfg, o[:, None], d[:, None], pos[i], rot_rows(quat[i]), scl[i], dns[i])
            cp = torch.cumprod(torch.where(acc, 1 - alpha, torch.ones_like(alpha)), 1)
            T_before = T[:, None] * torch.cat([torch.ones_like(cp[:, :1]), cp[:, :-1]], 1)
            taken.append(acc & (T_before >= float(cfg.min_transmittance)))
            T = T * cp[:, -1]
        taken = torch.cat(taken, 1) if taken else torch.zeros((m, 0), dtype=torch.bool, device=dev)
        K = int(taken.sum(1).max()) if L else 0
        order = torch.sort(torch.where(taken, torch.arange(L, device=dev), torch.full_like(taken, L, dtype=torch.long)), 1).values[:, :K]
    valid = order < L
    return torch.where(valid, order, torch.zeros_like(order)), valid


def render_tile(cfg, o_w, d_w, width, height, pos, dns, quat, scl, feats, sorted_values, ranges, tile):
    """One tile: (pixel indices [m], features + opacity [m,25], dist [m], hits [m], longest composited list K, number of composited
    pairs whose alpha is clamped at max_alpha).  Autograd runs over
    the gathered composited pairs only, with the transmittance in front of each from a cumprod."""
    dev = pos.device
    pix = torch.as_tensor(tile_pixels(tile, width, height), device=dev)
    o, d = o_w[pix], d_w[pix]
    b, e = (int(v) for v in ranges[tile])
    entries = torch.as_tensor(np.asarray(sorted_values[b:e], np.int64), device=dev)
    k, valid = accepted_pairs(cfg, o, d, pos, quat, scl, dns, entries)
    i = entries[k]
    gro, grd, pd, alpha, t, _, clamped = _pairs(cfg, o[:, None], d[:, None], pos[i], rot_rows(quat[i]), scl[i], dns[i])
    alpha = torch.where(valid, alpha, torch.zeros_like(alpha))
    cp = torch.cumprod(1 - alpha, 1)
    w = alpha * torch.cat([torch.ones_like(cp[:, :1]), cp[:, :-1]], 1)
    Fe = (w[..., None] * features_at(gro + grd * pd, feats[i])).sum(1)
    T = cp[:, -1] if cp.shape[1] else torch.ones(len(pix), dtype=pos.dtype, device=dev)
    D = (w * t).sum(1)
    H = (valid & (w > 0)).sum(1).to(pos.dtype)
    return pix, torch.cat([Fe, (1 - T)[:, None]], 1), D, H, k.shape[1], int((clamped & valid).sum())


def world_rays(cam_inv, ro, rd, dtype, device):
    inv = torch.as_tensor(np.asarray(cam_inv), dtype=dtype, device=device)
    o_w = torch.as_tensor(np.asarray(ro).reshape(-1, 3), dtype=dtype, device=device) @ inv[:3] + inv[3]
    d_w = torch.as_tensor(np.asarray(rd).reshape(-1, 3), dtype=dtype, device=device) @ inv[:3]
    return o_w, d_w


def render(cfg, cam_inv, width, height, ro, rd, pos, dns, quat, scl, feats, sorted_values, ranges, tiles=None):
    """Composite NHT features over the sorted tile lists.  cam_inv: the [4,3] sensor->world columns of gut_oracle.sensor_matrices;
    ro / rd [H*W,3] sensor-space rays; pos [N,3], dns [N], quat [N,4] (wxyz), scl [N,3], feats [N,48] (tensors of one floating
    dtype -- float64 for the oracle, float32 for its yardstick -- optionally requiring grad).  tiles: the tile indices to render
    (default all); other pixels stay zero.  Returns (features + opacity [H,W,25], dist [H,W,1], hits [H,W,1]) in that dtype."""
    dt, dev = pos.dtype, pos.device
    o_w, d_w = world_rays(cam_inv, ro, rd, dt, dev)
    tiles = range(ranges.shape[0]) if tiles is None else tiles
    out = [render_tile(cfg, o_w, d_w, width, height, pos, dns, quat, scl, feats, sorted_values, ranges, int(t)) for t in tiles]
    P = width * height
    pix = torch.cat([r[0] for r in out]) if out else torch.zeros(0, dtype=torch.long, device=dev)
    cat = lambda j, shape: torch.cat([r[j] for r in out]) if out else torch.zeros(shape, dtype=dt, device=dev)  # noqa: E731
    img = torch.zeros((P, NHT_OUT + 1), dtype=dt, device=dev).index_put((pix,), cat(1, (0, NHT_OUT + 1)))
    dist = torch.zeros(P, dtype=dt, device=dev).index_put((pix,), cat(2, (0,)))
    hits = torch.zeros(P, dtype=dt, device=dev).index_put((pix,), cat(3, (0,)))
    return img.reshape(height, width, NHT_OUT + 1), dist.reshape(height, width, 1), hits.reshape(height, width, 1)


def leaves(particles: np.ndarray, feats: np.ndarray, device="cpu", requires_grad=True, dtype=F64):
    """Leaf tensors (pos, dns, quat, scl, feats) of a [N,12] particle record and [N,48] features, in `dtype`."""
    p = torch.as_tensor(np.asarray(particles, np.float32), device=device).to(dtype)
    ts = [p[:, 0:3], p[:, 3], p[:, 4:8], p[:, 8:11], torch.as_tensor(np.asarray(feats, np.float32), device=device).to(dtype)]
    return [t.clone().requires_grad_(requires_grad) for t in ts]


def frame(cfg, cam, sc_particles, feats, ro, rd, go, d_out=None, d_dist=None, device="cpu", tiles=None, dtype=F64, pr=None, bn=None):
    """Forward (and with d_out / d_dist, the backward by autograd) of one frame over the C oracle's lists (or the given pr / bn).
    tiles: the tiles to render (default all); with gradients, those outside them must be zero there to mean the full frame's backward.
    The backward runs tile by tile, so the autograd graph of one tile is alive at a time.  Returns a dict of numpy arrays (float64):
    out, dist, hits, longest (the longest composited list of a pixel), clamped (composited pairs with alpha clamped) and, with gradients, dp [N,12] (pos, density,
    quat, scale, 0) and df [N,48]."""
    n = sc_particles.shape[0]
    if pr is None:
        pr = go.project(cfg, cam, sc_particles, np.zeros((n, 48), np.float32), 0)
        bn = go.bin_tiles(cfg, cam, pr)
    _, inv, _ = go.sensor_matrices(cam)
    W, H = cam.width, cam.height
    grads = d_out is not None
    lv = leaves(sc_particles, feats, device, requires_grad=grads, dtype=dtype)
    o_w, d_w = world_rays(inv, ro, rd, dtype, device)
    if grads:
        g_out = torch.as_tensor(np.asarray(d_out).reshape(W * H, NHT_OUT + 1), dtype=dtype, device=device)
        g_dist = torch.as_tensor(np.asarray(d_dist).reshape(W * H), dtype=dtype, device=device)
        acc = [torch.zeros_like(t) for t in lv]
    img = np.zeros((W * H, NHT_OUT + 1))
    dist, hits = np.zeros(W * H), np.zeros(W * H)
    longest = clamped = 0
    for t in (range(bn.ranges.shape[0]) if tiles is None else tiles):
        pix, o, dd, hh, K, nc = render_tile(cfg, o_w, d_w, W, H, *lv, bn.sorted_values, bn.ranges, int(t))
        longest, clamped = max(longest, K), clamped + nc
        p = pix.cpu().numpy()
        img[p], dist[p], hits[p] = o.detach().cpu().double().numpy(), dd.detach().cpu().double().numpy(), hh.cpu().double().numpy()
        if grads and o.requires_grad:
            loss = (o * g_out[pix]).sum() + (dd * g_dist[pix]).sum()
            for a, g in zip(acc, torch.autograd.grad(loss, lv, allow_unused=True)):
                if g is not None:
                    a += g
    res = dict(out=img.reshape(H, W, NHT_OUT + 1), dist=dist.reshape(H, W, 1), hits=hits.reshape(H, W, 1), longest=longest, clamped=clamped,
               pr=pr, bn=bn)
    if grads:
        gp, gd, gq, gs, gf = (a.detach().cpu().double() for a in acc)
        dp = torch.cat([gp, gd[:, None], gq, gs, torch.zeros((n, 1), dtype=torch.float64)], 1)
        res.update(dp=dp.numpy(), df=gf.numpy())
    return res

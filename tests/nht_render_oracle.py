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
    r, x, y, z = q[0], q[1], q[2], q[3]
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y)]),
        torch.stack([2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x)]),
        torch.stack([2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y)])])


def render(cfg, cam_inv, width, height, ro, rd, pos, dns, quat, scl, feats, sorted_values, ranges):
    """Composite NHT features over the sorted tile lists.  cam_inv: the [4,3] sensor->world columns of gut_oracle.sensor_matrices;
    ro / rd [H*W,3] sensor-space rays; pos [N,3], dns [N], quat [N,4] (wxyz), scl [N,3], feats [N,48] (float64 tensors, optionally
    requiring grad).  Returns (features + opacity [H,W,25], dist [H,W,1], hits [H,W,1]) as float64 tensors."""
    dev = pos.device
    inv = torch.as_tensor(np.asarray(cam_inv), dtype=F64, device=dev)
    o_w = torch.as_tensor(np.asarray(ro).reshape(-1, 3), dtype=F64, device=dev) @ inv[:3] + inv[3]
    d_w = torch.as_tensor(np.asarray(rd).reshape(-1, 3), dtype=F64, device=dev) @ inv[:3]
    deg4 = int(cfg.kernel_degree) == 4
    gx = (width + 15) // 16
    P = width * height
    out = [None] * ranges.shape[0]
    for tile in range(ranges.shape[0]):
        b, e = (int(v) for v in ranges[tile])
        tx, ty = tile % gx, tile // gx
        ys, xs = np.meshgrid(np.arange(ty * 16, min(height, ty * 16 + 16)), np.arange(tx * 16, min(width, tx * 16 + 16)), indexing="ij")
        pix = torch.as_tensor((ys * width + xs).reshape(-1), device=dev)
        o, d = o_w[pix], d_w[pix]
        m = len(pix)
        T = torch.ones(m, dtype=F64, device=dev)
        alive = torch.ones(m, dtype=torch.bool, device=dev)
        Fe = torch.zeros((m, NHT_OUT), dtype=F64, device=dev)
        D = torch.zeros(m, dtype=F64, device=dev)
        H = torch.zeros(m, dtype=F64, device=dev)
        for k in range(b, e):
            i = int(sorted_values[k])
            R = rot_rows(quat[i])
            gro = ((o - pos[i]) @ R.T) / scl[i]
            grdu = (d @ R.T) / scl[i]
            grd = grdu / grdu.norm(dim=1, keepdim=True)
            gray = torch.linalg.cross(grd, gro).pow(2).sum(1)
            gres = torch.exp(-0.0555555555556 * gray * gray) if deg4 else torch.exp(-0.5 * gray)
            alpha = torch.clamp(gres * dns[i], max=float(cfg.max_alpha))
            pd = -(grd * gro).sum(1, keepdim=True)
            t = (scl[i] * grd * pd).norm(dim=1)
            acc = alive & (gres > float(cfg.min_kernel_density)) & (alpha > float(cfg.min_alpha)) & (t > 0)
            if not bool(acc.any()):
                continue
            w = torch.where(acc, alpha * T, torch.zeros_like(T))
            Fe = Fe + w[:, None] * features_at(gro + grd * pd, feats[i])
            D = D + w * t
            H = H + (acc & (w > 0)).to(F64)
            T = torch.where(acc, T * (1 - alpha), T)
            alive = alive & ~(T < float(cfg.min_transmittance))
        out[tile] = (pix, torch.cat([Fe, (1 - T)[:, None]], 1), D, H)
    img = torch.zeros((P, NHT_OUT + 1), dtype=F64, device=dev)
    dist = torch.zeros(P, dtype=F64, device=dev)
    hits = torch.zeros(P, dtype=F64, device=dev)
    pix = torch.cat([t[0] for t in out])
    img = img.index_put((pix,), torch.cat([t[1] for t in out]))
    dist = dist.index_put((pix,), torch.cat([t[2] for t in out]))
    hits = hits.index_put((pix,), torch.cat([t[3] for t in out]))
    return img.reshape(height, width, NHT_OUT + 1), dist.reshape(height, width, 1), hits.reshape(height, width, 1)


def leaves(particles: np.ndarray, feats: np.ndarray, device="cpu", requires_grad=True):
    """float64 leaf tensors (pos, dns, quat, scl, feats) of a [N,12] particle record and [N,48] features."""
    p = torch.as_tensor(np.asarray(particles, np.float32), device=device).to(F64)
    ts = [p[:, 0:3], p[:, 3], p[:, 4:8], p[:, 8:11], torch.as_tensor(np.asarray(feats, np.float32), device=device).to(F64)]
    return [t.clone().requires_grad_(requires_grad) for t in ts]


def frame(cfg, cam, sc_particles, feats, ro, rd, go, d_out=None, d_dist=None, device="cpu"):
    """Forward (and with d_out / d_dist, the backward by autograd) of one frame over the C oracle's lists.  Returns a dict of numpy
    arrays: out, dist, hits and, with gradients, dp [N,12] (pos, density, quat, scale, 0) and df [N,48]."""
    n = sc_particles.shape[0]
    pr = go.project(cfg, cam, sc_particles, np.zeros((n, 48), np.float32), 0)
    bn = go.bin_tiles(cfg, cam, pr)
    _, inv, _ = go.sensor_matrices(cam)
    pos, dns, quat, scl, ft = leaves(sc_particles, feats, device, requires_grad=d_out is not None)
    img, dist, hits = render(cfg, inv, cam.width, cam.height, ro, rd, pos, dns, quat, scl, ft, bn.sorted_values, bn.ranges)
    res = dict(out=img.detach().cpu().numpy(), dist=dist.detach().cpu().numpy(), hits=hits.detach().cpu().numpy(), pr=pr, bn=bn)
    if d_out is not None:
        loss = (img * torch.as_tensor(d_out, dtype=F64, device=device)).sum() + (dist * torch.as_tensor(d_dist, dtype=F64, device=device)).sum()
        gp, gd, gq, gs, gf = torch.autograd.grad(loss, [pos, dns, quat, scl, ft], allow_unused=True)
        z = lambda g, shape: torch.zeros(shape, dtype=F64, device=device) if g is None else g  # noqa: E731
        dp = torch.cat([z(gp, (n, 3)), z(gd, (n,))[:, None], z(gq, (n, 4)), z(gs, (n, 3)), torch.zeros((n, 1), dtype=F64, device=device)], 1)
        res.update(dp=dp.cpu().numpy(), df=z(gf, (n, 48)).cpu().numpy())
    return res

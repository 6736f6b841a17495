"""Float64 restatement of the ray normals of the 3DGRT forward (render.enable_normals with SH radiance).  TEST INFRASTRUCTURE ONLY.

It sums over the hit lists of the brute-force C oracle (grt_nht_oracle.trace_lists: per ray, the candidates that grt_oracle_trace /
grt_ico_oracle_trace process, in order), so the accepted hits, their order and the transmittance before each are the oracle's, for
both primitives.  Restated from the reference (not copied):
  threedgrt_tracer/src/kernels/cuda/referenceOptix.cu:103-186                   processHit(..., &rayNormal) on every processed hit
  threedgrt_tracer/include/3dgrt/kernels/cuda/gaussianParticles.cuh:337-404    processHit: for an accepted hit, weight = alpha T and
      normal += weight * safe_normalize((gro + grd (dot(grd, -gro) - sqrt(9 - grayDist))) * (particleRotation * particleScale))
  threedgrt_tracer/include/3dgrt/kernels/cuda/gaussianParticles.cuh:179-192    fetchParticleDensity: the float33 of quaternionWXYZToMatrix
  threedgrt_tracer/include/3dgrt/mathUtils.h:390-393, 450-455                   safe_normalize; operator*(float33, float3) = sum_i p_i m[i]
The normals have no backward in the reference (referenceBwdOptix.cu never reads them), so there is none here either.
"""
from __future__ import annotations

import numpy as np
import torch

import grt_nht_oracle as gno

F64 = torch.float64
ELLIPSOID_SQ_RADIUS = 9.0


def hit_normals(o, d, pos, quat, scl):
    """The unit (safe-normalised) normal of each hit: o / d [M,3] world rays, pos [M,3], quat [M,4] wxyz (as stored, not normalised),
    scl [M,3]; float64 tensors.  A hit with 9 - grayDist < 0 gives NaN, as the reference's sqrtf does."""
    Rm = gno._rot_rows(quat)                                   # m[0..2]: rows of quaternionWXYZToMatrix
    gro = torch.einsum("mab,mb->ma", Rm, o - pos) / scl        # (gposc * particleRotation) / scale
    grdu = torch.einsum("mab,mb->ma", Rm, d) / scl
    grd = grdu / grdu.norm(dim=1, keepdim=True)
    gray = torch.linalg.cross(grd, gro).pow(2).sum(1, keepdim=True)
    rs = torch.einsum("mab,ma->mb", Rm, scl)                   # particleRotation * particleScale = sum_i s_i m[i]
    t = -(grd * gro).sum(1, keepdim=True) - torch.sqrt(ELLIPSOID_SQ_RADIUS - gray)
    v = (gro + grd * t) * rs
    l2 = v.pow(2).sum(1, keepdim=True)
    return torch.where(l2 > 0, v / torch.sqrt(torch.where(l2 > 0, l2, torch.ones_like(l2))), v)


def normals(lists, o, d, particles):
    """The unnormalised normal sum of every ray [R,3] (float64) over the oracle's lists.  o / d [R,3] float64 world rays; particles the
    [N,12] record.  Only the oracle's accept decisions (alpha > 0 in the lists) are kept; alpha, weights and normals are recomputed."""
    p = torch.as_tensor(np.asarray(particles, np.float32)).to(F64)
    pos, dns, quat, scl = p[:, 0:3], p[:, 3], p[:, 4:8], p[:, 8:11]
    R = o.shape[0]
    count = torch.as_tensor(lists["count"]).long()
    pid_all = torch.as_tensor(lists["pid"]).long()
    alpha_all = torch.as_tensor(lists["alpha"])
    N = torch.zeros((R, 3), dtype=F64)
    T = torch.ones(R, dtype=F64)
    for s in range(pid_all.shape[1]):
        on = (count > s) & (alpha_all[:, s] > 0)
        if not bool(on.any()):
            continue
        idx = torch.nonzero(on).squeeze(1)
        pp = pid_all[idx, s]
        alpha = alpha_all[idx, s]                              # the oracle's float64 alpha of this hit
        w = alpha * T[idx]
        N = N.index_add(0, idx, w[:, None] * hit_normals(o[idx], d[idx], pos[pp], quat[pp], scl[pp]))
        T = T.index_put((idx,), T[idx] * (1 - alpha))
    return N


def frame(cfg, particles, rays_o, rays_d, ray_to_world, primitive="instances", clamping=True, lists_f64=True):
    """Normals [R,3] (numpy float64) of one frame, with the lists the sum ran over."""
    lists = gno.trace_lists(cfg, particles, rays_o, rays_d, ray_to_world, clamping=clamping, f64=lists_f64, primitive=primitive)
    o, d = gno.world_rays(rays_o, rays_d, ray_to_world)
    return normals(lists, o, d, particles).numpy(), lists

"""Float64 torch restatement of the 3DGRT forward with Neural Harmonic Texture (NHT) features; autograd gives its adjoint.
TEST INFRASTRUCTURE ONLY.

It composites over the hit lists of the brute-force C oracle (tests/host_emul/grt_trace_lists.c: per ray, the candidates that
grt_oracle_trace / grt_ico_oracle_trace process, in order, and `last`), so the set and order of (ray, particle) hits is the oracle's,
for both primitives.  Restated from the reference (not copied):
  threedgrt_tracer/src/kernels/cuda/referenceSlangOptix.cu:103-200      ordered integration, hit count / visibility where weight > 0
  threedgrt_tracer/include/3dgrt/kernels/slang/models/gaussianParticles.slang
    hit() / canonicalRayIntersection()   alpha = min(max_alpha, response density), P = gro + grd dot(grd, -gro), depth |scale (P - gro)|
  .../slang/models/neuralHarmonicFeaturesParticle.slang                  features (tests/nht_render_oracle.features_at)
Backward rule of referenceSlangBwdOptix.cu:141-229: the re-trace ends strictly before `last`, so the hits at the ray's last processed
distance get no gradient of their own; they still count in the outputs.  composite() reproduces that by reading those hits' parameters
from a frozen copy (by default the detached live parameters), so autograd gives the reference's adjoint.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import torch

from nht_render_oracle import NHT_OUT, features_at

F64 = torch.float64
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SRC = os.path.join(HERE, "host_emul", "grt_trace_lists.c")
DEPS = [SRC, os.path.join(HERE, "host_emul", "grt_icosahedron_oracle.c"), os.path.join(ROOT, "oracle", "gut_oracle.c"),
        os.path.join(ROOT, "oracle", "gut_oracle.h")]
_LIBS = {}


def _build(f64: bool) -> str:
    """Compiled on first use into a per-user temporary directory (the tree may be read-only), with oracle/Makefile's flags."""
    h = hashlib.sha256()
    for p in DEPS:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(b"f64" if f64 else b"f32")
    out_dir = os.path.join(tempfile.gettempdir(), f"grt_lists_oracle_{os.getuid()}")
    os.makedirs(out_dir, exist_ok=True)
    so = os.path.join(out_dir, f"libgrt_lists_oracle_{h.hexdigest()[:16]}.so")
    if not os.path.exists(so):
        cc = os.environ.get("CC", "gcc")
        flags = ["-O2", "-fPIC", "-fopenmp", "-ffp-contract=off", "-fno-fast-math", "-w"]
        if os.path.isdir("/usr/lib/gcc/x86_64-linux-gnu/13"):
            flags.insert(0, "-B/usr/lib/gcc/x86_64-linux-gnu/13")
        if f64:
            flags.append("-DORACLE_F64")
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.check_call([cc, *flags, "-shared", "-o", tmp, SRC, "-lm"])
        os.replace(tmp, so)
    return so


def lib(f64: bool = False):
    if f64 not in _LIBS:
        _LIBS[f64] = C.CDLL(_build(f64))
    return _LIBS[f64]


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def trace_lists(cfg, particles, rays_o, rays_d, ray_to_world, clamping=True, f64=False, primitive="instances", cap=64):
    """The oracle's processed candidates per ray: dict of count [R], pid / key / alpha / depth [R,L] (L = the longest list; alpha is 0
    for a rejected candidate) and last [R]."""
    if primitive not in ("instances", "icosahedron"):
        raise ValueError(f"unknown primitive {primitive!r}")
    particles = _f32(particles)
    ro, rd = _f32(rays_o).reshape(-1, 3), _f32(rays_d).reshape(-1, 3)
    r2w = _f32(np.asarray(ray_to_world)[:3, :4])
    n, r = particles.shape[0], ro.shape[0]
    fn = lib(f64).grt_ico_oracle_trace_lists if primitive == "icosahedron" else lib(f64).grt_oracle_trace_lists
    while True:
        count, last = np.zeros(r, np.int32), np.zeros(r, np.float32)
        pid, key = np.zeros((r, cap), np.int32), np.zeros((r, cap), np.float32)
        alpha, depth = np.zeros((r, cap), np.float64), np.zeros((r, cap), np.float64)
        fn(C.byref(cfg), C.c_int32(int(clamping)), C.c_int64(n), _p(particles, C.c_float), C.c_int64(r), _p(ro, C.c_float), _p(rd, C.c_float),
           _p(r2w, C.c_float), C.c_int32(cap), _p(count, C.c_int32), _p(pid, C.c_int32), _p(key, C.c_float), _p(alpha, C.c_double),
           _p(depth, C.c_double), _p(last, C.c_float))
        if r == 0 or count.max() <= cap:
            break
        cap = int(count.max())
    L = int(count.max()) if r else 0
    return dict(count=count, pid=pid[:, :L], key=key[:, :L], alpha=alpha[:, :L], depth=depth[:, :L], last=last)


def _rot_rows(q):
    """[M,4] wxyz (not normalised, as the kernels read them) -> [M,3,3] rows of the inverse rotation (canonical = rows @ (x - mu))."""
    r, x, y, z = q.unbind(-1)
    return torch.stack([
        torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y)], -1),
        torch.stack([2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x)], -1),
        torch.stack([2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def world_rays(rays_o, rays_d, ray_to_world, device="cpu"):
    """rayWorldOrigin / rayWorldDirection in float64 from the float32 inputs: [R,3] each."""
    m = torch.as_tensor(np.asarray(ray_to_world, np.float64)[:3, :4], device=device)
    ro = torch.as_tensor(_f32(rays_o).reshape(-1, 3), device=device).to(F64)
    rd = torch.as_tensor(_f32(rays_d).reshape(-1, 3), device=device).to(F64)
    return ro @ m[:, :3].T + m[:, 3], rd @ m[:, :3].T


def composite(cfg, lists, o, d, params, frozen=None):
    """NHT forward over the oracle's lists.  o / d [R,3] float64 world rays; params = (pos [N,3], dns [N,1], quat [N,4], scl [N,3],
    feats [N,48]) float64 tensors; frozen: the same tuple read for each ray's hits at its `last` distance (default: params detached).
    The oracle's accept decisions (alpha > 0 in the lists) are kept; alpha, depth and features are recomputed in float64.
    Returns (features [R,24], alpha [R], dist [R], hits [R])."""
    if frozen is None:
        frozen = tuple(t.detach() for t in params)
    dev = o.device
    R = o.shape[0]
    deg4 = int(cfg.kernel_degree) == 4
    count = torch.as_tensor(lists["count"], device=dev).long()
    pid_all = torch.as_tensor(lists["pid"], device=dev).long()
    key = torch.as_tensor(lists["key"], device=dev)
    acc_all = torch.as_tensor(lists["alpha"], device=dev) > 0
    last = torch.as_tensor(lists["last"], device=dev)
    F = torch.zeros((R, NHT_OUT), dtype=F64, device=dev)
    T = torch.ones(R, dtype=F64, device=dev)
    D = torch.zeros(R, dtype=F64, device=dev)
    H = torch.zeros(R, dtype=F64, device=dev)
    for s in range(pid_all.shape[1]):
        on = (count > s) & acc_all[:, s]
        if not bool(on.any()):
            continue
        idx = torch.nonzero(on).squeeze(1)
        p = pid_all[idx, s]
        at_last = (key[idx, s] == last[idx])[:, None]
        pos, dns, quat, scl, ft = (torch.where(at_last, fz[p].reshape(len(p), -1), lv[p].reshape(len(p), -1))
                                   for lv, fz in zip(params, frozen))
        dns = dns[:, 0]
        Rm = _rot_rows(quat)
        gro = torch.einsum("mab,mb->ma", Rm, o[idx] - pos) / scl
        grdu = torch.einsum("mab,mb->ma", Rm, d[idx]) / scl
        grd = grdu / grdu.norm(dim=1, keepdim=True)
        gray = torch.linalg.cross(grd, gro).pow(2).sum(1)
        gres = torch.exp(-0.0555555555556 * gray * gray) if deg4 else torch.exp(-0.5 * gray)
        alpha = torch.clamp(gres * dns, max=float(cfg.max_alpha))
        pd = -(grd * gro).sum(1, keepdim=True)
        t = (scl * grd * pd).norm(dim=1)
        Ti = T[idx]
        w = alpha * Ti
        F = F.index_add(0, idx, w[:, None] * features_at(gro + grd * pd, ft))
        D = D.index_add(0, idx, w * t)
        H = H.index_add(0, idx, (w > 0).to(F64))
        T = T.index_put((idx,), Ti * (1 - alpha))
    return F, 1 - T, D, H


def leaves(particles, feats, device="cpu", requires_grad=True):
    """float64 leaf tensors (pos [N,3], dns [N,1], quat [N,4], scl [N,3], feats [N,48]) of a [N,12] record and [N,48] features."""
    p = torch.as_tensor(np.asarray(particles, np.float32), device=device).to(F64)
    ts = [p[:, 0:3], p[:, 3:4], p[:, 4:8], p[:, 8:11], torch.as_tensor(np.asarray(feats, np.float32), device=device).to(F64)]
    return tuple(t.clone().requires_grad_(requires_grad) for t in ts)


def frame(cfg, particles, feats, rays_o, rays_d, ray_to_world, d_feat=None, d_alpha=None, d_dist=None, primitive="instances",
          clamping=True, device="cpu", lists_f64=True):
    """Forward (and with the output gradients, the backward by autograd) of one frame.  Returns numpy arrays: feat [R,24], alpha [R],
    dist [R,2] (integrated distance, last), hits [R], lists and, with gradients, dp [N,12] (pos, density, quat, scale, 0), df [N,48].
    lists_f64=False composites over the lists of the fp32 oracle instead (accept decisions in fp32): the other half of a yardstick."""
    n = np.asarray(particles).shape[0]
    lists = trace_lists(cfg, particles, rays_o, rays_d, ray_to_world, clamping=clamping, f64=lists_f64, primitive=primitive)
    o, d = world_rays(rays_o, rays_d, ray_to_world, device)
    params = leaves(particles, feats, device, requires_grad=d_feat is not None)
    F, A, D, H = composite(cfg, lists, o, d, params)
    res = dict(feat=F.detach().cpu().numpy(), alpha=A.detach().cpu().numpy(),
               dist=np.stack([D.detach().cpu().numpy(), lists["last"].astype(np.float64)], -1), hits=H.detach().cpu().numpy(), lists=lists)
    if d_feat is not None:
        t = lambda a: torch.as_tensor(np.asarray(a, np.float64), device=device).reshape(-1, *np.asarray(a).shape[-1:])  # noqa: E731
        loss = (F * t(d_feat).reshape(F.shape)).sum() + (A * t(d_alpha).reshape(A.shape)).sum() + (D * t(d_dist).reshape(D.shape)).sum()
        g = torch.autograd.grad(loss, params, allow_unused=True) if loss.requires_grad else [None] * len(params)
        z = [torch.zeros_like(p) if gi is None else gi for gi, p in zip(g, params)]
        dp = torch.cat([z[0], z[1], z[2], z[3], torch.zeros((n, 1), dtype=F64, device=device)], 1)
        res.update(dp=dp.cpu().numpy(), df=z[4].cpu().numpy())
    return res

"""CPU checks of the 3DGRT icosahedron proxies (`primitive_type: icosahedron`): the reference's vertex / face table, the
GPU's 10-slab shortcut against the oracle's world-space triangles, the inside-the-proxy rule, the oracle's adjoint against
fp64 autograd in the icosahedron's hit order, and the scene box."""
import os
import re

import numpy as np
import pytest

import grt_ico_oracle as gio
import scenes
from helpers import rel_l2
from oracle import gut_oracle as go

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHI = (1.0 + 5.0 ** 0.5) / 2.0


def gpu_slab_normals():
    """kIcoSlab of csrc/grt.cu (n_k * sqrt(3), one of each antipodal pair) as unit vectors."""
    src = open(os.path.join(ROOT, "3dgrut_b200", "csrc", "grt.cu")).read()
    body = re.search(r"kIcoSlab\[10\]\[3\]\s*=\s*\{(.*?)\};", src, re.S).group(1)
    body = body.replace("kInvPhi", repr(1.0 / PHI)).replace("kPhi", repr(PHI))
    body = re.sub(r"(?<=[\d.])f\b", "", body).replace("{", "[").replace("}", "]")
    n = np.array(eval("[" + body + "]"), np.float64)  # noqa: S307 (a literal table of our own source)
    assert n.shape == (10, 3)
    return n / np.linalg.norm(n, axis=1, keepdims=True)


def _canonical_table():
    v, tri = gio.table()
    return v.astype(np.float64) * gio.ICO_VRT_SCALE, tri


def test_table_geometry_and_gpu_normals():
    v, tri = _canonical_table()
    assert v.shape == (12, 3) and tri.shape == (20, 3)
    assert sorted(np.unique(tri).tolist()) == list(range(12))
    a, b, c = v[tri[:, 0]], v[tri[:, 1]], v[tri[:, 2]]
    nrm = np.cross(b - a, c - a)
    centroid = (a + b + c) / 3.0
    # counter-clockwise seen from outside: the winding normal points away from the centre
    assert np.all(np.einsum("ij,ij->i", nrm, centroid) > 0)
    unit = nrm / np.linalg.norm(nrm, axis=1, keepdims=True)
    dist = np.einsum("ij,ij->i", unit, a)
    assert np.allclose(dist, 1.0, atol=1e-6), dist  # inradius 1 in kernelScale * scale units
    # 10 antipodal pairs ...
    pair = [int(np.argmin(np.linalg.norm(unit + u, axis=1))) for u in unit]
    assert all(np.allclose(unit[pair[i]], -unit[i], atol=1e-6) and pair[pair[i]] == i for i in range(20))
    # ... equal, up to sign, to the directions the GPU code hard-codes
    g = gpu_slab_normals()
    for u in unit:
        assert np.min(np.minimum(np.linalg.norm(g - u, axis=1), np.linalg.norm(g + u, axis=1))) < 1e-6
    for u in g:
        assert np.min(np.linalg.norm(unit - u, axis=1)) < 1e-6 and np.min(np.linalg.norm(unit + u, axis=1)) < 1e-6


def _instance_rays(particles, kscl, o, d):
    """o_i = A^-1 (o - mu), d_i = A^-1 d for every particle (A = R diag(kernelScale * scale)), float64."""
    P = particles.astype(np.float64)
    r, x, y, z = P[:, 4], P[:, 5], P[:, 6], P[:, 7]
    Rt = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y + r * z), 2 * (x * z - r * y)], -1),
                   np.stack([2 * (x * y - r * z), 1 - 2 * (x * x + z * z), 2 * (y * z + r * x)], -1),
                   np.stack([2 * (x * z + r * y), 2 * (y * z - r * x), 1 - 2 * (x * x + y * y)], -1)], 1)  # [N,3,3]
    oi = np.einsum("nij,rnj->rni", Rt, o[:, None, :] - P[None, :, 0:3]) / kscl[None]
    di = np.einsum("nij,rj->rni", Rt, d) / kscl[None]
    return oi, di


def slab_entry(oi, di, tmin=0.0):
    """numpy restatement of the GPU test: entry = max of the 10 slab entries, exit = min of the exits, candidate when
    entry <= exit and entry > tmin; +inf otherwise."""
    n = gpu_slab_normals()
    s, sd = oi @ n.T, di @ n.T
    with np.errstate(divide="ignore", invalid="ignore"):
        q0, q1 = (-1.0 - s) / sd, (1.0 - s) / sd
    tin = np.nanmax(np.minimum(q0, q1), -1)
    tout = np.nanmin(np.maximum(q0, q1), -1)
    return np.where((tin <= tout) & (tin > tmin), tin, np.inf)


def _edge_distance(p):
    """distance of canonical points [..., 3] from the nearest edge of the icosahedron"""
    v, tri = _canonical_table()
    edges = {tuple(sorted((int(f[i]), int(f[(i + 1) % 3])))) for f in tri for i in range(3)}
    assert len(edges) == 30
    best = np.full(p.shape[:-1], np.inf)
    for a, b in edges:
        e = v[b] - v[a]
        u = np.clip(((p - v[a]) @ e) / (e @ e), 0.0, 1.0)
        best = np.minimum(best, np.linalg.norm(p - (v[a] + u[..., None] * e), axis=-1))
    return best


def _world_rays(sc, cam_index):
    c2w = np.asarray(sc.camera(cam_index, 10), np.float64)
    ro, rd = sc.rays()
    o = ro[0].reshape(-1, 3).astype(np.float64) @ c2w[:3, :3].T + c2w[:3, 3]
    d = rd[0].reshape(-1, 3).astype(np.float64) @ c2w[:3, :3].T
    return o.astype(np.float32), d.astype(np.float32)


def test_slab_shortcut_equals_reference_triangles():
    sc = scenes.scene_c1(n=1000, width=40, height=40)
    cfg = go.grt_config()
    o, d = _world_rays(sc, 3)
    kscl, _ = go.grt_proxies(cfg, sc.particles, clamping=False)
    t_tri = gio.entry_t(cfg, sc.particles, o, d, 0.0, clamping=False, f64=True)     # [R,N], oracle: world-space triangles
    oi, di = _instance_rays(sc.particles, kscl.astype(np.float64), o.astype(np.float64), d.astype(np.float64))
    t_slab = slab_entry(oi, di)                                                       # [R,N], the GPU's rule in float64
    hit_tri, hit_slab = np.isfinite(t_tri), np.isfinite(t_slab)
    assert hit_tri.sum() > 5000
    same_set = np.all(hit_tri == hit_slab, axis=1)
    print(f"[ico] candidate pairs {int(hit_tri.sum())}, rays with identical candidate sets {same_set.mean():.5f}")
    assert same_set.mean() >= 0.999
    both = hit_tri & hit_slab
    rel = np.abs(t_tri[both] - t_slab[both]) / np.maximum(np.abs(t_slab[both]), 1e-6)
    print(f"[ico] entry t: max relative difference {rel.max():.2e}")
    assert rel.max() <= 1e-5, rel.max()
    # every disagreement is a ray grazing an edge
    r, i = np.nonzero(hit_tri != hit_slab)
    if r.size:
        t = np.where(hit_tri[r, i], t_tri[r, i], t_slab[r, i]).astype(np.float64)
        p = oi[r, i] + t[:, None] * di[r, i]
        assert _edge_distance(p).max() <= 1e-5


def test_ray_origin_inside_the_proxy_sees_no_particle():
    sc = scenes.scene_c1(n=50, seed=3)
    parts = sc.particles[:1].copy()
    parts[0, 3] = 0.8  # accepted by the hit test wherever the ray passes through the centre
    cfg = go.grt_config()
    kscl, _ = go.grt_proxies(cfg, parts, clamping=False)
    d = np.array([0.3, -0.2, 0.93], np.float32)
    d /= np.linalg.norm(d)
    # 0.3 canonical units behind the centre along the ray: inside both the instance box and the icosahedron, t* > 0 ahead
    o = (parts[0, 0:3] - 0.3 * float(kscl[0].min()) * d).astype(np.float32)
    ro, rd = o.reshape(1, 1, 3), d.reshape(1, 1, 3)
    eye = np.eye(4, dtype=np.float32)
    rgb_i, alpha_i, _, hits_i, vis_i = gio.grt_trace(cfg, parts, sc.sph, 3, ro, rd, eye, clamping=False, primitive="instances")
    rgb_c, alpha_c, _, hits_c, vis_c = gio.grt_trace(cfg, parts, sc.sph, 3, ro, rd, eye, clamping=False, primitive="icosahedron")
    assert float(hits_i.sum()) == 1 and float(vis_i.sum()) == 1 and float(alpha_i.max()) > 0.5
    assert float(hits_c.sum()) == 0 and float(vis_c.sum()) == 0 and float(alpha_c.max()) == 0 and float(np.abs(rgb_c).max()) == 0
    # the same particle seen from outside is a candidate
    o2 = (parts[0, 0:3] - 5.0 * float(kscl[0].max()) * d).astype(np.float32)
    _, _, _, hits_o, _ = gio.grt_trace(cfg, parts, sc.sph, 3, o2.reshape(1, 1, 3), rd, eye, clamping=False, primitive="icosahedron")
    assert float(hits_o.sum()) == 1


@pytest.mark.parametrize("degree", [4, 2])
def test_grt_icosahedron_oracle_backward_equals_autograd(degree):
    """The model and tolerance of test_grt_oracle.test_grt_oracle_backward_equals_autograd with the icosahedron's hit order:
    candidates keyed by the front-face entry t, the paper configs' kernel degree and no density clamping."""
    from test_oracle_autograd import _rot_rows, _sh

    sc = scenes.scene_c1(n=40, seed=5, width=20, height=16)
    cfg = gio.paper_config(degree)
    c2w = np.asarray(sc.camera(2, 7), np.float32)
    ro, rd = sc.rays()
    rgb, alpha, dist, hits, vis = gio.grt_trace(cfg, sc.particles, sc.sph, 3, ro[0], rd[0], c2w, clamping=False, primitive="icosahedron")
    assert hits.max() >= 3
    rng = np.random.default_rng(0)
    d_rgb = rng.normal(size=rgb.shape).astype(np.float32)
    d_alpha = rng.normal(size=alpha.shape).astype(np.float32)
    d_dist = (0.2 * rng.normal(size=alpha.shape)).astype(np.float32)
    dp, ds = gio.grt_trace_bwd(cfg, sc.particles, sc.sph, 3, ro[0], rd[0], c2w, rgb, alpha, dist, d_rgb, d_alpha, d_dist, clamping=False,
                               primitive="icosahedron")

    f64 = torch.float64
    Pt = torch.tensor(sc.particles, dtype=f64)
    pos, dns, quat, scl = (Pt[:, 0:3].clone().requires_grad_(True), Pt[:, 3].clone().requires_grad_(True),
                           Pt[:, 4:8].clone().requires_grad_(True), Pt[:, 8:11].clone().requires_grad_(True))
    sph = torch.tensor(sc.sph, dtype=f64).reshape(-1, 16, 3).clone().requires_grad_(True)
    _, bb = gio.grt_proxies(cfg, sc.particles, clamping=False, primitive="icosahedron")
    R, t = c2w[:3, :3].astype(np.float64), c2w[:3, 3].astype(np.float64)
    ro2, rd2 = ro[0].reshape(-1, 3).astype(np.float64), rd[0].reshape(-1, 3).astype(np.float64)
    wo, wd = (ro2 @ R.T + t).astype(np.float32), (rd2 @ R.T).astype(np.float32)
    last = dist.reshape(-1, 2)[:, 1]
    a_exp = -4.5 / 3.0 ** degree
    loss = torch.zeros((), dtype=f64)
    for k in range(ro2.shape[0]):
        o, d = wo[k].astype(np.float64), wd[k].astype(np.float64)
        with np.errstate(divide="ignore"):
            t0s, t1s = (bb[:3] - o) / d, (bb[3:] - o) / d
        tmin, tmax = max(0.0, np.minimum(t0s, t1s).max()), np.maximum(t0s, t1s).min()
        if not tmin <= tmax:
            continue
        keys = gio.entry_t(cfg, sc.particles, wo[k:k + 1], wd[k:k + 1], max(0.0, tmin - 1e-9), clamping=False)[0]
        order = sorted((float(keys[i]), i) for i in np.nonzero(np.isfinite(keys) & (keys < tmax + 1e-9))[0])
        ot, dt = torch.tensor(o, dtype=f64), torch.tensor(d, dtype=f64)
        T = torch.ones((), dtype=f64)
        C, D = torch.zeros(3, dtype=f64), torch.zeros((), dtype=f64)
        for (ts, i) in order:
            if float(T) <= 1e-3:
                break
            Rr = _rot_rows(quat[i])
            gro = (Rr @ (ot - pos[i])) / scl[i]
            grdu = (Rr @ dt) / scl[i]
            grd = grdu / grdu.norm()
            gray = torch.linalg.cross(grd, gro).pow(2).sum()
            gres = torch.exp(a_exp * gray ** (degree / 2.0))
            a = torch.clamp(gres * dns[i], max=0.99)
            if not (float(gres) > 0.0113 and float(a) > 1.0 / 255.0):
                continue
            tt = (scl[i] * grd * (-(grd * gro).sum())).norm()
            col = torch.clamp(_sh(sph[i], dt), min=0.0)
            # the backward's re-trace stops strictly before the last processed hit (entry t here): no gradient of its own
            if ts >= float(last[k]) * (1.0 - 1e-5):
                tt, col, a = tt.detach(), col.detach(), a.detach()
            w = a * T
            C = C + w * col
            D = D + w * tt
            T = T * (1 - a)
        loss = loss + (C * torch.tensor(d_rgb.reshape(-1, 3)[k], dtype=f64)).sum() + (1 - T) * float(d_alpha.reshape(-1)[k]) \
            + D * float(d_dist.reshape(-1)[k])
    loss.backward()
    assert rel_l2(pos.grad.numpy(), dp[:, 0:3]) < 2e-3
    assert rel_l2(dns.grad.numpy(), dp[:, 3]) < 2e-3
    assert rel_l2(quat.grad.numpy(), dp[:, 4:8]) < 2e-3
    assert rel_l2(scl.grad.numpy(), dp[:, 8:11]) < 2e-3
    assert rel_l2(sph.grad.numpy().reshape(-1, 48), ds) < 2e-3


def test_scene_aabb_is_the_box_of_all_vertices():
    sc = scenes.scene_c1(n=300, seed=9)
    cfg = gio.paper_config(2)
    vrt, bb = gio.grt_proxies(cfg, sc.particles, clamping=False, primitive="icosahedron")
    # the reference's formula in float64: (V_i * kernelScale * scale * icosaVrtScale) * rot + pos
    kscl, _ = go.grt_proxies(cfg, sc.particles, clamping=False)
    v, _ = gio.table()
    P = sc.particles.astype(np.float64)
    r, x, y, z = P[:, 4], P[:, 5], P[:, 6], P[:, 7]
    R = np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], -1),
                  np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], -1),
                  np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], -1)], 1)
    w = np.einsum("nij,nvj->nvi", R, v.astype(np.float64)[None] * (kscl.astype(np.float64) * gio.ICO_VRT_SCALE)[:, None, :]) + P[:, None, 0:3]
    assert np.allclose(vrt, w, rtol=1e-5, atol=1e-6)
    box = np.concatenate([w.reshape(-1, 3).min(0), w.reshape(-1, 3).max(0)])
    assert np.allclose(bb, box, rtol=1e-6, atol=1e-6)

"""Float64 brute-force oracle of the playground render (grtb200_trace_playground, DESIGN.md section 22).  TEST INFRASTRUCTURE ONLY.

Restated from the issue's definition and the reference's Playground (not copied):
  closest_hit       every triangle tested (Moller-Trumbore, both faces), t in (1e-5, 1e5), ties to the lowest index   <- trace.cuh:traceMesh
  reflect / refract the mirror law about the normal turned against the ray, Snell with n1 = 1.0003 and total internal reflection as a
                    mirror bounce                                                          <- playgroundKernel.cu handleMirror / refract / handleGlass
  segment           the 3DGRT forward of one ray (instances proxy) on a segment (a, b) with a carried transmittance: every proxy the ray
                    segment meets, in order of its hit distance, integrated while T > min_transmittance (the brute-force twin of
                    oracle/gut_oracle.py: grt_trace, extended by the segment and T; the C oracle's entries stay as they are)
  render            the bounce loop: at most 32 mirror / TIR bounces, 1000 segments, stop at alpha 0.995, one front-to-back T through
                    every segment; diffuse adds T c |dot(d, n)| and ends the ray; the background on 1 - alpha, clamped to [0, 1]
"""
from __future__ import annotations

import numpy as np

T_MIN, T_MAX = 1e-5, 1e5
N_OUTSIDE = 1.0003
MAX_BOUNCES, MAX_SEGMENTS, STOP_ALPHA, REFRACT_SHIFT, BOUNCE_TMIN = 32, 1000, 0.995, 1e-5, 1e-9
MIRROR, GLASS, DIFFUSE = 0, 1, 2


# ---- meshes -----------------------------------------------------------------------------------------------------------------------

def closest_hit(v0, e1, e2, o, d):
    """Brute force over all triangles (float64) for rays o / d [R,3]: (t [R], u [R], v [R], tri [R]; tri -1 and t 1e5 on a miss)."""
    o, d = np.atleast_2d(np.asarray(o, np.float64)), np.atleast_2d(np.asarray(d, np.float64))
    R = o.shape[0]
    best_t, best_u, best_v, best_i = np.full(R, T_MAX), np.zeros(R), np.zeros(R), np.full(R, -1)
    for r in range(R):
        p = np.cross(d[r], e2)
        det = (e1 * p).sum(1)
        with np.errstate(divide="ignore", invalid="ignore"):
            inv = 1.0 / det
            s = o[r] - v0
            u = (s * p).sum(1) * inv
            q = np.cross(s, e1)
            v = (q @ d[r]) * inv
            t = (e2 * q).sum(1) * inv
        ok = np.nonzero((det != 0) & (u >= 0) & (u <= 1) & (v >= 0) & (u + v <= 1) & (t > T_MIN) & (t < T_MAX))[0]
        if len(ok):
            k = ok[np.argmin(t[ok])]  # argmin returns the first (lowest) index of a tie
            best_t[r], best_u[r], best_v[r], best_i[r] = t[k], u[k], v[k], k
    return best_t, best_u, best_v, best_i


def reflect(d, n):
    """Unit mirror direction of unit d about unit n turned against d: d - 2 dot(d, f) f with f = n or -n so that dot(d, f) <= 0."""
    f = n if np.dot(d, n) < 0 else -n
    r = d - 2 * np.dot(d, f) * f
    return r / np.linalg.norm(r)


def refract(d, n, ior):
    """(direction, refracted) of unit d at a glass surface of index `ior` with unit normal n: entering when dot(d, n) < 0 (ratio n1/ior),
    leaving otherwise (ior/n1); total internal reflection returns the mirror direction and False."""
    eta = ior / N_OUTSIDE
    front = np.dot(d, n) < 0
    ri, f = (1 / eta, n) if front else (eta, -n)
    ct = min(-np.dot(d, f), 1.0)
    st = np.sqrt(max(0.0, 1 - ct * ct))
    if ri * st > 1:
        return reflect(d, n), False
    perp = ri * (d + ct * f)
    out = perp - np.sqrt(abs(1 - perp @ perp)) * f
    return out / np.linalg.norm(out), True


def packed_triangles(vertices, faces):
    v = np.asarray(vertices, np.float64)[np.asarray(faces)]
    return v[:, 0], v[:, 1] - v[:, 0], v[:, 2] - v[:, 0]


# ---- Gaussians --------------------------------------------------------------------------------------------------------------------

def _rot(q):
    """Rotation matrices [N,3,3] of wxyz quaternions (as stored)."""
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y)], 1),
                     np.stack([2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x)], 1),
                     np.stack([2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], 1)], 1)


def sh_basis(d, deg=3):
    x, y, z = d
    b = np.zeros(16)
    b[0] = 0.28209479177387814
    if deg > 0:
        b[1], b[2], b[3] = -0.4886025119029199 * y, 0.4886025119029199 * z, -0.4886025119029199 * x
    if deg > 1:
        xx, yy, zz = x * x, y * y, z * z
        b[4], b[5] = 1.0925484305920792 * x * y, -1.0925484305920792 * y * z
        b[6], b[7] = 0.31539156525252005 * (2 * zz - xx - yy), -1.0925484305920792 * x * z
        b[8] = 0.5462742152960396 * (xx - yy)
    if deg > 2:
        b[9] = -0.5900435899266435 * y * (3 * xx - yy)
        b[10] = 2.890611442640554 * x * y * z
        b[11] = -0.4570457994644658 * y * (4 * zz - xx - yy)
        b[12] = 0.3731763325901154 * z * (2 * zz - 3 * xx - 3 * yy)
        b[13] = -0.4570457994644658 * x * (4 * zz - xx - yy)
        b[14] = 1.445305721320277 * z * (xx - yy)
        b[15] = -0.5900435899266435 * x * (xx - 3 * yy)
    return b


class Scene:
    """The Gaussians of a frame ([N,12] record, [N,48] SH) with the render settings of grtb200_config (instances proxies)."""

    def __init__(self, particles, sph, sph_degree=3, degree=4, min_response=0.0113, min_alpha=1 / 255, max_alpha=0.99, clamping=True,
                 min_transmittance=0.001):
        p = np.asarray(particles, np.float64)
        self.mu, self.dns, self.R, self.s = p[:, 0:3], p[:, 3], _rot(p[:, 4:8]), p[:, 8:11]
        self.sph = np.asarray(sph, np.float64).reshape(-1, 16, 3)
        self.sph_degree, self.degree, self.min_response, self.min_alpha, self.max_alpha = sph_degree, degree, min_response, min_alpha, max_alpha
        self.min_t = min_transmittance
        minr = np.minimum(min_response / (self.dns if clamping else 1.0), 0.97)
        ks = (np.log(minr) / (-4.5 / 3.0 ** degree)) ** (1.0 / degree)
        self.k = ks[:, None] * self.s                                   # proxy half extents (instance scale)
        half = (np.abs(self.R) * self.k[:, None, :]).sum(2)             # world box of the oriented box
        self.box = np.concatenate([(self.mu - half).min(0), (self.mu + half).max(0)]) if len(p) else np.zeros(6)

    def _clip(self, o, d):
        with np.errstate(divide="ignore", invalid="ignore"):
            a, b = (self.box[:3] - o) / d, (self.box[3:] - o) / d
        return max(0.0, np.nanmax(np.minimum(a, b))), np.nanmin(np.maximum(a, b))

    def segment(self, o, d, a, b, T, C):
        """The Gaussians of the ray o + t d on (a, b) (inside the scene box), front to back from transmittance T and radiance C [3];
        returns (T, C)."""
        if len(self.mu) == 0:
            return T, C
        t0, t1 = self._clip(o, d)
        lo, hi = max(t0, a), min(t1, b)
        if not lo <= hi or not T > self.min_t:
            return T, C
        v = o - self.mu
        oi = np.einsum("nji,nj->ni", self.R, v) / self.k                # R^T (o - mu) / k
        di = np.einsum("nji,j->ni", self.R, d) / self.k
        with np.errstate(divide="ignore", invalid="ignore"):
            q0, q1 = (-1 - oi) / di, (1 - oi) / di
            tin = np.maximum(lo, np.nanmax(np.minimum(q0, q1), 1))
            tout = np.minimum(hi, np.nanmin(np.maximum(q0, q1), 1))
            dd = (di * di).sum(1)
            ht = -(oi * di).sum(1) / dd
            nrm = di / np.sqrt(dd)[:, None]
            cr = (np.cross(nrm, oi) ** 2).sum(1) / dd
        cand = np.nonzero((tin <= tout) & (ht > lo) & (ht < hi) & (cr < 9))[0]
        basis = sh_basis(d, self.sph_degree)
        C = np.array(C, np.float64)
        for i in cand[np.argsort(ht[cand], kind="stable")]:
            if not T > self.min_t:
                break
            gro = self.R[i].T @ v[i] / self.s[i]
            grd = self.R[i].T @ d / self.s[i]
            grd = grd / np.linalg.norm(grd)
            gray = (np.cross(grd, gro) ** 2).sum()
            gres = np.exp(-gray * gray / 18.0) if self.degree == 4 else np.exp(-0.5 * gray)
            alpha = min(self.max_alpha, gres * self.dns[i])
            if not (gres > self.min_response and alpha > self.min_alpha):
                continue
            rgb = np.maximum(0.5 + basis @ self.sph[i], 0.0)
            C = C + rgb * alpha * T
            T = T * (1 - alpha)
        return T, C


# ---- the bounce loop --------------------------------------------------------------------------------------------------------------

def render_ray(scene: Scene, tris, vnormals, faces, tri_material, materials, o, d, background=(0, 0, 0), smooth=True, ray_max_t=1e9):
    """One world ray -> (rgb [3], alpha, path) with path the list of (triangle, material kind) it met.  tris = packed_triangles(...),
    materials [M,8] rows (kind, ior, 0, 0, r, g, b, 0)."""
    v0, e1, e2 = tris
    o, d = np.asarray(o, np.float64), np.asarray(d, np.float64)
    T, C = 1.0, np.zeros(3)
    t, u, v, tri = (x[0] for x in closest_hit(v0, e1, e2, o[None], d[None]))
    T, C = scene.segment(o, d, 0.0, t if tri >= 0 else ray_max_t, T, C)
    bounces, segments, path = 0, 1, []
    while tri >= 0:
        mk = materials[tri_material[tri]]
        kind = int(mk[0])
        path.append((int(tri), kind))
        if smooth:
            f = faces[tri]
            n = (1 - u - v) * vnormals[f[0]] + u * vnormals[f[1]] + v * vnormals[f[2]]
        else:
            n = np.cross(e1[tri], e2[tri])
        n = n / np.linalg.norm(n)
        dn = d / np.linalg.norm(d)
        if kind == DIFFUSE:
            C = C + T * np.asarray(mk[4:7], np.float64) * abs(dn @ n)
            T = 0.0
            break
        if kind == MIRROR:
            nd, bounced = reflect(dn, n), True
        else:
            nd, refracted = refract(dn, n, mk[1])
            bounced = not refracted
            if refracted:
                t = t + REFRACT_SHIFT
        bounces += int(bounced)
        o, d = o + t * d, nd
        if not (1 - T < STOP_ALPHA) or bounces >= MAX_BOUNCES or segments >= MAX_SEGMENTS:
            break
        t, u, v, tri = (x[0] for x in closest_hit(v0, e1, e2, o[None], d[None]))
        T, C = scene.segment(o, d, BOUNCE_TMIN, t if tri >= 0 else ray_max_t, T, C)
        segments += 1
    alpha = 1 - T
    rgb = np.clip(C + np.asarray(background, np.float64) * (1 - alpha), 0, 1)
    return rgb, float(np.clip(alpha, 0, 1)), path

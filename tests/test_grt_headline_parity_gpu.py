"""Oracle parity of the CUDA 3DGRT tracer AT THE HEADLINE SCALES, through the C ABI (b200_native.GrtContext): the C4 workload of bench.py
(scene_c2(): 300k Gaussians, 800x800) on two cameras, the paper's icosahedron config, the C3-like unbounded scene (400k, 1237x822), the
hit-list overflow + re-trace backward, a "ray soup" of incoherent rays starting inside the cloud, and NHT features.  The C1-scale tests
(test_grt_parity_gpu.py, test_grt_icosahedron_gpu.py, test_grt_nht_gpu.py) never reach a deep LBVH, several k-nearest queries per ray
or tens of hits per ray; here the GPU traces and differentiates the whole frame with its production packets, warps and hit lists.

The brute-force oracle is O(N) per ray, so it runs on a seeded SAMPLE of the rays (the last row and column added; every ray of the soup).
It treats rays independently, so on the sample it is exact, not an approximation; and with the output gradient zero on every other ray
the GPU backward of the full frame is the oracle's backward of the sampled rays alone (tests/test_grt_ray_sample_oracle.py pins both).

Bars (DESIGN.md sections 5, 9), P = rays compared: rgb (or 24 features) + alpha mean |diff| <= 1e-5, max <= 2e-2, |diff| > 1e-4 on at most
max(3, 2e-4 P) rays; distance the same relative to max(1, max |dist|); hit counts equal on >= 99.9 % of the rays; every particle the
oracle's sampled rays accept is visible on the GPU (which traced a superset of the rays), at most 0.1 % missing -- equal on >= 99.9 % of
the particles for the soup; no non-finite value anywhere.  Gradients per tensor, the policy of test_gut_headline_parity_gpu.py:
err <= max(1e-3, 1.5 x yardstick), yardstick = the oracle's fp32 vs fp64 evaluation of the same rays (NHT: the composite over the fp32
oracle's hit lists vs the fp64 one's), AND err <= 1e-3 flat once the ten particles with the largest yardstick error (picked from the
oracle pair, never from the GPU output) are removed.  Rays on which the reference's own backward drops an accepted hit (its proxy box
begins beyond the ray's last distance, see _rays_past_box_end) get no output gradient; at most 1 % of the rays may be such rays."""
import dataclasses
import functools
import math
import os
import time

import numpy as np
import pytest

import grt_ico_oracle as gio
import scenes
from helpers import image_error_report, ray_sample, rel_l2
from oracle import gut_oracle as go

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import grt_nht_oracle as gno  # noqa: E402

CORES = len(os.sched_getaffinity(0))
RAYS = 8192 if CORES >= 16 else 4096  # sampled pixels per frame (plus the last row and column): the oracle's cost is O(N) per ray
NHT_RAYS = 4096
MIN_T = 1e-3
GRADS = ("pos", "dns", "quat", "scl", "feat")


@functools.lru_cache(maxsize=None)
def _c2():
    return scenes.scene_c2()


@functools.lru_cache(maxsize=None)
def _c3():
    return scenes.scene_c3(n=400_000)


@dataclasses.dataclass
class _Frame:
    label: str
    particles: np.ndarray
    sph: np.ndarray
    ro: np.ndarray      # [H,W,3] ray origins, ray space
    rd: np.ndarray      # [H,W,3]
    c2w: np.ndarray     # ray-to-world
    idx: np.ndarray     # sorted flat indices of the rays compared with the oracle
    seed: int
    degree: int = 4
    prim: str = "instances"
    clamping: bool = True

    @property
    def cfg(self):
        cfg = go.grt_config()
        cfg.kernel_degree = self.degree
        return cfg


def _camera_frame(label, sc, cam, n_cams, seed, **kw):
    ro, rd = sc.rays()
    return _Frame(label, sc.particles, sc.sph, ro[0], rd[0], np.asarray(sc.camera(cam, n_cams), np.float32),
                  ray_sample(sc.height, sc.width, RAYS, seed), seed, **kw)


def _ray_soup():
    """16,384 rays laid out as 128x128: origins uniform in the cloud's cube, directions uniform on the sphere, identity ray-to-world."""
    rng = np.random.default_rng(41)
    ro = rng.uniform(-1.3, 1.3, (128, 128, 3)).astype(np.float32)
    rd = rng.normal(size=(128, 128, 3))
    rd = (rd / np.linalg.norm(rd, axis=-1, keepdims=True)).astype(np.float32)
    sc = _c2()
    return _Frame("F soup", sc.particles, sc.sph, ro, rd, np.eye(4, dtype=np.float32), np.arange(128 * 128), 41)


FRAMES = {
    "A": lambda: _camera_frame("A c4 cam3", _c2(), 3, 100, 3),
    "B": lambda: _camera_frame("B c4 cam41", _c2(), 41, 100, 41),
    "C": lambda: _camera_frame("C c4 cam3 icosahedron d2", _c2(), 3, 100, 3, degree=2, prim="icosahedron", clamping=False),
    "D": lambda: _camera_frame("D c3-like 400k cam1", _c3(), 1, 10, 1),
    "F": _ray_soup,
}


def _out_grads(P, seed, channels=3):
    rng = np.random.default_rng(seed)
    return (rng.normal(size=(P, channels)).astype(np.float32), rng.normal(size=P).astype(np.float32),
            (0.1 * rng.normal(size=P)).astype(np.float32))


def _sampled(fr):
    return fr.ro.reshape(-1, 3)[fr.idx], fr.rd.reshape(-1, 3)[fr.idx]


def _rays_past_box_end(fr, ro, rd):
    """Rays (bool [P]) with an accepted `instances` hit whose proxy box begins beyond the ray's last processed distance: its t* lies
    before the box entry (the ray clips a corner of the proxy).  The reference's backward re-trace ends at that distance, so OptiX (and
    the oracle) cull the box and the hit gets no gradient; the replayed hit list keeps it (DESIGN.md section 9).  Picked from the oracle's
    lists and proxies, never from the GPU output."""
    L = gno.trace_lists(fr.cfg, fr.particles, ro, rd, fr.c2w, clamping=fr.clamping)
    kscl, _ = go.grt_proxies(fr.cfg, fr.particles, fr.clamping)
    o, d = (t.numpy() for t in gno.world_rays(ro, rd, fr.c2w))
    r, s = np.nonzero((np.arange(L["pid"].shape[1])[None] < L["count"][:, None]) & (L["alpha"] > 0))
    pid = L["pid"][r, s]
    p = fr.particles[pid].astype(np.float64)
    rows = gno._rot_rows(torch.from_numpy(p[:, 4:8])).numpy()
    k = kscl[pid].astype(np.float64)
    oi, di = np.einsum("mab,mb->ma", rows, o[r] - p[:, 0:3]) / k, np.einsum("mab,mb->ma", rows, d[r]) / k
    with np.errstate(divide="ignore"):
        entry = np.minimum((-1 - oi) / di, (1 - oi) / di).max(1)
    out = np.zeros(len(ro), bool)
    out[r[entry > L["last"][r]]] = True
    return out


def _sh_oracle(fr):
    """Forward + backward of the oracle on the sampled rays, in fp32 and in fp64 (the yardstick)."""
    ro, rd = _sampled(fr)
    kw = dict(clamping=fr.clamping, primitive=fr.prim)
    grads = _out_grads(len(fr.idx), fr.seed)
    t0 = time.perf_counter()
    if fr.prim == "instances":  # icosahedron hits are box entries: no such hit exists
        past = _rays_past_box_end(fr, ro, rd)
        print(f"\n[grt-headline] {fr.label}: {int(past.sum())} of {len(past)} rays have an accepted hit whose proxy box begins beyond the "
              f"ray's last distance; they get no output gradient")
        assert past.mean() <= 0.01
        grads = tuple(g * (~past).reshape(-1, *([1] * (g.ndim - 1))) for g in grads)
    res = {}
    for tag, f64 in (("", False), ("64", True)):
        rgb, alpha, dist, hits, vis = gio.grt_trace(fr.cfg, fr.particles, fr.sph, 3, ro, rd, fr.c2w, f64=f64, **kw)
        dp, ds = gio.grt_trace_bwd(fr.cfg, fr.particles, fr.sph, 3, ro, rd, fr.c2w, rgb, alpha, dist, *grads, f64=f64, **kw)
        res[tag] = dict(rgb=rgb, alpha=alpha[:, 0], dist=dist[:, 0], hits=hits[:, 0], vis=vis[:, 0] != 0,
                        grads=_split(dp, ds))
    res["grads_in"] = grads
    res["secs"] = time.perf_counter() - t0
    return res


def _split(dp, df):
    return dict(pos=dp[:, 0:3], dns=dp[:, 3:4], quat=dp[:, 4:8], scl=dp[:, 8:11], feat=df)


class _Oracle:
    """Each frame's oracle results, computed once for the module."""

    def __init__(self):
        self._sh = {}

    def sh(self, fid):
        if fid not in self._sh:
            fr = FRAMES[fid]()
            self._sh[fid] = (fr, _sh_oracle(fr))
        return self._sh[fid]


@pytest.fixture(scope="module")
def oracle():
    return _Oracle()


class _Gpu:
    """One native 3DGRT context over a whole frame: the BVH, the rays and the outputs its backward replays."""

    def __init__(self, fr, max_alpha=None):
        import b200_native as nat

        c = nat.grt_default_config()
        c.kernel_degree, c.density_clamping, c.primitive = fr.degree, int(fr.clamping), nat.GRT_PRIMITIVES[fr.prim]
        if max_alpha is not None:
            c.max_alpha = max_alpha
        self.ctx = nat.GrtContext(c, 0)
        self.stream = torch.cuda.current_stream().cuda_stream
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()  # noqa: E731
        self.n = int(fr.particles.shape[0])
        self.p, self.sph = t(fr.particles), t(fr.sph)
        self.ro, self.rd = t(fr.ro), t(fr.rd)
        self.h, self.w = (int(v) for v in fr.ro.shape[:2])
        self.R = self.h * self.w
        self.r2w = np.ascontiguousarray(np.asarray(fr.c2w, np.float32)[:3, :4])
        self.ctx.build_bvh_packed(self.stream, self.n, self.p.data_ptr())

    def _rays(self):
        return (MIN_T, 1, self.h, self.w, self.ro.data_ptr(), self.rd.data_ptr(), self.r2w.ctypes.data)

    def _outputs(self, channels):
        nan = float("nan")  # every output must be written
        R = self.R
        return [torch.full((R, channels), nan, device="cuda"), torch.full((R,), nan, device="cuda"), torch.full((R, 2), nan, device="cuda"),
                torch.full((R,), nan, device="cuda"), torch.full((self.n,), nan, device="cuda")]

    def counters(self, label):
        vis = torch.zeros(self.n, device="cuda")
        c = self.ctx.trace_counters(self.stream, self.n, self.p.data_ptr(), self.sph.data_ptr(), 3, *self._rays(), vis.data_ptr())
        packet, queries = c["packet_rays"] / c["rays"], c["queries"] / c["rays"]
        print(f"[grt-headline] {label}: trace counters {c}; packet-walked rays {100 * packet:.1f} %, {queries:.2f} k-nearest queries "
              f"and {c['accepted_hits'] / c['rays']:.2f} accepted hits per ray")
        return packet, queries

    def trace(self):
        self.out = self._outputs(3)
        self.ctx.trace(self.stream, self.n, self.p.data_ptr(), self.sph.data_ptr(), 3, *self._rays(), *[o.data_ptr() for o in self.out])
        torch.cuda.synchronize()
        return self._numpy(self.out)

    def trace_bwd(self, idx, d_rgb, d_alpha, d_dist):
        d = self._scatter(idx, d_rgb, d_alpha, d_dist)
        dp, ds = torch.full((self.n, 12), float("nan"), device="cuda"), torch.full((self.n, 48), float("nan"), device="cuda")
        self.ctx.trace_bwd(self.stream, self.n, self.p.data_ptr(), self.sph.data_ptr(), 3, *self._rays(), *[o.data_ptr() for o in self.out[:3]],
                           *[t.data_ptr() for t in d], dp.data_ptr(), ds.data_ptr())
        torch.cuda.synchronize()
        return dp.cpu().numpy(), ds.cpu().numpy()

    def trace_nht(self, feats16):
        self.f = feats16
        self.out = self._outputs(24)
        self.ctx.trace_nht(self.stream, self.n, self.p.data_ptr(), self.f.data_ptr(), 48, 1, *self._rays(), *[o.data_ptr() for o in self.out])
        torch.cuda.synchronize()
        return self._numpy(self.out)

    def trace_bwd_nht(self, idx, d_feat, d_alpha, d_dist):
        d = self._scatter(idx, d_feat, d_alpha, d_dist)
        dp, df = torch.full((self.n, 12), float("nan"), device="cuda"), torch.full((self.n, 48), float("nan"), device="cuda")
        self.ctx.trace_bwd_nht(self.stream, self.n, self.p.data_ptr(), self.f.data_ptr(), 48, 1, *self._rays(),
                               *[o.data_ptr() for o in self.out[:3]], *[t.data_ptr() for t in d], dp.data_ptr(), df.data_ptr())
        torch.cuda.synchronize()
        return dp.cpu().numpy(), df.cpu().numpy()

    def _scatter(self, idx, *grads):
        """Output gradients of the full frame: the sampled rays' values, exactly zero on every other ray."""
        out = []
        for g in grads:
            full = np.zeros((self.R, *g.shape[1:]), np.float32)
            full[idx] = g
            out.append(torch.from_numpy(full).cuda())
        return out

    @staticmethod
    def _numpy(out):
        rgb, alpha, dist, hits, vis = (o.cpu().numpy() for o in out)
        return dict(rgb=rgb, alpha=alpha, dist=dist[:, 0], hits=hits, vis=vis.view(np.int32) != 0, raw=(rgb, alpha, dist, hits, vis))


def _finite(label, *arrays):
    for a in arrays:
        assert np.isfinite(a).all(), f"{label}: non-finite values in an output or gradient"


def _check_outputs(label, got, ref, idx, vis_equal=False):
    """Images, distances, hit counts and visibility of the GPU's full frame at the sampled rays against the oracle."""
    _finite(label, *got["raw"])
    P = len(idx)
    ch = got["rgb"].shape[1]
    g = np.concatenate([got["rgb"][idx], got["alpha"][idx, None]], -1)[:, None]
    w = np.concatenate([ref["rgb"], ref["alpha"][:, None]], -1)[:, None]
    mean, mx, bad = image_error_report(f"{label} {'rgb' if ch == 3 else 'features'}+alpha", g, w)
    assert mean <= 1e-5 and mx <= 2e-2 and bad <= max(3, int(2e-4 * P)), (mean, mx, bad)
    scale = max(1.0, float(np.abs(ref["dist"]).max()))
    mean, mx, bad = image_error_report(f"{label} dist", got["dist"][idx, None, None], ref["dist"][:, None, None], atol=1e-4 * scale)
    assert mean <= 1e-5 * scale and mx <= 2e-2 * scale and bad <= max(3, int(2e-4 * P)), (mean, mx, bad)
    same = float(np.mean(got["hits"][idx] == ref["hits"]))
    print(f"[grt-headline] {label}: hit counts equal on {100 * same:.3f} % of {P} rays")
    assert same >= 0.999
    if vis_equal:
        eq = float(np.mean(got["vis"] == ref["vis"]))
        print(f"[grt-headline] {label}: visibility equal on {100 * eq:.4f} % of the particles")
        assert eq >= 0.999
    else:
        missing = int((ref["vis"] & ~got["vis"]).sum())
        print(f"[grt-headline] {label}: {int(ref['vis'].sum())} particles visible to the oracle's rays, {missing} of them not visible on the "
              f"GPU ({int(got['vis'].sum())} visible in the full frame)")
        assert missing <= 1e-3 * ref["vis"].sum()


def _check_grads(label, got, ref, other):
    """got / ref / other: dicts of the five gradient tensors (GPU, oracle, the oracle's other precision)."""
    errs = {k: rel_l2(got[k], ref[k]) for k in GRADS}
    yard = {k: rel_l2(ref[k], other[k]) for k in GRADS}
    n = ref["pos"].shape[0]
    e2 = np.zeros(n)
    for k in GRADS:
        a, b = np.asarray(ref[k], np.float64).reshape(n, -1), np.asarray(other[k], np.float64).reshape(n, -1)
        e2 += ((a - b) ** 2).sum(1) / max(float((b ** 2).sum()), 1e-300)
    keep = np.ones(n, bool)
    keep[np.argsort(-e2)[:10]] = False
    robust = {k: rel_l2(got[k][keep], ref[k][keep]) for k in GRADS}
    fmt = lambda d: {k: f"{v:.2e}" for k, v in d.items()}  # noqa: E731
    print(f"[grt-headline] {label} gradient rel-L2 vs oracle:", fmt(errs))
    print(f"[grt-headline] {label} yardstick (oracle fp32 vs fp64, same rays):", fmt(yard))
    print(f"[grt-headline] {label} gradient rel-L2 without the oracle's 10 flip particles:", fmt(robust))
    for k in GRADS:
        assert errs[k] <= max(1e-3, 1.5 * yard[k]), (k, errs[k], yard[k])
        assert robust[k] <= 1e-3, (k, robust[k])


def _describe(fr, ref, secs):
    h = ref["hits"]
    print(f"\n[grt-headline] {fr.label}: N={fr.particles.shape[0]} frame {fr.ro.shape[1]}x{fr.ro.shape[0]}, {len(fr.idx)} rays compared "
          f"(RAYS={RAYS}, {CORES} cores), oracle hits per ray mean {h.mean():.2f} max {int(h.max())}, {100 * np.mean(h > 0):.1f} % of the "
          f"rays hit; oracle wall time {secs:.1f} s")


def _check_sh_frame(fr, ref, packet_min=None, packet_max=None, vis_equal=False):
    _describe(fr, ref[""], ref["secs"])
    g = _Gpu(fr)
    packet, queries = g.counters(fr.label)
    if packet_min is not None:
        assert packet >= packet_min
    if packet_max is not None:
        assert packet <= packet_max
    assert queries > 1.0
    got = g.trace()
    _check_outputs(fr.label, got, ref[""], fr.idx, vis_equal)
    dp, ds = g.trace_bwd(fr.idx, *ref["grads_in"])
    _finite(fr.label, dp, ds)
    assert np.all(dp[:, 11] == 0)
    _check_grads(fr.label, _split(dp, ds), ref[""]["grads"], ref["64"]["grads"])
    g.ctx.close()
    return got


@pytest.mark.parametrize("fid", ["A", "B", "C", "D"])
def test_camera_frame_matches_the_oracle(oracle, fid):
    """A, B: the C4 workload of bench.py (default config: instances, degree 4, clamping); C: the paper config (icosahedron proxies,
    degree 2, no density clamping); D: the C3-like unbounded scene, background out to radius 50, the camera inside the cloud, a ragged
    frame whose last row and column are partly filled 8x4 ray blocks.  Every block of a camera frame walks the tree as a packet."""
    fr, ref = oracle.sh(fid)
    _check_sh_frame(fr, ref, packet_min=0.9)


def test_hit_list_overflow_and_retrace_match_the_oracle(oracle, monkeypatch):
    """Frame A with a hit-list capacity of 8 (GRTB200_HITCAP, read at every trace): most hitting rays overflow their list and the
    backward re-traces them instead of replaying, against the same oracle results as frame A."""
    fr, ref = oracle.sh("A")
    h = ref[""]["hits"]
    over = float(np.mean(h[h > 0] > 8))
    print(f"[grt-headline] E: {100 * over:.1f} % of the sampled rays that hit ({100 * np.mean(h > 8):.1f} % of all sampled rays) have more "
          f"than 8 oracle hits")
    assert over > 0.5
    monkeypatch.setenv("GRTB200_HITCAP", "8")
    got = _check_sh_frame(dataclasses.replace(fr, label="E c4 cam3 hit cap 8"), ref, packet_min=0.9)
    print(f"[grt-headline] E: {int((got['hits'] > 8).sum())} of {got['hits'].size} rays of the full frame overflow a list of 8")


def test_ray_soup_matches_the_oracle(oracle):
    """Incoherent rays starting inside the cloud: the per-thread walk (no packets), every ray compared."""
    fr, ref = oracle.sh("F")
    _check_sh_frame(fr, ref, packet_max=0.1, vis_equal=True)


def test_nht_frame_matches_the_oracle():
    """C4 camera 3 with fp16 NHT features at the *_3dgrt_mcmc_nht settings (instances, degree 4, max_alpha 0.999) and every 7th density
    at 3.0 so that hits reach the clamp; the float64 list oracle (tests/grt_nht_oracle.py) on 4,096 sampled rays."""
    sc = _c2()
    particles = sc.particles.copy()
    particles[::7, 3] = 3.0
    feats = np.random.default_rng(7).uniform(-math.pi / 2, math.pi / 2, (sc.n, 48)).astype(np.float16)
    ro, rd = sc.rays()
    fr = _Frame("G c4 cam3 NHT fp16", particles, sc.sph, ro[0], rd[0], np.asarray(sc.camera(3, 100), np.float32),
                ray_sample(sc.height, sc.width, NHT_RAYS, 5), 5)
    cfg = fr.cfg
    cfg.max_alpha = 0.999
    ros, rds = _sampled(fr)
    grads = _out_grads(len(fr.idx), fr.seed, 24)
    f32 = feats.astype(np.float32)  # what the kernel reads
    t0 = time.perf_counter()
    ref = gno.frame(cfg, particles, f32, ros, rds, fr.c2w, *grads, device="cuda")
    ref32 = gno.frame(cfg, particles, f32, ros, rds, fr.c2w, *grads, device="cuda", lists_f64=False)
    secs = time.perf_counter() - t0
    want = dict(rgb=ref["feat"], alpha=ref["alpha"], dist=ref["dist"][:, 0], hits=ref["hits"], vis=np.zeros(sc.n, bool))
    want["vis"][ref["lists"]["pid"][(ref["lists"]["alpha"] > 0)]] = True
    _describe(fr, want, secs)
    clamped = int((ref["lists"]["alpha"] == np.float32(0.999)).sum())
    print(f"[grt-headline] {fr.label}: {clamped} oracle hits clamped at max_alpha 0.999")
    assert clamped > 0

    g = _Gpu(fr, max_alpha=0.999)
    packet, queries = g.counters(fr.label)
    assert packet >= 0.9 and queries > 1.0
    got = g.trace_nht(torch.from_numpy(feats).cuda())
    _check_outputs(fr.label, got, want, fr.idx)
    dp, df = g.trace_bwd_nht(fr.idx, *grads)
    _finite(fr.label, dp, df)
    _check_grads(fr.label, _split(dp, df), _split(ref["dp"], ref["df"]), _split(ref32["dp"], ref32["df"]))
    g.ctx.close()

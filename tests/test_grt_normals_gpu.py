"""3DGRT normals (render.enable_normals with SH radiance, grtb200_trace_normals) on the GPU: the raw normal sums against the float64
oracle over the brute-force oracle's hit lists (tests/grt_normals_oracle.py), the other outputs untouched, the backward unchanged,
Tracer.render's pred_normals, and the training steps with the key on.

Bars of test_grt_parity_gpu.py (DESIGN.md sections 5, 9, 17): mean |diff| <= 1e-5, |diff| <= 1e-4 on all but max(3, 2e-4 P) rays, max
<= 2e-2 (an accept-test flip moves one hit's weight)."""
import dataclasses

import numpy as np
import pytest

import scenes
from helpers import image_error_report, packet_share, permute_pixels, ray_sample, rel_l2, shuffled_pixels, unpermute_pixels
from oracle import gut_oracle as go
from train_step import raw_params

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
import grt_normals_oracle as gnr  # noqa: E402

MIN_T = 1e-3


class _Gpu:
    """One native 3DGRT context with a BVH over the particles, and the device buffers of a frame."""

    def __init__(self, particles, sph, c2w, ro, rd, deg=4, prim="instances", clamping=True):
        import b200_native as nat

        c = nat.grt_default_config()
        c.kernel_degree, c.primitive, c.density_clamping = deg, nat.GRT_PRIMITIVES[prim], int(clamping)
        self.ctx = nat.GrtContext(c, 0)
        self.stream = torch.cuda.current_stream().cuda_stream
        self.n = int(particles.shape[0])
        self.p = torch.from_numpy(np.ascontiguousarray(particles, np.float32)).cuda()
        self.s = torch.from_numpy(np.ascontiguousarray(sph, np.float32)).cuda()
        self.ro = torch.from_numpy(np.ascontiguousarray(ro, np.float32)).cuda()
        self.rd = torch.from_numpy(np.ascontiguousarray(rd, np.float32)).cuda()
        self.b, self.h, self.w = (int(v) for v in self.ro.shape[:3])
        self.R = self.b * self.h * self.w
        self.r2w = np.ascontiguousarray(np.asarray(c2w, np.float32)[:3, :4])
        self.ctx.build_bvh_packed(self.stream, self.n, self.p.data_ptr())

    def _args(self):
        return (self.stream, self.n, self.p.data_ptr(), self.s.data_ptr(), 3, MIN_T, self.b, self.h, self.w, self.ro.data_ptr(),
                self.rd.data_ptr(), self.r2w.ctypes.data)

    def forward(self, normals, fill=float("nan")):
        """Outputs prefilled with `fill`, so that a ray the trace does not write shows up."""
        R = self.R
        self.rgb, self.alpha = torch.full((R, 3), fill, device="cuda"), torch.full((R,), fill, device="cuda")
        self.dist, self.hits = torch.full((R, 2), fill, device="cuda"), torch.full((R,), fill, device="cuda")
        self.vis = torch.full((self.n,), fill, device="cuda")
        outs = (self.rgb.data_ptr(), self.alpha.data_ptr(), self.dist.data_ptr(), self.hits.data_ptr(), self.vis.data_ptr())
        if normals:
            self.nrm = torch.full((R, 3), fill, device="cuda")
            self.ctx.trace_normals(*self._args(), *outs, self.nrm.data_ptr())
        else:
            self.ctx.trace(*self._args(), *outs)
        torch.cuda.synchronize()
        return {k: getattr(self, k).cpu().numpy() for k in (("rgb", "alpha", "dist", "hits", "vis") + (("nrm",) if normals else ()))}

    def backward(self, grads):
        d_rgb, d_alpha, d_dist = (torch.from_numpy(g).cuda() for g in grads)
        dp, ds = torch.empty((self.n, 12), device="cuda"), torch.empty((self.n, 48), device="cuda")
        before = self.ctx.launch_count()
        self.ctx.trace_bwd(*self._args(), self.rgb.data_ptr(), self.alpha.data_ptr(), self.dist.data_ptr(), d_rgb.data_ptr(),
                           d_alpha.data_ptr(), d_dist.data_ptr(), dp.data_ptr(), ds.data_ptr())
        torch.cuda.synchronize()
        return dp.cpu().numpy(), ds.cpu().numpy(), self.ctx.launch_count() - before


def _check_parity(label, got, ref):
    P = ref.shape[0]
    assert np.isfinite(got).all() and np.isfinite(ref).all()
    mean_e, max_e, bad = image_error_report(label, got[:, None, :], ref[:, None, :])
    assert mean_e <= 1e-5 and max_e <= 2e-2 and bad <= max(3, int(2e-4 * P))


def _fisheye_c1():
    base = scenes.scene_c1()
    f = 0.9 * base.width
    return dataclasses.replace(base, fx=f, fy=f, fisheye=(0.05, -0.01, 0.002, -0.0003, 0.6))


# (scene, camera, kernel degree, primitive, density clamping): the default config on both proxies, the degree-2 paper config
# (icosahedron, no clamping), clamping off on instances, a dense scene and a fisheye ray set
CASES = {
    "c1 instances d4": (lambda: scenes.scene_c1(), 1, 4, "instances", True),
    "c1 icosahedron d4": (lambda: scenes.scene_c1(), 6, 4, "icosahedron", True),
    "c1 icosahedron d2 paper": (lambda: scenes.scene_c1(width=75, height=53), 3, 2, "icosahedron", False),
    "c1 instances d2 no clamping": (lambda: scenes.scene_c1(width=75, height=53), 0, 2, "instances", False),
    "dense instances d4": (lambda: scenes.scene_c1(n=5000, seed=8, width=64, height=64), 2, 4, "instances", True),
    "fisheye instances d4": (_fisheye_c1, 2, 4, "instances", True),
}


def _walk_rays(sc, c2w, ro, rd, walk, deg, prim, clamping=True):
    """The rays of `walk`: "packet" the camera's order, where every warp's rays are coherent; "per-lane" a seeded pixel order that no
    warp's rays are coherent in.  Returns (ro, rd, perm), perm None for the camera's order."""
    import b200_native as nat

    perm = shuffled_pixels(sc.height, sc.width) if walk == "per-lane" else None
    if perm is not None:
        ro, rd = permute_pixels(ro, perm), permute_pixels(rd, perm)
    share = packet_share(sc.particles, sc.sph, c2w, ro, rd, kernel_degree=deg, primitive=nat.GRT_PRIMITIVES[prim],
                         density_clamping=int(clamping))
    assert share >= 0.9 if perm is None else share <= 0.1
    return ro, rd, perm


def _unpermuted(out, perm):
    return out if perm is None else {k: (v if k == "vis" else unpermute_pixels(v, perm)) for k, v in out.items()}


@pytest.mark.parametrize("walk", ["packet", "per-lane"])
@pytest.mark.parametrize("case", list(CASES))
def test_normals_match_the_f64_oracle(case, walk):
    """per-lane: the same rays in a seeded pixel order, so that every warp takes the per-lane walk instead of the packet walk."""
    make, cam, deg, prim, clamping = CASES[case]
    sc = make()
    ro, rd = sc.rays()
    c2w = np.asarray(sc.camera(cam, 10), np.float32)
    cfg = go.grt_config()
    cfg.kernel_degree = deg
    ref, lists = gnr.frame(cfg, sc.particles, ro[0], rd[0], c2w, primitive=prim, clamping=clamping)
    assert (lists["count"] > 0).sum() > 100
    wro, wrd, perm = _walk_rays(sc, c2w, ro, rd, walk, deg, prim, clamping)
    out = _unpermuted(_Gpu(sc.particles, sc.sph, c2w, wro, wrd, deg, prim, clamping).forward(normals=True), perm)
    _check_parity(f"normals {case} {walk} walk", out["nrm"], ref)
    none = out["hits"] == 0  # rays that accepted no hit (the fisheye frame's corners): written, and zero
    assert np.array_equal(out["nrm"][none], np.zeros((int(none.sum()), 3), np.float32))


@pytest.mark.parametrize("frame", ["c4 cam3 instances", "c4 cam3 icosahedron d2"])
def test_normals_at_c4_on_a_ray_sample(frame):
    """C4 (bench.py's workload: 300k Gaussians, 800x800): the GPU traces the whole frame, the oracle a seeded sample of its rays (plus the
    last row and column); rays are independent, so on the sample the comparison is exact."""
    sc = scenes.scene_c2()
    ro, rd = sc.rays()
    c2w = np.asarray(sc.camera(3, 100), np.float32)
    deg, prim, clamping = (4, "instances", True) if frame.endswith("instances") else (2, "icosahedron", False)
    idx = ray_sample(sc.height, sc.width, 2048, 3)
    cfg = go.grt_config()
    cfg.kernel_degree = deg
    ref, lists = gnr.frame(cfg, sc.particles, ro[0].reshape(-1, 3)[idx], rd[0].reshape(-1, 3)[idx], c2w, primitive=prim, clamping=clamping)
    assert (lists["count"] > 0).sum() > 1000
    out = _Gpu(sc.particles, sc.sph, c2w, ro, rd, deg, prim, clamping).forward(normals=True)
    assert np.isfinite(out["nrm"]).all()
    _check_parity(f"normals {frame}", out["nrm"][idx], ref)


@pytest.mark.parametrize("walk", ["packet", "per-lane"])
@pytest.mark.parametrize("prim", ["instances", "icosahedron"])
@pytest.mark.parametrize("deg", [4, 2])
def test_normals_leave_every_other_output_bit_identical(deg, prim, walk):
    sc = scenes.scene_c2(n=40_000, width=160, height=128)
    c2w = np.asarray(sc.camera(2, 10), np.float32)
    ro, rd, _ = _walk_rays(sc, c2w, *sc.rays(), walk, deg, prim)
    g = _Gpu(sc.particles, sc.sph, c2w, ro, rd, deg, prim)
    plain, with_n = g.forward(normals=False), g.forward(normals=True)
    assert plain["hits"].sum() > 1000
    for k in ("rgb", "alpha", "dist", "hits", "vis"):
        assert np.array_equal(plain[k].view(np.uint32), with_n[k].view(np.uint32)), k
    assert np.isfinite(with_n["nrm"]).all() and np.abs(with_n["nrm"]).max() > 0
    none = with_n["hits"] == 0  # the background: written, and zero
    assert none.sum() > 1000 and np.array_equal(with_n["nrm"][none], np.zeros((int(none.sum()), 3), np.float32))


@pytest.mark.parametrize("replay", [True, False])
@pytest.mark.parametrize("prim", ["instances", "icosahedron"])
def test_backward_after_a_normals_forward_is_the_plain_backward(prim, replay):
    """The normals forward records the plain forward's hit lists under the plain forward's key: the SH backward replays them (two launches:
    the replay and the re-trace of overflowed rays) exactly when it replays the plain forward's.  The gradients are the same up to the
    order of the backward's float atomics, which differs from launch to launch of the same backward."""
    sc = scenes.scene_c2(n=40_000, width=160, height=128)
    ro, rd = sc.rays()
    g = _Gpu(sc.particles, sc.sph, np.asarray(sc.camera(2, 10), np.float32), ro, rd, 4, prim)
    g.ctx.set_replay(replay)
    rng = np.random.default_rng(5)
    grads = (rng.normal(size=(g.R, 3)).astype(np.float32), rng.normal(size=g.R).astype(np.float32),
             (0.1 * rng.normal(size=g.R)).astype(np.float32))
    g.forward(normals=False)
    dp0, ds0, launches0 = g.backward(grads)
    g.forward(normals=True)
    dp1, ds1, launches1 = g.backward(grads)
    assert launches0 == launches1 == (2 if replay else 1)
    assert np.abs(dp0).max() > 0
    for a, b in ((dp1, dp0), (ds1, ds0)):
        assert rel_l2(a, b) <= 1e-5


class _Gaussians:
    def __init__(self, sc, device):
        p = torch.from_numpy(sc.particles).to(device)
        self.positions = p[:, 0:3].clone().requires_grad_(True)
        self.density = p[:, 3:4].clone().requires_grad_(True)
        self.rotation = p[:, 4:8].clone().requires_grad_(True)
        self.scale = p[:, 8:11].clone().requires_grad_(True)
        self._sph = torch.from_numpy(sc.sph).to(device).requires_grad_(True)
        self.n_active_features = sc.sph_degree
        self.rotation_activation = self.scale_activation = self.density_activation = lambda t: t

    def get_rotation(self):
        return self.rotation

    def get_scale(self):
        return self.scale

    def get_density(self):
        return self.density

    def get_features(self):
        return self._sph

    def grads(self):
        return [t.grad.detach().cpu().numpy() for t in (self.positions, self.density, self.rotation, self.scale, self._sph)]


class _Batch:
    def __init__(self, sc, c2w, device):
        ro, rd = sc.rays()
        self.rays_ori, self.rays_dir = torch.from_numpy(ro).to(device), torch.from_numpy(rd).to(device)
        self.T_to_world = torch.from_numpy(np.asarray(c2w, np.float32))[None].to(device)


@pytest.mark.parametrize("prim", ["instances", "icosahedron"])
def test_tracer_render_pred_normals_and_their_missing_gradient(prim):
    """pred_normals = the raw sums normalised (unit where a hit was accepted, zero elsewhere); a loss on them adds no gradient."""
    import threedgrt_tracer

    dev = torch.device("cuda", 0)
    sc = scenes.scene_c1(width=96, height=80)
    c2w = np.asarray(sc.camera(1, 10), np.float32)
    batch = _Batch(sc, c2w, dev)
    d_rgb = torch.from_numpy(np.random.default_rng(2).normal(size=(1, sc.height, sc.width, 3)).astype(np.float32)).to(dev)
    runs = {}
    for normals in (False, True):
        tr = threedgrt_tracer.Tracer({"render": {"min_transmittance": MIN_T, "primitive_type": prim, "enable_normals": normals}})
        g = _Gaussians(sc, dev)
        tr.build_acc(g, rebuild=True)
        out = tr.render(g, batch, train=True)
        loss = (out["pred_features"] * d_rgb).sum()
        if normals:
            loss = loss + (out["pred_normals"] * d_rgb.flip(-1)).sum()
        loss.backward()
        torch.cuda.synchronize()
        runs[normals] = (out, g.grads())
    out = runs[True][0]
    nrm = out["pred_normals"][0].detach().cpu().numpy()
    length = np.linalg.norm(nrm.astype(np.float64), axis=-1)
    hit = out["hits_count"][0, ..., 0].detach().cpu().numpy() > 0
    assert hit.mean() > 0.2
    assert np.abs(length[hit] - 1).max() <= 1e-5 and np.array_equal(length[~hit], np.zeros((~hit).sum()))
    assert float(runs[False][0]["pred_normals"].abs().max()) == 0  # the key off: zeros, as before
    for a, b in zip(runs[True][1], runs[False][1]):
        assert rel_l2(a, b) <= 1e-5


LRS = dict(positions=2e-3, density=0.05, rotation=1e-3, scale=5e-3, features_albedo=1e-2, features_specular=5e-4)


def _no_normals_entry(monkeypatch):
    import b200_native as nat

    def refuse(*a, **k):
        raise AssertionError("a training step traced normals")

    monkeypatch.setattr(nat.GrtContext, "trace_normals", refuse)


def test_grt_train_step_ignores_the_normals_key(monkeypatch):
    """The step's loss reads no normals, so the key changes nothing: the step never calls the normals forward, launches the same kernels and
    ends with the same parameters (up to the order of the backward's float atomics)."""
    import train_step_grt

    _no_normals_entry(monkeypatch)
    dev = torch.device("cuda", 0)
    sc = scenes.scene_c1(n=600, width=96, height=96)
    ro, rd = sc.rays()
    rays_o, rays_d = torch.from_numpy(ro).to(dev), torch.from_numpy(rd).to(dev)
    P, S = torch.from_numpy(sc.particles).to(dev), torch.from_numpy(sc.sph).to(dev)
    poses = [torch.from_numpy(np.asarray(sc.camera(i, 6), np.float32))[None] for i in range(6)]
    target = (torch.rand((96, 96, 3), device=dev, generator=torch.Generator(device=dev).manual_seed(3)) * 0.8).contiguous()
    ends = {}
    for normals in (False, True):
        step = train_step_grt.GaussianTrainStepGRT(raw_params(P, S), LRS, conf={"render": {"enable_normals": normals}})
        for i in range(3):
            step.step(rays_o, rays_d, poses[i], target)
        torch.cuda.synchronize()
        ends[normals] = ({k: v.detach().cpu().numpy() for k, v in step.params.items()}, step.tracer.tracer_wrapper.native_context(dev).launch_count())
    assert ends[True][1] == ends[False][1]
    for k, v in ends[False][0].items():
        assert rel_l2(ends[True][0][k], v) <= 1e-5, k


def test_hybrid_train_step_steps_with_the_normals_key(monkeypatch):
    import train_step_hybrid as th
    from test_hybrid_train_step_gpu import _setup

    _no_normals_entry(monkeypatch)
    sc, rays_o, rays_d, P, S, poses, sensor = _setup()
    step = th.GaussianTrainStepHybrid(raw_params(P, S), LRS, conf={"render": {"enable_normals": True}})
    target = (torch.rand((sc.height, sc.width, 3), device=P.device, generator=torch.Generator(device=P.device).manual_seed(3)) * 0.8).contiguous()
    before = step.params["positions"].detach().clone()
    losses = [float(step.step(rays_o, rays_d, sensor, poses[1], target)) for _ in range(2)]
    assert all(np.isfinite(losses)) and not torch.equal(before, step.params["positions"])

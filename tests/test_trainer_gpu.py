"""The training loop on the GPU: it is only sequencing (its parameters equal a hand-written step loop over the same view stream), a resume
continues the run, and whole runs on small synthetic folders write every artefact and learn the scene.  The folders are rendered from a
C1-like scene by the repository's own renderer and written into tmp_path."""
from __future__ import annotations

import json
import os

import numpy as np
import pytest
import torch

import scenes
import scene_data
import step_config
import trainer
from scene_fixtures import rotmat_to_qvec, run_conf, write_colmap, write_nerf, write_png

pytestmark = pytest.mark.gpu

W = H = 64


def _truth_step(sc):
    from train_step import GaussianTrainStep, raw_params

    params = raw_params(torch.from_numpy(sc.particles).cuda(), torch.from_numpy(sc.sph).cuda())
    return GaussianTrainStep(params, {k: 0.0 for k in params}, sph_degree=3)


def _render_u8(truth, c2w, fx):
    ro, rd = scenes.pinhole_rays(H, W, fx, fx, W / 2, H / 2)
    pose = scenes.pose7_from_c2w(c2w)
    import threedgut_tracer.tracer as tr

    sensor = tr.fromOpenCVPinholeCameraModelParameters([W, H], tr.ShutterType.GLOBAL, [W / 2, H / 2], [fx, fx], np.zeros(6), np.zeros(2), np.zeros(4))
    rgba = truth.render(torch.from_numpy(ro).cuda(), torch.from_numpy(rd).cuda(), sensor, pose)[0]
    return (rgba[..., :3].clamp(0, 1) * 255).round().byte().cpu().numpy()


@pytest.fixture(scope="module")
def nerf_folder(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("nerf"))
    sc = scenes.scene_c1(n=1000, width=W, height=H)
    truth = _truth_step(sc)
    frames = {}
    for split, n, off in (("train", 16, 0.0), ("val", 2, 0.31), ("test", 4, 0.57)):
        rows = []
        for i in range(n):
            c2w = scenes.orbit_c2w(i + off, n, sc.camera_radius)
            img = _render_u8(truth, c2w, sc.fx)
            nerf_c2w = c2w.copy()
            nerf_c2w[:, 1:3] *= -1
            rows.append((nerf_c2w, img, None))
        frames[split] = rows
    write_nerf(root, frames, camera_angle_x=0.6911112070083618)
    return root


@pytest.fixture(scope="module")
def colmap_folder(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("colmap"))
    sc = scenes.scene_c1(n=1000, width=W, height=H)
    truth = _truth_step(sc)
    images = []
    for i in range(16):
        c2w = scenes.orbit_c2w(i, 16, sc.camera_radius)
        w2c = np.linalg.inv(c2w)
        name = f"img_{i:03d}.png"
        images.append(dict(id=i + 1, qvec=rotmat_to_qvec(w2c[:3, :3]), tvec=w2c[:3, 3], camera_id=1, name=name, xys=np.zeros((0, 2)),
                           point3D_ids=np.zeros(0, np.int64)))
        write_png(os.path.join(root, "images", name), _render_u8(truth, c2w, sc.fx))
    rng = np.random.default_rng(5)
    pts = sc.particles[rng.choice(sc.n, 400, replace=False), :3].astype(np.float64)
    write_colmap(root, {1: ("PINHOLE", W, H, [sc.fx, sc.fx, W / 2, H / 2])}, images, binary=True,
                 points=(pts, rng.integers(0, 256, (400, 3), dtype=np.uint8)))
    return root


def _record(monkeypatch):
    """Patch build_step so that every step it builds keeps a copy of its initial parameters and logs what each `step` call receives:
    (frame, the view's pose bytes, the target's bytes, whether a mask was given)."""
    built = []
    real = step_config.build_step

    def build(*a, **k):
        step = real(*a, **k)
        step.initial = {g: step.params[g].clone() for g in step.GROUPS}
        step.calls = []
        inner = step.step

        def logged(*args, **kw):
            view, target = args[:-1], args[-1]
            pose = view[-1].numpy() if torch.is_tensor(view[-1]) else np.asarray(view[-1])
            step.calls.append((step.frame, pose.tobytes(), target.cpu().numpy().tobytes(), kw.get("mask") is not None))
            return inner(*args, **kw)

        step.step = logged
        built.append(step)
        return step

    monkeypatch.setattr(step_config, "build_step", build)
    monkeypatch.setattr(trainer.step_config, "build_step", build)
    return built


def _manual(conf, k):
    """K steps of step.step by hand on the view stream of `conf` (what train() must reduce to)."""
    scene = scene_data.SceneData(conf)
    method = conf["render"]["method"]
    step = step_config.build_step(conf, trainer.initial_params(conf, scene, torch.device("cuda")), scene.scene_extent)
    stream = trainer.ViewStream(len(scene.train), conf["seed_initialization"])
    for s in range(k):
        i = stream[s]
        step.step(*scene.train.view(i, method), scene.train.target(i), mask=scene.train.mask(i))
    torch.cuda.synchronize()
    return step


# The steps do not repeat bit for bit from run to run (their gradient sums use atomics; densification then amplifies the differences
# into different clone / split decisions), so the loop is checked by what it hands the step: the same starting parameters, bit for bit,
# and the same (frame, view, target, mask) at every step as a hand-written loop over the same view stream.
@pytest.mark.parametrize("kind", ["3dgut_gs", "3dgrt_mcmc"])
def test_loop_is_only_sequencing(nerf_folder, colmap_folder, tmp_path, monkeypatch, kind):
    method, strategy = kind.split("_")
    folder, dataset = (nerf_folder, "nerf") if method == "3dgut" else (colmap_folder, "colmap")
    k = 24
    conf = run_conf(folder, str(tmp_path), dataset=dataset, method=method, strategy=strategy, n_iterations=k, test_last=False,
                 checkpoint={"iterations": []}, export_ply={"enabled": False, "path": ""})
    built = _record(monkeypatch)
    out = trainer.train(conf)
    manual = _manual(conf, k)
    loop = out["step"]
    assert built == [loop, manual]
    assert all(torch.equal(loop.initial[g], manual.initial[g]) for g in loop.GROUPS)
    assert len(loop.calls) == k and loop.calls == manual.calls
    if strategy == "gs":
        assert out["n_gaussians"] != 2000, "densification did not change the number of Gaussians"


def _clone(x):
    if torch.is_tensor(x):
        return x.detach().clone()
    if isinstance(x, dict):
        return {k: _clone(v) for k, v in x.items()}
    return x


def _equal(a, b, where=""):
    """Bit-for-bit equality of nested dicts / lists of tensors and plain values; the first difference is named."""
    if torch.is_tensor(a) or torch.is_tensor(b):
        a, b = torch.as_tensor(a).cpu(), torch.as_tensor(b).cpu()
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), where
    elif isinstance(a, dict):
        assert set(a) == set(b), (where, sorted(a), sorted(b))
        for k in a:
            _equal(a[k], b[k], f"{where}.{k}")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _equal(x, y, f"{where}[{i}]")
    else:
        assert a == b, (where, a, b)


def test_resume_continues_the_run(nerf_folder, tmp_path, monkeypatch):
    import checkpoint as ck

    k = 12
    built = _record(monkeypatch)
    saved_states, loaded_states = {}, []
    real_save, real_load = ck.save, ck.load

    def save(step, path, **kw):  # what the run held when it wrote each checkpoint
        saved_states[os.path.basename(path)] = _clone(step.state_dict())
        return real_save(step, path, **kw)

    def load(path, step, **kw):  # what the resumed run holds right after loading, before its first step
        out = real_load(path, step, **kw)
        loaded_states.append(_clone(step.state_dict()))
        return out

    monkeypatch.setattr(trainer.checkpoint, "save", save)
    monkeypatch.setattr(trainer.checkpoint, "load", load)
    off = {"test_last": False, "export_ply": {"enabled": False, "path": ""}}
    full = trainer.train(run_conf(nerf_folder, str(tmp_path / "a"), n_iterations=2 * k, checkpoint={"iterations": [k]}, **off))
    ckpt = os.path.join(full["run_dir"], f"ours_{k}", f"ckpt_{k}.pt")
    resumed = trainer.train(run_conf(nerf_folder, str(tmp_path / "c"), n_iterations=2 * k, resume=ckpt, checkpoint={"iterations": []},
                                     **off))
    assert resumed["global_step"] == 2 * k and len(built) == 2 and len(loaded_states) == 1
    # the resumed step holds, bit for bit, what the first run held at step k: parameters, both moments and the Adam counts, frame, rates,
    # SH degree, the densifier's gradient statistics and generator, and the schedule
    _equal(loaded_states[0], saved_states[f"ckpt_{k}.pt"], "state")
    assert built[1].calls == built[0].calls[k:]  # then the same views, frames and targets from step k on, with no sampler state


# (settings, least test-PSNR gain in dB over the initial Gaussians).  Measured on an H100 80GB HBM3 (700 W) over 200 steps: nerf_3dgut_gs
# 8.40 -> 10.80 dB (2000 random Gaussians), colmap_3dgrt_mcmc 2.68 -> 9.29 dB, colmap_3dgut_mcmc_nht 9.62 -> 18.87 dB; each bar is about
# half the measured gain
RUNS = {"nerf_3dgut_gs": (dict(dataset="nerf", method="3dgut", strategy="gs", feature_type="sh"), 1.0),
        "colmap_3dgrt_mcmc": (dict(dataset="colmap", method="3dgrt", strategy="mcmc", feature_type="sh"), 5.0),
        "colmap_3dgut_mcmc_nht": (dict(dataset="colmap", method="3dgut", strategy="mcmc", feature_type="nht"), 4.0)}


@pytest.mark.parametrize("name", list(RUNS))
def test_whole_run_writes_everything_and_learns(nerf_folder, colmap_folder, tmp_path, name):
    import evaluate

    kw, min_gain = RUNS[name]
    n = 200
    conf = run_conf(nerf_folder if kw["dataset"] == "nerf" else colmap_folder, str(tmp_path), n_iterations=n, **kw)
    scene = scene_data.SceneData(conf)
    init = step_config.build_step(conf, trainer.initial_params(conf, scene, torch.device("cuda")), scene.scene_extent)
    psnr0 = evaluate.evaluate(init, scene.test.views(conf["render"]["method"]))["mean_psnr"]
    out = trainer.train(conf, scene=scene)
    d = out["run_dir"]
    files = ["parsed.yaml", f"ours_{n // 2}/ckpt_{n // 2}.pt", "ckpt_last.pt", "metrics.json", f"ours_{n}/renders/00000.png", "train_log.jsonl"]
    files += ["export_last.ply"] if kw["feature_type"] == "sh" else []
    for f in files:
        assert os.path.isfile(os.path.join(d, f)), f
    with open(os.path.join(d, "metrics.json")) as f:
        psnr = json.load(f)["mean_psnr"]
    print(f"{name}: test PSNR {psnr0:.2f} -> {psnr:.2f} dB")
    with open(os.path.join(d, "train_log.jsonl")) as f:
        rows = [json.loads(ln) for ln in f]
    assert [r["step"] for r in rows] == list(range(0, n, 10))
    assert psnr > psnr0 + min_gain, (psnr0, psnr)

"""Whole-run training throughput: trainer.train() against a bare step.step loop over the same view stream, in one process.

Writes a C2-like NeRF-synthetic folder (100 training views at 800x800 rendered from scenes.scene_c2, plus 2 val and 4 test views) into a
temporary directory, then, for the GS and the MCMC strategy of nerf_synthetic_3dgut-like settings (100k random initial Gaussians, L1 +
SSIM, configs/strategy/*.yaml), times K steps of train() (validation, checkpoints and test off, log_frequency 100) and K steps of the
bare loop, `--repeats` pairs in alternating order.  K defaults to 1500, so that the strategies (which start at step 500) densify, prune,
relocate and add inside the timed window.  Reports steps/s of each, the loop's median overhead per step beside the range of each, and
from a separate bare run the per-phase device time (phase_events), the densifier's per-step gradient buffer on its own, the number of
steps on which the strategy changed the Gaussians, the dataset start-up time, and the card (benchkit.card).  One JSON line.

    python scripts/bench_train.py --steps 1500 --repeats 4
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time

import benchkit

sys.path.insert(0, os.path.join(benchkit.ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import scenes  # noqa: E402
import scene_data  # noqa: E402
import step_config  # noqa: E402
import trainer  # noqa: E402
from scene_fixtures import run_conf, write_nerf  # noqa: E402


def write_scene(root, views=100):
    from train_step import GaussianTrainStep, raw_params

    sc = scenes.scene_c2()
    params = raw_params(torch.from_numpy(sc.particles).cuda(), torch.from_numpy(sc.sph).cuda())
    truth = GaussianTrainStep(params, {k: 0.0 for k in params}, sph_degree=3)
    ro, rd = (torch.from_numpy(a).cuda() for a in scenes.pinhole_rays(sc.height, sc.width, sc.fx, sc.fy, sc.cx, sc.cy))
    sensor = sc.pinhole_sensor()
    frames = {}
    for split, n, off in (("train", views, 0.0), ("val", 2, 0.31), ("test", 4, 0.57)):
        rows = []
        for i in range(n):
            c2w = scenes.orbit_c2w(i + off, n, sc.camera_radius)
            rgba = truth.render(ro, rd, sensor, scenes.pose7_from_c2w(c2w))[0]
            img = torch.cat([rgba[..., :3] / rgba[..., 3:].clamp_min(1e-6), rgba[..., 3:]], -1).clamp(0, 1)
            nerf = c2w.copy()
            nerf[:, 1:3] *= -1
            rows.append((nerf, (img * 255).round().byte().cpu().numpy(), None))
        frames[split] = rows
    write_nerf(root, frames, camera_angle_x=0.6911112070083618)


def conf_for(root, out_dir, strategy, steps):
    c = run_conf(root, out_dir, strategy=strategy, n_iterations=steps, test_last=False, checkpoint={"iterations": []},
              export_ply={"enabled": False, "path": ""}, log_frequency=100)
    c["initialization"]["num_gaussians"] = 100_000
    c["model"]["progressive_training"]["increase_frequency"] = 1000
    c["strategy"] = {  # configs/strategy/{gs,mcmc}.yaml
        "gs": {"method": "GSStrategy", "densify": {"params": "positions", "frequency": 300, "start_iteration": 500, "end_iteration": 15000,
                                                   "clone_grad_threshold": 0.0002, "split_grad_threshold": 0.0002, "relative_size_threshold": 0.01,
                                                   "split": {"n_gaussians": 2}},
               "prune": {"frequency": 100, "start_iteration": 500, "end_iteration": 15000, "density_threshold": 0.005},
               "reset_density": {"frequency": 3000, "start_iteration": 0, "end_iteration": 15000, "new_max_density": 0.01},
               "density_decay": {"start_iteration": -1}, "prune_weight": {"start_iteration": -1}, "prune_scale": {"start_iteration": -1}},
        "mcmc": {"method": "MCMCStrategy", "binom_n_max": 51, "opacity_threshold": 0.005,
                 "relocate": {"start_iteration": 500, "end_iteration": 25000, "frequency": 100},
                 "add": {"start_iteration": 500, "end_iteration": 25000, "frequency": 100, "max_n_gaussians": 1000000},
                 "perturb": {"start_iteration": 0, "end_iteration": 27500, "frequency": 1, "noise_lr": 500000.0}}}[strategy]
    return c


def bare(conf, scene, steps, phases=False):
    """steps/s of a bare step.step loop over the run's view stream; with phases, also the per-phase device time (phase_events), the
    device and host time of the densifier's per-step gradient buffer (update_gradient_buffer, GS), and the number of steps on which the
    strategy changed the Gaussians."""
    method = conf["render"]["method"]
    step = step_config.build_step(conf, trainer.initial_params(conf, scene, torch.device("cuda")), scene.scene_extent)
    stream = trainer.ViewStream(len(scene.train), conf["seed_initialization"])
    views = [scene.train.view(i, method) for i in range(len(scene.train))]
    grad_buffer = []
    if phases:
        step.phase_events = []
        if hasattr(step.densifier, "update_gradient_buffer"):
            inner = step.densifier.update_gradient_buffer

            def timed(*a, **k):
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                t = time.perf_counter()
                inner(*a, **k)
                grad_buffer.append((start, end, time.perf_counter() - t))
                end.record()

            step.densifier.update_gradient_buffer = timed
    torch.cuda.synchronize()
    t = time.perf_counter()
    changes, n = 0, step.n
    for s in range(steps):
        i = stream[s]
        step.step(*views[i], scene.train.target(i), mask=scene.train.mask(i))
        if phases and step.n != n:
            changes, n = changes + 1, step.n
    torch.cuda.synchronize()
    elapsed = time.perf_counter() - t
    if not phases:
        return steps / elapsed, None
    ev = step.phase_events
    per = {}
    for (_, a), (name, b) in zip(ev[:-1], ev[1:]):
        per[name] = per.get(name, 0.0) + a.elapsed_time(b)
    total = sum(per.values())
    out = {"share": {k: round(v / total, 4) for k, v in per.items()}, "steps_changing_n": changes, "n_gaussians_end": step.n,
           "densify_phase_ms_per_step": round(per.get("densify", 0.0) / steps, 4)}
    if grad_buffer:
        out["update_gradient_buffer"] = {"device_ms_per_step": round(sum(s.elapsed_time(e) for s, e, _ in grad_buffer) / len(grad_buffer), 4),
                                         "host_ms_per_step": round(1e3 * sum(h for _, _, h in grad_buffer) / len(grad_buffer), 4),
                                         "share_of_step_device_time": round(sum(s.elapsed_time(e) for s, e, _ in grad_buffer) / total, 4)}
    return steps / elapsed, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1500, help="timed steps per window (the shipped strategies start at step 500)")
    ap.add_argument("--repeats", type=int, default=4, help="(train(), bare loop) pairs, their order alternating")
    ap.add_argument("--views", type=int, default=100)
    args = ap.parse_args()
    result = {"card": benchkit.card(benchkit.cuda_device("bench_train.py")), "steps": args.steps, "repeats": args.repeats}
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "c2")
        t = time.perf_counter()
        write_scene(root, args.views)
        result["scene_write_s"] = round(time.perf_counter() - t, 2)
        for strategy in ("gs", "mcmc"):
            conf = conf_for(root, os.path.join(tmp, "runs"), strategy, args.steps)
            t = time.perf_counter()
            scene = scene_data.SceneData(conf)
            torch.cuda.synchronize()
            startup = time.perf_counter() - t
            bare(conf, scene, 20)  # warm-up of every shape
            loop, plain = [], []
            for r in range(args.repeats):  # the order alternates, so neither loop always runs first
                for which in (("train", "bare") if r % 2 == 0 else ("bare", "train")):
                    if which == "train":
                        loop.append(trainer.train(conf, scene=scene)["steps_per_s"])
                    else:
                        plain.append(bare(conf, scene, args.steps)[0])
            _, phases = bare(conf, scene, args.steps, phases=True)
            ms = lambda r: 1e3 / np.asarray(r)  # noqa: E731
            result[strategy] = {"train_steps_per_s": [round(v, 2) for v in loop], "bare_steps_per_s": [round(v, 2) for v in plain],
                                "overhead_ms_per_step_median": round(float(np.median(ms(loop)) - np.median(ms(plain))), 4),
                                "train_ms_per_step_range": [round(float(v), 4) for v in (ms(loop).min(), ms(loop).max())],
                                "bare_ms_per_step_range": [round(float(v), 4) for v in (ms(plain).min(), ms(plain).max())],
                                "phases": phases, "dataset_startup_s": round(startup, 2)}
    print(json.dumps(result))


if __name__ == "__main__":
    main()

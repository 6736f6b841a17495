"""Train a scene from disk: the reference's Trainer3DGRUT (threedgrut/trainer.py:116-410, 941-1084, 1119-1440) over this repository's
fused training steps.

    python 3dgrut_b200/trainer.py --config-dir <reference>/configs --config-name apps/nerf_synthetic_3dgut.yaml path=<scene> out_dir=runs
    python 3dgrut_b200/trainer.py --config <run>/parsed.yaml n_iterations=7000

Under torchrun the CLI initialises NCCL and trains view-parallel: each rank renders one view of every step.

The loop is sequencing only: the dataset (scene_data), the start (initialization.initialize, a `resume` checkpoint or an `import_ply`
file), the step (step_config.build_step), validation and test (evaluate), checkpoints (checkpoint.save) and the PLY export.  A step that
validates, checkpoints and logs nothing adds one uint8 -> float conversion of its target to the training step, and no host
synchronisation, host -> device copy or allocation: step losses stay on the device and are read back in one transfer every
max(log_frequency, 100) steps.

View order is stateless, so that a resume needs no sampler state: the stream of training views is the concatenation of per-epoch
permutations, one torch.randperm per epoch from a CPU generator seeded by (seed_initialization, epoch), and global step s on rank r of g
takes stream element s * g + r."""
from __future__ import annotations

import argparse
import json
import os
import time
from datetime import datetime
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

import checkpoint
import config as config_mod
import evaluate
import initialization
import scene_data
import step_config
from b200_native import cfg_get

LOG_FLUSH_MIN = 100


# ---- the view stream -----------------------------------------------------------------------------------------------------------------

def epoch_permutation(n_views: int, seed: int, epoch: int) -> torch.Tensor:
    """The order of the training views in `epoch`: torch.randperm(n_views) from a CPU generator seeded by (seed, epoch)."""
    g = torch.Generator().manual_seed(((int(seed) & 0xFFFFFFFF) << 31 | int(epoch)) & 0x7FFFFFFFFFFFFFFF)
    return torch.randperm(int(n_views), generator=g)


class ViewStream:
    """Stream element e is epoch_permutation(n, seed, e // n)[e % n]; `step_views(s, g)` are the g views of global step s, rank order."""

    def __init__(self, n_views: int, seed: int):
        if n_views <= 0:
            raise ValueError("the training split has no views")
        self.n, self.seed, self._perm = int(n_views), int(seed), {}

    def __getitem__(self, e: int) -> int:
        epoch = e // self.n
        if epoch not in self._perm:
            self._perm = {epoch: epoch_permutation(self.n, self.seed, epoch).tolist()}  # only the current epoch is kept
        return self._perm[epoch][e % self.n]

    def step_views(self, s: int, world: int = 1) -> list:
        return [self[s * world + r] for r in range(world)]


# ---- PLY -----------------------------------------------------------------------------------------------------------------------------

def ply_attributes(n_albedo: int = 3, n_specular: int = initialization.SPECULAR_DIM) -> list:
    """The vertex properties in the reference's order (export/formats/ply.py:42-56)."""
    return (["x", "y", "z", "nx", "ny", "nz"] + [f"f_dc_{i}" for i in range(n_albedo)] + [f"f_rest_{i}" for i in range(n_specular)]
            + ["opacity"] + [f"scale_{i}" for i in range(3)] + [f"rot_{i}" for i in range(4)])


def export_ply(params: dict, path: str) -> None:
    """The SH parameters as a binary little-endian 3DGS PLY (export/formats/ply.py:58-91): pre-activation values, normals (0,0,1),
    f_rest channel-major.  The inverse of initialization.read_gaussian_ply."""
    host = {k: params[k].detach().float().cpu().numpy() for k in ("positions", "density", "rotation", "scale", "features_albedo",
                                                                    "features_specular")}
    n = host["positions"].shape[0]
    spec = host["features_specular"].reshape(n, -1, 3).transpose(0, 2, 1).reshape(n, -1)
    names = ply_attributes(host["features_albedo"].shape[1], spec.shape[1])
    table = np.concatenate([host["positions"], np.repeat(np.float32([[0, 0, 1]]), n, 0), host["features_albedo"], spec, host["density"],
                            host["scale"], host["rotation"]], axis=1).astype("<f4")
    header = "ply\nformat binary_little_endian 1.0\n" + f"element vertex {n}\n" + "".join(f"property float {a}\n" for a in names) + "end_header\n"
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path, "wb") as f:
        f.write(header.encode("ascii"))
        f.write(np.ascontiguousarray(table).tobytes())


# ---- the run -------------------------------------------------------------------------------------------------------------------------

def check_train_config(conf) -> None:
    """Every refusal of a run (NotImplementedError naming the key), before any image is read."""
    step_config.check_config(conf)
    if str(cfg_get(conf, "model.feature_type", "sh")).lower() == "nht":
        if bool(cfg_get(conf, "export_ply.enabled", False)):
            raise NotImplementedError("export_ply.enabled=true with model.feature_type='nht': the PLY layout holds SH coefficients")
        if bool(cfg_get(conf, "import_ply.enabled", False)):
            raise NotImplementedError("import_ply.enabled=true with model.feature_type='nht': the PLY layout holds SH coefficients")


def run_dir(conf, group=None) -> str:
    """{out_dir}/{experiment_name}/{stem(path)}-{%d%m_%H%M%S} (utils/misc.py:151-160), named by rank 0."""
    name = [os.path.join(str(cfg_get(conf, "out_dir", "./runs")), str(cfg_get(conf, "experiment_name", "") or ""),
                         f"{Path(str(cfg_get(conf, 'path', ''))).stem}-{datetime.now().strftime('%d%m_%H%M%S')}")]
    if dist.is_available() and dist.is_initialized():
        dist.broadcast_object_list(name, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
    return name[0]


def _start_params(conf, scene, device):
    """(params, first global step, checkpoint path to resume or None)."""
    resume = str(cfg_get(conf, "resume", "") or "")
    if resume:
        ckpt = torch.load(resume, map_location=device, weights_only=False)
        ft = str(cfg_get(conf, "model.feature_type", "sh")).lower()
        params = checkpoint.from_reference_layout(ckpt, feature_type=ft)["params"]
        return {k: v.detach().to(device=device, dtype=torch.float32).clone().contiguous() for k, v in params.items()}, None, resume
    if bool(cfg_get(conf, "import_ply.enabled", False)):
        g = initialization.read_gaussian_ply(str(cfg_get(conf, "import_ply.path", "")))
        params = {k: torch.from_numpy(v).to(device).contiguous() for k, v in g.items()}
        return params, int(cfg_get(conf, "import_ply.init_global_step", 0)), None
    return initial_params(conf, scene, device), None, None


def initial_params(conf, scene, device) -> dict:
    """initialization.initialize on the scene, with torch's generators seeded seed_initialization first: the `random` method draws from
    the default generator, and every rank must draw the same Gaussians."""
    torch.manual_seed(int(cfg_get(conf, "seed_initialization", 42)))
    return initialization.initialize(conf, observers=scene.observer_points, points_transform=scene.points_transform, device=device)


def sensor_positions(step, split, method: str) -> np.ndarray:
    """[F,3] float32 world positions of every frame's sensor, as the step computes its own view's."""
    out = []
    for i in range(len(split)):
        view = split.view(i, method)
        if method == "3dgrt":
            out.append(step.sensor_position(view[2]))
        else:
            cam = split.cameras[split.camera_of[i]]
            out.append(step.raster.sensor_position(view[2], view[3], view[3], cam.width, cam.height))
    return np.stack(out).astype(np.float32)


def train(conf: dict, group=None, device=None, scene=None) -> dict:
    """Train the run `conf` describes (config.load's dict); every rank of `group` calls it.  scene: a loaded scene_data.SceneData to reuse
    (default: read from conf.path).  Returns {"run_dir", "step" (the trained step), "global_step", "n_gaussians", "validation" [(step,
    means)], "test" (evaluate's metrics dict or None), "startup_s" (dataset read), "train_s" (the loop, synchronised), "steps_per_s"}."""
    check_train_config(conf)
    world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
    rank = dist.get_rank(group) if world > 1 else 0
    device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    method = str(cfg_get(conf, "render.method", "3dgut")).lower()

    t0 = time.perf_counter()
    if scene is None:
        scene = scene_data.SceneData(conf, device)
    startup = time.perf_counter() - t0
    out_dir = run_dir(conf, group)
    if rank == 0:
        os.makedirs(out_dir, exist_ok=True)
        import yaml

        with open(os.path.join(out_dir, "parsed.yaml"), "w") as f:
            yaml.safe_dump(conf, f, sort_keys=False)

    params, first, resume = _start_params(conf, scene, device)
    step = step_config.build_step(conf, params, scene.scene_extent, group=group)
    if resume:
        checkpoint.load(resume, step)
    elif first:
        step.frame = first
        if step.schedule is not None:
            lrs, step.sph_degree = step.schedule.advance_to(first).initial_lrs(), step.schedule.sph_degree
            step.optimizer.lrs.update(lrs)

    train_split = scene.train
    stream = ViewStream(len(train_split), int(cfg_get(conf, "seed_initialization", 42)))
    positions = sensor_positions(step, train_split, method)
    views = [train_split.view(i, method) for i in range(len(train_split))]
    n_iterations = int(cfg_get(conf, "n_iterations", 30000))
    val_frequency = int(cfg_get(conf, "val_frequency", 5000))
    validate_first = bool(cfg_get(conf, "validate_first", False))
    ckpt_steps = {int(s) for s in (cfg_get(conf, "checkpoint.iterations", []) or [])}
    log_frequency = max(int(cfg_get(conf, "log_frequency", 1)), 1)
    flush_every = max(log_frequency, LOG_FLUSH_MIN)
    loss_log = torch.zeros(flush_every // log_frequency + 1, dtype=torch.float32, device=device)
    pending = []  # (global step, slot, n_gaussians, lrs) of the logged steps since the last read-back
    log_path = os.path.join(out_dir, "train_log.jsonl")
    validation = []

    def flush():
        if not pending:
            return
        host = loss_log.cpu().numpy()  # the one read-back of the logged losses
        if rank == 0:
            with open(log_path, "a") as f:
                for s, slot, n, lrs in pending:
                    f.write(json.dumps({"step": s, "loss": float(host[slot]), "n_gaussians": n, "lrs": lrs}) + "\n")
        pending.clear()

    torch.cuda.synchronize(device)
    t_loop = time.perf_counter()
    s0 = step.frame
    while step.frame < n_iterations:
        s = step.frame
        if (s > 0 or validate_first) and s % val_frequency == 0:
            validation.append((s, evaluate.validate(step, scene.val.views(method, device))["mean"]))
        idx = stream.step_views(s, world)
        i = idx[rank]
        loss = step.step(*views[i], train_split.target(i), all_sensor_positions=positions[idx] if world > 1 else None,
                         mask=train_split.mask(i))
        if s % log_frequency == 0:
            slot = len(pending)
            loss_log[slot].copy_(loss)
            pending.append((s, slot, step.n, dict(step.optimizer.lrs)))
        if (s + 1) % flush_every == 0:
            flush()
        if step.frame in ckpt_steps:
            flush()
            os.makedirs(os.path.join(out_dir, f"ours_{step.frame}"), exist_ok=True)
            checkpoint.save(step, os.path.join(out_dir, f"ours_{step.frame}", f"ckpt_{step.frame}.pt"), conf=conf,
                            epoch=(step.frame * world) // len(train_split))
    flush()
    torch.cuda.synchronize(device)
    train_s = time.perf_counter() - t_loop
    checkpoint.save(step, os.path.join(out_dir, "ckpt_last.pt"), conf=conf, epoch=(step.frame * world) // len(train_split))
    test = None
    if rank == 0 and bool(cfg_get(conf, "test_last", True)):
        test = evaluate.evaluate(step, scene.test.views(method, device), out_dir=out_dir, save_gt=False)["metrics"]
    if rank == 0 and bool(cfg_get(conf, "export_ply.enabled", False)):
        export_ply(step.params, str(cfg_get(conf, "export_ply.path", "") or "") or os.path.join(out_dir, "export_last.ply"))
    done = step.frame - s0
    return {"run_dir": out_dir, "step": step, "global_step": step.frame, "n_gaussians": step.n, "validation": validation, "test": test,
            "startup_s": startup, "train_s": train_s, "steps_per_s": done / train_s if train_s > 0 else float("nan")}


# ---- CLI -----------------------------------------------------------------------------------------------------------------------------

def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--config-dir", help="the reference's configs/ directory")
    ap.add_argument("--config-name", help="a config under --config-dir, e.g. apps/nerf_synthetic_3dgut.yaml")
    ap.add_argument("--config", help="one YAML file, e.g. a run's parsed.yaml")
    ap.add_argument("overrides", nargs="*", help="key=value or +key=value")
    args = ap.parse_args(argv)
    conf = config_mod.load(config_dir=args.config_dir, config_name=args.config_name, config_file=args.config, overrides=args.overrides)
    check_train_config(conf)
    distributed = int(os.environ.get("WORLD_SIZE", "1")) > 1
    if distributed:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        dist.init_process_group("nccl")
    try:
        out = train(conf)
        if not distributed or dist.get_rank() == 0:
            print(json.dumps({k: out[k] for k in ("run_dir", "global_step", "n_gaussians", "test", "startup_s", "train_s", "steps_per_s")}))
    finally:
        if distributed:
            dist.destroy_process_group()


if __name__ == "__main__":
    main()

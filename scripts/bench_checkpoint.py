"""Save and load wall time, file size and peak extra device memory of checkpoint.save / checkpoint.load for a 3DGUT training step
(train_step.GaussianTrainStep, GS densification, random background) at C2 (300k Gaussians) and C3 (6M).

    python scripts/bench_checkpoint.py [--sizes 300000,6000000] [--reps 3] [--dir DIR]

The step's parameters and both Adam moments are 3 x 59 floats per Gaussian (about 4.2 GB at C3).  Save is timed from a synchronised
device to the file renamed into place; load from the call to the step holding the state, synchronised.  Peak extra device memory is
torch.cuda.max_memory_allocated during the call over what was allocated before it (the loading step is built at 1,000 Gaussians, so what
it replaces is negligible).  The files go to --dir (default: the system's temporary directory) and are deleted at the end; the
filesystem and its device are printed, since the disk dominates.  A load right after a save may read the file from the page cache: the
load times are those of a warm cache, not of a cold disk."""
from __future__ import annotations

import argparse
import os
import tempfile
import time

import numpy as np

import benchkit

LRS = dict(positions=2e-3, density=0.05, rotation=1e-3, scale=5e-3, features_albedo=2.5e-3, features_specular=1.25e-4)


def _filesystem(path: str) -> str:
    """The mount holding `path` (device, mount point, type) from /proc/mounts."""
    path, best = os.path.realpath(path), ("?", "", "?")
    try:
        with open("/proc/mounts") as f:
            for line in f:
                dev, mnt, fstype = line.split()[:3]
                if (path == mnt or path.startswith(mnt.rstrip("/") + "/")) and len(mnt) >= len(best[1]):
                    best = (dev, mnt, fstype)
    except OSError:
        pass
    return f"{best[0]} on {best[1] or '?'} ({best[2]})"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--sizes", default="300000,6000000", help="Gaussians per run, comma-separated")
    ap.add_argument("--reps", type=int, default=3, help="saves and loads per size")
    ap.add_argument("--dir", default=tempfile.gettempdir(), help="directory the checkpoints are written to")
    args = ap.parse_args()

    import torch

    import checkpoint
    import densify
    import train_step

    dev = benchkit.cuda_device("bench_checkpoint.py")
    print(f"device: {benchkit.card(dev)}")
    print(f"checkpoint directory: {args.dir} on {_filesystem(args.dir)}")
    workdir = tempfile.mkdtemp(prefix="bench_checkpoint_", dir=args.dir)

    def make(n, seed):
        g = torch.Generator(device=dev).manual_seed(seed)
        widths = dict(positions=3, density=1, rotation=4, scale=3, features_albedo=3, features_specular=45)
        raw = {k: torch.randn((n, w), device=dev, generator=g) for k, w in widths.items()}
        return train_step.GaussianTrainStep(raw, LRS, densify_conf=densify.DensifyConfig(), background="random")

    try:
        for n in [int(s) for s in args.sizes.split(",")]:
            a = make(n, 0)
            for k in a.GROUPS:  # trained-like moments and counts
                a.optimizer.exp_avg[k].normal_()
                a.optimizer.exp_avg_sq[k].uniform_()
            a.optimizer.steps = a.frame = 1000
            a.densifier.grad_norm_accum.uniform_()
            state_bytes = sum(t.numel() * 4 for k in a.GROUPS for t in (a.params[k], a.optimizer.exp_avg[k], a.optimizer.exp_avg_sq[k]))
            path = os.path.join(workdir, "ckpt.pt")
            saves, loads, peaks = [], [], []
            for _ in range(args.reps):
                torch.cuda.synchronize(dev)
                base = torch.cuda.memory_allocated(dev)
                torch.cuda.reset_peak_memory_stats(dev)
                t0 = time.perf_counter()
                checkpoint.save(a, path)
                saves.append(time.perf_counter() - t0)
                save_peak = torch.cuda.max_memory_allocated(dev) - base
                b = make(1000, 1)
                torch.cuda.synchronize(dev)
                base = torch.cuda.memory_allocated(dev)
                torch.cuda.reset_peak_memory_stats(dev)
                t0 = time.perf_counter()
                checkpoint.load(path, b)
                torch.cuda.synchronize(dev)
                loads.append(time.perf_counter() - t0)
                peaks.append(torch.cuda.max_memory_allocated(dev) - base)
                assert b.n == n and all(torch.equal(b.params[k], a.params[k]) and torch.equal(b.optimizer.exp_avg_sq[k], a.optimizer.exp_avg_sq[k])
                                        for k in a.GROUPS), "the loaded state differs from the saved one"
                del b
                torch.cuda.empty_cache()
            size = os.path.getsize(path)
            s, ld = np.array(saves), np.array(loads)
            print(f"N={n}: state (parameters + moments) {state_bytes / 1e9:.3f} GB, file {size / 1e9:.3f} GB; "
                  f"save {np.median(s):.2f} s ({s.min():.2f}-{s.max():.2f}, {size / np.median(s) / 1e9:.2f} GB/s, peak extra device memory "
                  f"{save_peak / 1e9:.3f} GB); load {np.median(ld):.2f} s ({ld.min():.2f}-{ld.max():.2f}, {size / np.median(ld) / 1e9:.2f} GB/s); "
                  f"peak extra device memory on load {max(peaks) / 1e9:.3f} GB = {max(peaks) / state_bytes:.2f} x the state; {args.reps} reps")
            os.remove(path)
            del a
            torch.cuda.empty_cache()
    finally:
        for f in os.listdir(workdir):
            os.remove(os.path.join(workdir, f))
        os.rmdir(workdir)


if __name__ == "__main__":
    main()

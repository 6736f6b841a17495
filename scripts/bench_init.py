"""Time the exact k-nearest-neighbour search (initialization.nearest_neighbors) and the whole initialisation from points
(initialization.from_points) on the GPU, beside the CPU KD-tree the reference uses for the same points in the same run.

    python scripts/bench_init.py [--sizes 100000,1000000,6000000] [--reps 5] [--cpu-6m]

Workloads: self k = 1 (the `random` initialisation's nearest other point) and k = 3 (the 3 nearest other points of `fused_point_cloud` and
`use_observation_points: false`) on uniform points in [-1.5, 1.5]^3 and on C3-like clouds (70 % within radius 3, 30 % out to radius 50),
and the 1-NN of 1M C3-like points to 300 and to 10,000 observers.  GPU times are CUDA events around the call, after one warm-up call, the
median of --reps.  The CPU column is scikit-learn's KDTree.query(k=2) / NearestNeighbors(n_neighbors=4) when scikit-learn is installed,
else scipy's cKDTree with as many neighbours (marked), one run, on this host's CPUs; at 6M points it is skipped unless --cpu-6m, since it
takes minutes."""
from __future__ import annotations

import argparse
import os
import time

import numpy as np

import benchkit


def _cloud(kind: str, n: int, seed: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    if kind == "uniform":
        return rng.uniform(-1.5, 1.5, (n, 3)).astype(np.float32)
    n_in = int(0.7 * n)
    dirs = rng.normal(size=(n, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    rad = np.concatenate([3.0 * rng.uniform(0, 1, n_in) ** 0.5, rng.uniform(3.0, 50.0, n - n_in)])
    pos = dirs * rad[:, None]
    pos[:, 2] *= 0.35
    return pos.astype(np.float32)


def _cuda_ms(fn, reps: int) -> float:
    import torch

    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times))


def _cpu_ms(points: np.ndarray, k: int, targets: np.ndarray | None) -> tuple[float, str]:
    """One CPU KD-tree query as the reference runs it: self k (+1 for the point itself) or 1-NN to the targets."""
    try:
        import sklearn.neighbors as skn

        t0 = time.perf_counter()
        if targets is not None:
            skn.KDTree(targets).query(points, k=1)
        elif k == 1:
            skn.KDTree(points).query(points, k=2)
        else:
            skn.NearestNeighbors(n_neighbors=k + 1, metric="euclidean").fit(points).kneighbors(points)
        return (time.perf_counter() - t0) * 1e3, "sklearn"
    except ImportError:
        from scipy.spatial import cKDTree

        t0 = time.perf_counter()
        if targets is not None:
            cKDTree(targets).query(points, k=1, workers=-1)
        else:
            cKDTree(points).query(points, k=k + 1, workers=-1)
        return (time.perf_counter() - t0) * 1e3, "scipy"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--sizes", default="100000,1000000,6000000", help="points per self-search workload, comma-separated")
    ap.add_argument("--reps", type=int, default=5, help="timed GPU calls per workload (median)")
    ap.add_argument("--cpu-6m", action="store_true", help="also time the CPU KD-tree at 6M points (minutes)")
    args = ap.parse_args()

    import torch

    import initialization as I

    dev = benchkit.cuda_device("bench_init.py")
    print(f"device: {benchkit.card(dev)}  CPU threads: {os.cpu_count()}  torch {torch.__version__}")
    conf_pts = {"initialization": {"use_observation_points": False}}
    print(f"{'workload':<34} {'N':>9} {'knn ms':>9} {'from_points ms':>15} {'CPU KD-tree ms':>16}")
    for kind in ("uniform", "c3_like"):
        for n in (int(s) for s in args.sizes.split(",")):
            pts_np = _cloud(kind, n)
            pts = torch.from_numpy(pts_np).to(dev)
            for k in (1, 3):
                knn = _cuda_ms(lambda: I.nearest_neighbors(pts, k), args.reps)
                init = _cuda_ms(lambda: I.from_points(pts, None, None, conf_pts), args.reps) if k == 3 else float("nan")
                if n >= 6_000_000 and not args.cpu_6m:
                    cpu, src = float("nan"), "skipped"
                else:
                    cpu, src = _cpu_ms(pts_np, k, None)
                name = f"{kind} self k={k}"
                print(f"{name:<34} {n:>9} {knn:>9.2f} {init:>15.2f} {cpu:>12.0f} ({src})", flush=True)
            del pts
            torch.cuda.empty_cache()
    pts_np = _cloud("c3_like", 1_000_000, seed=1)
    pts = torch.from_numpy(pts_np).to(dev)
    for m in (300, 10_000):
        obs_np = np.random.default_rng(2).uniform(-10, 10, (m, 3)).astype(np.float32)
        obs = torch.from_numpy(obs_np).to(dev)
        knn = _cuda_ms(lambda: I.nearest_neighbors(pts, 1, targets=obs), args.reps)
        init = _cuda_ms(lambda: I.from_points(pts, None, obs, {"initialization": {"use_observation_points": True}}), args.reps)
        cpu, src = _cpu_ms(pts_np, 1, obs_np)
        name = f"c3_like 1-NN to {m} observers"
        print(f"{name:<34} {1_000_000:>9} {knn:>9.2f} {init:>15.2f} {cpu:>12.0f} ({src})", flush=True)


if __name__ == "__main__":
    main()

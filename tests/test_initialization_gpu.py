"""initialization.py on the GPU: the exact k-nearest-neighbour search against scipy's cKDTree in float64 on seeded clouds that break
grids and naive trees (far outliers, dense cores, duplicates, planes, lines, tiny sets, separate observer sets, C3 at 6M); the
initialisations against the torch restatement of the reference (tests/init_oracle.py); and their output through three training steps."""
import numpy as np
import pytest

import init_oracle as oracle
import scenes

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
from scipy.spatial import cKDTree  # noqa: E402

DEV = "cuda:0"


def _check(points, k, targets=None, rows=None):
    """points [N,3] float32 numpy; targets [M,3] or None (self); rows: the query rows checked (None: all)."""
    import initialization as I

    P = torch.from_numpy(np.ascontiguousarray(points, np.float32)).to(DEV)
    T = None if targets is None else torch.from_numpy(np.ascontiguousarray(targets, np.float32)).to(DEV)
    d, idx = I.nearest_neighbors(P, k, targets=T)
    d2, idx2 = I.nearest_neighbors(P, k, targets=T)
    assert torch.equal(d, d2) and torch.equal(idx, idx2), "two calls differ"
    d, idx = d.cpu().numpy(), idx.cpu().numpy()
    p64 = P.cpu().numpy().astype(np.float64)
    t64 = p64 if T is None else T.cpu().numpy().astype(np.float64)
    rows = np.arange(len(p64)) if rows is None else rows
    d, idx = d[rows], idx[rows]
    extra = 1 if T is None else 0
    kq = min(k + 1 + extra, len(t64))  # one rank beyond k, where there is one, for the gap after rank k-1
    od, oi = cKDTree(t64).query(p64[rows], k=kq)
    od, oi = od.reshape(len(rows), kq), oi.reshape(len(rows), kq)
    if T is None:  # drop the query itself, or the last column when duplicates pushed it out
        keep = oi != rows[:, None]
        keep[keep.sum(1) == kq, -1] = False
        od, oi = od[keep].reshape(len(rows), kq - 1), oi[keep].reshape(len(rows), kq - 1)
    assert (np.diff(d, axis=1) >= 0).all(), "a row is not ascending"
    if T is None:
        assert (idx != rows[:, None]).all(), "a row holds its own index"
    mine = np.linalg.norm(p64[rows][:, None, :] - t64[idx], axis=-1)
    assert (mine <= od[:, :k] * (1 + 2.0 ** -20)).all(), f"farther than the oracle: {np.max(mine - od[:, :k])}"
    # where the oracle's ranks are separated by more than 1e-6 relative, the index is determined
    gap = lambda a, b: (b - a) > 1e-6 * np.maximum(b, 1e-30)  # noqa: E731
    sure = np.ones((len(rows), k), bool)
    for r in range(k):
        if r > 0:
            sure[:, r] &= gap(od[:, r - 1], od[:, r])
        if r + 1 < od.shape[1]:
            sure[:, r] &= gap(od[:, r], od[:, r + 1])
    assert (idx[sure] == oi[:, :k][sure]).all(), f"{int((idx[sure] != oi[:, :k][sure]).sum())} determined indices differ"


def _c3_like(n, seed):
    rng = np.random.default_rng(seed)
    n_in = int(0.7 * n)
    dirs = rng.normal(size=(n, 3))
    dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
    rad = np.concatenate([3.0 * rng.uniform(0, 1, n_in) ** 0.5, rng.uniform(3.0, 50.0, n - n_in)])
    pos = dirs * rad[:, None]
    pos[:, 2] *= 0.35
    return pos.astype(np.float32)


def _clouds():
    rng = np.random.default_rng(0)
    dup_base = rng.uniform(-1, 1, (20_000, 3))
    dup = np.repeat(dup_base, rng.integers(1, 6, len(dup_base)), axis=0)
    dup = dup[rng.permutation(len(dup))]
    core = np.concatenate([rng.uniform(0, 1e-3, (99_000, 3)), rng.uniform(-500, 500, (1_000, 3))])
    plane = np.concatenate([rng.uniform(-2, 2, (50_000, 2)), np.zeros((50_000, 1))], 1)
    grid = np.stack(np.meshgrid(np.arange(60), np.arange(60), [3.0], indexing="ij"), -1).reshape(-1, 3)  # coplanar, tied distances
    t = rng.uniform(-5, 5, 30_000)
    line = np.stack([t, 2 * t + 1, -t], 1)
    return {"uniform_100k": rng.uniform(-1.5, 1.5, (100_000, 3)), "c2_300k": scenes.scene_c2().particles[:, :3],
            "c3_like_1m": _c3_like(1_000_000, 1), "core_and_outliers": core, "duplicates": dup, "coplanar": plane,
            "coplanar_grid": grid[rng.permutation(len(grid))], "collinear": line}


CLOUDS = ("uniform_100k", "c2_300k", "c3_like_1m", "core_and_outliers", "duplicates", "coplanar", "coplanar_grid", "collinear")


@pytest.fixture(scope="module")
def clouds():
    return _clouds()


@pytest.mark.parametrize("name", CLOUDS)
def test_knn_matches_the_kd_tree(clouds, name):
    for k in (1, 3) if name in ("c2_300k", "c3_like_1m") else (1, 2, 3, 4):
        _check(clouds[name], k)


def test_knn_tiny_sets():
    rng = np.random.default_rng(4)
    for n in range(2, 6):
        pts = rng.normal(size=(n, 3))
        for k in range(1, min(n - 1, 4) + 1):
            _check(pts, k)
            _check(np.zeros((n, 3)), k)  # all duplicates: every neighbour at 0, any other index


def test_knn_to_a_separate_target_set():
    rng = np.random.default_rng(5)
    q = _c3_like(100_000, 6)
    for m in (1, 7, 300, 10_000):
        obs = rng.uniform(-10, 10, (m, 3)).astype(np.float32)
        for k in (1, 4) if m >= 4 else (1,):
            _check(q, k, targets=obs)


def test_knn_c3_full_scale():
    pos = scenes.scene_c3().particles[:, :3]
    rows = np.sort(np.random.default_rng(7).choice(len(pos), 20_000, replace=False))
    for k in (1, 3):
        _check(pos, k, rows=rows)


def test_knn_refuses_non_finite_points():
    import initialization as I

    p = torch.zeros((10, 3), device=DEV)
    p[3, 1] = float("inf")
    with pytest.raises(ValueError, match="non-finite"):
        I.nearest_neighbors(p, 1)
    with pytest.raises(ValueError, match="k=5"):
        I.nearest_neighbors(torch.rand((10, 3), device=DEV), 5)


# ---- the initialisations against the restatement of the reference ----------------------------------------------------------------------

def _conf(nht, use_obs, seed=42, **model):
    conf = {"seed_initialization": seed, "initialization": {"use_observation_points": use_obs, "observation_scale_factor": 0.01},
            "model": {"default_density": 0.5, "default_scale_factor": 0.1, "feature_type": "nht" if nht else "sh", **model}}
    if nht:
        conf["model"]["nht_features"] = {"dim": 48, "init_min": -1.5707963267948966, "init_max": 1.5707963267948966}
    return conf


def _compare(got, want, nb_mine, nb_oracle):
    assert set(got) == set(want)
    for k in want:
        assert got[k].dtype == torch.float32 and got[k].is_contiguous() and got[k].device == want[k].device, k
        if k != "scale":
            assert torch.equal(got[k], want[k].float()), k
    same = (nb_mine == nb_oracle).all(dim=1)
    assert torch.equal(got["scale"][same], want["scale"][same])
    ulp = torch.abs(torch.nextafter(want["scale"], torch.full_like(want["scale"], float("inf"))) - want["scale"])
    assert (torch.abs(got["scale"] - want["scale"]) <= ulp).all()
    return int((~same).sum())


@pytest.mark.parametrize("nht", [False, True])
@pytest.mark.parametrize("use_obs", [False, True])
@pytest.mark.parametrize("colours", [False, True])
def test_from_points_matches_the_reference(nht, use_obs, colours):
    import initialization as I

    rng = np.random.default_rng(8)
    pts = torch.from_numpy(_c3_like(30_000, 9)).to(DEV)
    obs = torch.from_numpy(rng.uniform(-20, 20, (300, 3)).astype(np.float32)).to(DEV)
    rgb = torch.from_numpy(rng.integers(0, 256, (30_000, 3)).astype(np.uint8)).to(DEV) if colours else None
    conf = _conf(nht, use_obs)
    got = I.from_points(pts, rgb, obs, conf)
    nht_kw = dict(nht=nht, init_min=-1.5707963267948966, init_max=1.5707963267948966)
    want, nb = oracle.from_points(pts, obs, rgb, use_obs, 42, 0.01, 0.1, 0.5, **nht_kw)
    if use_obs:
        _, mine = I.nearest_neighbors(pts, 1, targets=obs)
    else:
        _, mine = I.nearest_neighbors(pts, 3)
    _compare(got, want, mine, nb)


@pytest.mark.parametrize("nht", [False, True])
def test_random_point_cloud_matches_the_reference(nht):
    import initialization as I

    conf = _conf(nht, False)
    torch.manual_seed(123)
    got = I.random_point_cloud(20_000, -1.5, 1.5, conf=conf, device=DEV)
    torch.manual_seed(123)
    want, nb = oracle.random_point_cloud(20_000, -1.5, 1.5, 0.1, 0.5, nht=nht, init_min=-1.5707963267948966, init_max=1.5707963267948966,
                                         device=DEV)
    _, mine = I.nearest_neighbors(got["positions"], 1)
    assert _compare(got, want, mine, nb) == 0  # uniform points: no near ties, so every scale is bit-identical too


def test_lidar_and_fused_colours_are_seeded(tmp_path):
    """A cloud without colours draws them from numpy's RandomState(seed_initialization), so two calls agree; lidar subsamples with the
    reference's randperm before initialising."""
    import initialization as I
    from test_initialization import write_ply

    pts = _c3_like(5_000, 10).astype(np.float64)
    write_ply(tmp_path / "fused.ply", "binary_little_endian", [("float", "x"), ("float", "y"), ("float", "z")], pts)
    conf = _conf(False, False)
    conf["initialization"].update(method="fused_point_cloud", fused_point_cloud_path=str(tmp_path / "fused.ply"))
    a, b = I.initialize(conf, device=DEV), I.initialize(conf, device=DEV)
    assert all(torch.equal(a[k], b[k]) for k in a)
    rgb = np.random.RandomState(42).randint(0, 256, size=(5_000, 3), dtype=np.uint8)
    want = I.from_points(torch.tensor(pts.astype(np.float32), device=DEV), torch.tensor(rgb, device=DEV), None, conf)
    assert all(torch.equal(a[k], want[k]) for k in a)
    lidar = _conf(False, True)
    lidar["initialization"].update(method="lidar", num_points=1_000)
    obs = np.zeros((1, 3), np.float32)
    got = I.initialize(lidar, observers=obs, point_cloud=(torch.from_numpy(pts.astype(np.float32)), torch.from_numpy(rgb)), device=DEV)
    keep = torch.randperm(5_000, generator=torch.Generator().manual_seed(42))[:1_000]
    assert torch.equal(got["positions"].cpu(), torch.from_numpy(pts.astype(np.float32))[keep])


# ---- through the steps -----------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["gut", "grt", "gut_nht"])
def test_initialized_params_train(kind, tmp_path):
    """initialize(...) builds each step as it comes; three steps on a C1-size view have finite losses, and the state converts to the
    reference's checkpoint layout."""
    import checkpoint
    import initialization as I
    from test_initialization import _cloud, write_points3d_bin
    from test_schedule_step_gpu import LRS_NHT, LRS_SH, _Run

    nht = kind.endswith("nht")
    run = _Run(kind)
    if nht:
        conf = _conf(True, False)
        conf["initialization"].update(method="random", num_gaussians=1_000)
        params = I.initialize(conf, device=run.dev)
    else:
        xyz, rgb, tracks = _cloud(1_000)
        (tmp_path / "sparse" / "0").mkdir(parents=True)
        write_points3d_bin(tmp_path / "sparse" / "0" / "points3D.bin", xyz * 0.1, rgb, tracks)
        conf = _conf(False, True)
        conf.update(path=str(tmp_path))
        conf["initialization"]["method"] = "colmap"
        params = I.initialize(conf, observers=np.array([[0, 0, 4.0], [4.0, 0, 0]], np.float32), device=run.dev)
    st = run.make(params, LRS_NHT if nht else LRS_SH)
    for v in range(3):
        loss = run.step(st, v)
        assert torch.isfinite(torch.as_tensor(loss)).all(), (kind, v)
    ckpt = checkpoint.reference_layout(st.state_dict())
    assert ckpt["positions"].shape == (1_000, 3)

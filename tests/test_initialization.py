"""initialization.py without a GPU: the k-nearest-neighbour entry points are declared, exported and bound; the COLMAP, PLY and 3DGS PLY
readers read back what is written here; the points transform; every configuration refusal names its key; the lidar subsample; the
checkpoint method returns the stored parameters."""
import os
import struct

import numpy as np
import pytest
import torch

from helpers import declared

NEW = ("gutb200_knn", "gutb200_knn_workspace_bytes")


def test_knn_entry_points_are_exported():
    import b200_native as nat

    lib = nat.load()
    for name in NEW:
        assert name in declared("gut_b200.h") and name in nat.EXPORTS, name
        assert hasattr(lib, name) and getattr(lib, name).argtypes is not None, name
    # the workspace needs no device; it grows with the targets and is 0 outside 1..INT32_MAX
    assert 0 < lib.gutb200_knn_workspace_bytes(10) < lib.gutb200_knn_workspace_bytes(100_000)
    assert lib.gutb200_knn_workspace_bytes(0) == 0 and lib.gutb200_knn_workspace_bytes(2**31) == 0


@pytest.mark.parametrize("k, n, self_, msg", [(0, 10, True, "k=0"), (5, 10, True, "k=5"), (3, 3, True, "n_targets=3 < 4"),
                                              (3, 2, False, "n_targets=2 < 3"), (1, 2**31, False, "INT32_MAX")])
def test_knn_refusals_name_the_argument(k, n, self_, msg):
    """The argument checks run before any device work: NULL pointers with a bad argument return 1 and name it."""
    import b200_native as nat

    lib = nat.load()
    q = None if self_ else 8
    rc = lib.gutb200_knn(None, n, 8, n if self_ else 4, q, k, 8, 1 << 40, 8, None)
    assert rc == 1 and msg in lib.gutb200_last_error(None).decode()
    rc = lib.gutb200_knn(None, 100, 8, 100, None, 2, 8, 16, 8, None)
    assert rc == 1 and "workspace_bytes=16" in lib.gutb200_last_error(None).decode()


# ---- COLMAP -----------------------------------------------------------------------------------------------------------------------------

def _cloud(n=257, seed=3):
    rng = np.random.default_rng(seed)
    xyz = rng.normal(size=(n, 3)) * 10.0
    rgb = rng.integers(0, 256, (n, 3)).astype(np.uint8)
    tracks = rng.integers(0, 6, n)
    tracks[:3] = 0
    return xyz, rgb, tracks


def write_points3d_bin(path, xyz, rgb, tracks):
    with open(path, "wb") as f:
        f.write(struct.pack("<Q", len(xyz)))
        for i in range(len(xyz)):
            f.write(struct.pack("<QdddBBBd", i + 1, *xyz[i], *[int(c) for c in rgb[i]], 0.5))
            f.write(struct.pack("<Q", int(tracks[i])))
            f.write(struct.pack("<" + "ii" * int(tracks[i]), *range(2 * int(tracks[i]))))


def write_points3d_txt(path, xyz, rgb, tracks):
    with open(path, "w") as f:
        f.write("# 3D point list with one line of data per point:\n#   POINT3D_ID, X, Y, Z, R, G, B, ERROR, TRACK[]\n")
        for i in range(len(xyz)):
            tr = " ".join(f"{j} {j + 1}" for j in range(int(tracks[i])))
            f.write(f"{i + 1} {float(xyz[i, 0])!r} {float(xyz[i, 1])!r} {float(xyz[i, 2])!r} {rgb[i, 0]} {rgb[i, 1]} {rgb[i, 2]} 0.25 {tr}\n")
            if i == 5:
                f.write("# a comment between points\n\n")


def test_colmap_bin_and_txt_read_back(tmp_path):
    import initialization as I

    xyz, rgb, tracks = _cloud()
    write_points3d_bin(tmp_path / "points3D.bin", xyz, rgb, tracks)
    write_points3d_txt(tmp_path / "points3D.txt", xyz, rgb, tracks)
    for reader, name in ((I.read_colmap_points3d_bin, "points3D.bin"), (I.read_colmap_points3d_txt, "points3D.txt")):
        got_xyz, got_rgb = reader(str(tmp_path / name))
        assert got_xyz.dtype == np.float64 and got_rgb.dtype == np.uint8
        np.testing.assert_array_equal(got_xyz, xyz)
        np.testing.assert_array_equal(got_rgb, rgb)
    with open(tmp_path / "points3D.bin", "r+b") as f:  # a truncated file raises
        f.truncate(os.path.getsize(tmp_path / "points3D.bin") - 4)
    with pytest.raises(ValueError, match="truncated"):
        I.read_colmap_points3d_bin(str(tmp_path / "points3D.bin"))


def test_colmap_paths(tmp_path, monkeypatch):
    """bin before txt under sparse/0; scannetpp reads colmap/points3D.txt; the points are transformed before from_points."""
    import initialization as I

    xyz, rgb, tracks = _cloud(40)
    (tmp_path / "sparse" / "0").mkdir(parents=True)
    (tmp_path / "colmap").mkdir()
    write_points3d_txt(tmp_path / "sparse" / "0" / "points3D.txt", xyz, rgb, tracks)
    write_points3d_txt(tmp_path / "colmap" / "points3D.txt", xyz[:20], rgb[:20], tracks[:20])
    seen = []
    monkeypatch.setattr(I, "_device", lambda device: torch.device("cpu"))
    monkeypatch.setattr(I, "from_points", lambda pts, colors, obs, conf, use_observer_pts: seen.append((pts, colors, use_observer_pts)))
    T = np.diag([2.0, 2.0, 2.0, 1.0])
    T[:3, 3] = [1, 2, 3]
    conf = {"path": str(tmp_path), "initialization": {"method": "colmap", "use_observation_points": False}}
    I.initialize(conf, points_transform=T)
    want = torch.tensor(xyz, dtype=torch.float32)
    torch.testing.assert_close(seen[-1][0], want @ torch.tensor(T[:3, :3], dtype=torch.float32).T + torch.tensor(T[:3, 3], dtype=torch.float32),
                               rtol=0, atol=0)
    assert torch.equal(seen[-1][1].cpu(), torch.from_numpy(rgb)) and seen[-1][2] is False
    write_points3d_bin(tmp_path / "sparse" / "0" / "points3D.bin", xyz[:30], rgb[:30], tracks[:30])
    I.initialize(conf)
    assert seen[-1][0].shape[0] == 30
    I.initialize({**conf, "dataset": {"type": "scannetpp"}})
    assert seen[-1][0].shape[0] == 20


# ---- PLY --------------------------------------------------------------------------------------------------------------------------------

def write_ply(path, fmt, props, values, extra_element=True, endian="<"):
    """props: [(ply type, name)], values: [N, len(props)] (float64 holding every column).  extra_element: a face element with a list
    property before the vertices and a one-property element after them."""
    np_type = {"float": "f4", "double": "f8", "uchar": "u1", "int": "i4"}
    n = len(values)
    head = ["ply", f"format {fmt} 1.0", "comment written by the test"]
    if extra_element:
        head += ["element face 2", "property list uchar int vertex_indices"]
    head += [f"element vertex {n}"] + [f"property {t} {name}" for t, name in props]
    if extra_element:
        head += ["element extra 1", "property float w"]
    head.append("end_header")
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode())
        if fmt == "ascii":
            if extra_element:
                f.write(b"3 0 1 2\n4 0 1 2 3\n")
            for row in values:
                f.write((" ".join(repr(float(v)) if t in ("float", "double") else str(int(v)) for (t, _), v in zip(props, row)) + "\n").encode())
            if extra_element:
                f.write(b"0.5\n")
        else:
            if extra_element:
                f.write(struct.pack(endian + "Biii", 3, 0, 1, 2) + struct.pack(endian + "Biiii", 4, 0, 1, 2, 3))
            rec = np.zeros(n, dtype=[(name, endian + np_type[t]) for t, name in props])
            for j, (_, name) in enumerate(props):
                rec[name] = values[:, j]
            f.write(rec.tobytes())
            if extra_element:
                f.write(struct.pack(endian + "f", 0.5))


@pytest.mark.parametrize("fmt", ["ascii", "binary_little_endian"])
@pytest.mark.parametrize("colour", [True, False])
@pytest.mark.parametrize("xyz_type", ["float", "double"])
def test_ply_reader(tmp_path, fmt, colour, xyz_type):
    import initialization as I

    rng = np.random.default_rng(1)
    n = 50
    xyz = rng.normal(size=(n, 3)).astype(np.float32 if xyz_type == "float" else np.float64)
    rgb = rng.integers(0, 256, (n, 3))
    props = [(xyz_type, "x"), (xyz_type, "y"), (xyz_type, "z"), ("float", "nx"), ("float", "ny"), ("float", "nz"), ("double", "quality")]
    cols = [xyz.astype(np.float64), rng.normal(size=(n, 3)).astype(np.float32).astype(np.float64), rng.normal(size=(n, 1))]
    if colour:
        props += [("uchar", "red"), ("uchar", "green"), ("uchar", "blue")]
        cols.append(rgb.astype(np.float64))
    write_ply(tmp_path / "c.ply", fmt, props, np.concatenate(cols, 1))
    got_xyz, got_rgb = I.read_ply_points(str(tmp_path / "c.ply"))
    np.testing.assert_array_equal(got_xyz, xyz.astype(np.float32))
    if colour:
        np.testing.assert_array_equal(got_rgb, rgb.astype(np.uint8))
    else:
        assert got_rgb is None


def test_ply_refuses_other_formats(tmp_path):
    import initialization as I

    write_ply(tmp_path / "be.ply", "binary_big_endian", [("float", "x"), ("float", "y"), ("float", "z")], np.ones((3, 3)), endian=">")
    with pytest.raises(ValueError, match="binary_big_endian"):
        I.read_ply_points(str(tmp_path / "be.ply"))


def test_gaussian_ply_reorders_f_rest(tmp_path):
    """f_rest_* is stored channel-major (3 x 15): the params hold it coefficient-major (15 x 3), as init_from_pretrained_point_cloud
    reorders it."""
    import initialization as I

    rng = np.random.default_rng(2)
    n = 7
    names = ["x", "y", "z", "opacity", *(f"rot_{i}" for i in range(4)), *(f"scale_{i}" for i in range(3)), *(f"f_dc_{i}" for i in range(3)),
             *(f"f_rest_{i}" for i in range(45))]
    vals = rng.normal(size=(n, len(names))).astype(np.float32)
    write_ply(tmp_path / "point_cloud.ply", "binary_little_endian", [("float", k) for k in names], vals.astype(np.float64), extra_element=False)
    g = I.read_gaussian_ply(str(tmp_path / "point_cloud.ply"))
    col = {k: vals[:, j] for j, k in enumerate(names)}
    np.testing.assert_array_equal(g["positions"], np.stack([col["x"], col["y"], col["z"]], 1))
    np.testing.assert_array_equal(g["density"][:, 0], col["opacity"])
    rest = np.stack([col[f"f_rest_{i}"] for i in range(45)], 1)
    for c in range(3):
        for j in range(15):
            np.testing.assert_array_equal(g["features_specular"][:, 3 * j + c], rest[:, 15 * c + j])
    write_ply(tmp_path / "bad.ply", "ascii", [("float", k) for k in names[:-1]], vals[:, :-1].astype(np.float64), extra_element=False)
    with pytest.raises(ValueError, match="f_rest_44"):
        I.read_gaussian_ply(str(tmp_path / "bad.ply"))


# ---- transform, refusals, lidar, checkpoint -------------------------------------------------------------------------------------------

def test_points_transform():
    import initialization as I

    g = torch.Generator().manual_seed(0)
    p = torch.randn((100, 3), generator=g)
    T = torch.randn((4, 4), generator=g)
    assert torch.equal(I.apply_points_transform(p, T), p @ T[:3, :3].T + T[:3, 3])
    assert I.apply_points_transform(p, None) is p
    with pytest.raises(ValueError, match="4, 4"):
        I.apply_points_transform(p, torch.eye(3))
    bad = torch.eye(4)
    bad[0, 3] = float("nan")
    with pytest.raises(ValueError, match="finite"):
        I.apply_points_transform(p, bad)
    with pytest.raises(ValueError, match="N, 3"):
        I.apply_points_transform(p[:, :2], torch.eye(4))


@pytest.mark.parametrize("key, value, exc", [
    ("initialization.method", "sfm", ValueError),
    ("model.density_activation", "exp", NotImplementedError),
    ("model.scale_activation", "sigmoid", NotImplementedError),
    ("model.progressive_training.max_n_features", 2, NotImplementedError),
    ("model.nht_features.dim", 32, NotImplementedError),
])
def test_config_refusals_name_their_key(key, value, exc):
    import initialization as I

    conf = {"initialization": {"method": "random"}, "model": {"feature_type": "nht" if key == "model.nht_features.dim" else "sh"}}
    cur = conf
    parts = key.split(".")
    for p in parts[:-1]:
        cur = cur.setdefault(p, {})
    cur[parts[-1]] = value
    with pytest.raises(exc, match=key.replace(".", r"\.")) as err:
        I.initialize(conf, device="cuda:0")
    if key == "initialization.method":
        for m in I.METHODS:
            assert m in str(err.value)


def test_missing_inputs_are_refused():
    import initialization as I

    for method in ("colmap", "lidar"):
        with pytest.raises(ValueError, match="use_observation_points"):
            I.initialize({"initialization": {"method": method, "use_observation_points": True}}, device="cuda:0")
    with pytest.raises(ValueError, match="point_cloud"):
        I.initialize({"initialization": {"method": "lidar", "use_observation_points": False}}, device="cuda:0")
    with pytest.raises(ValueError, match="transform"):
        I.initialize({"initialization": {"method": "point_cloud"}}, points_transform=np.eye(4), device="cuda:0")
    with pytest.raises(ValueError, match="CUDA"):
        I.nearest_neighbors(torch.zeros((4, 3)), 1)


def test_lidar_subsample_is_the_reference_randperm():
    import initialization as I

    keep = I.lidar_subsample(1000, 300, 42)
    assert torch.equal(keep, torch.randperm(1000, generator=torch.Generator().manual_seed(42))[:300])
    assert I.lidar_subsample(300, 300, 42) is None


def test_checkpoint_returns_fresh_leaves(tmp_path, monkeypatch):
    """initialization.method: checkpoint reads the file's parameters only, as copies that share nothing with the file's tensors."""
    import checkpoint
    import initialization as I
    from test_checkpoint import _state

    monkeypatch.setattr(I, "_device", lambda device: torch.device("cpu"))
    for ft in ("sh", "nht"):
        state = _state(ft)
        path = tmp_path / f"ckpt_{ft}.pt"
        torch.save(checkpoint.reference_layout(state), path)
        conf = {"initialization": {"method": "checkpoint", "path": str(path)}, "model": {"feature_type": ft}}
        params = I.initialize(conf)
        assert tuple(params) == checkpoint.groups_of(ft)
        for k, v in params.items():
            assert torch.equal(v, state["params"][k].float()) and v.is_leaf and not v.requires_grad and v.is_contiguous()
            assert v.data_ptr() != state["params"][k].data_ptr()
        with pytest.raises(ValueError, match="feature_type"):
            I.initialize({**conf, "model": {"feature_type": "nht" if ft == "sh" else "sh"}})

"""Training from disk without a GPU: config composition, the NeRF-synthetic and COLMAP readers (poses, intrinsics, splits, extents,
images, masks, rays), the view stream, the PLY writer and the refusals.  Every fixture is written into tmp_path by the test."""
from __future__ import annotations

import os
import re

import numpy as np
import pytest
import torch
import yaml

import config
import initialization
import scene_data
import step_config
import trainer
from scene_fixtures import look_at_w2c, project, rotmat_to_qvec, write_colmap, write_nerf


# ---- configs -----------------------------------------------------------------------------------------------------------------------

def _write_tree(root):
    files = {
        "base.yaml": "defaults:\n  - _self_\n  - /strategy: gs\n  - override hydra/hydra_logging: disabled\n"
                     "path: ???\nn: 10\nname: run\nlr:\n  a: 0.0025\n  b: ${div:${lr.a},20}\n"
                     "checkpoint:\n  iterations: ${int_list:[ 7, 30 ]}\nrender:\n  pipeline_type: ref\n  bwd: ${render.pipeline_type}Bwd\n"
                     "  ref_n: ${n}\nhydra:\n  run:\n    dir: .\n",
        "base_mcmc.yaml": "# @package _global_\ndefaults:\n  - /base\n  - override /strategy: mcmc\n  - _self_\nn: 20\n",
        "strategy/gs.yaml": "method: GSStrategy\nfreq: 300\n",
        "strategy/mcmc.yaml": "method: MCMCStrategy\nfreq: 100\n",
        "dataset/colmap.yaml": "type: colmap\ndownsample_factor: 1\n",
        "render/a.yaml": "method: a\nk: 1\nonly_a: true\n",
        "render/b.yaml": "defaults:\n  - a\n  - _self_\nmethod: b\nk: 2\n",
        "apps/app.yaml": "# @package _global_\ndefaults:\n  - /base_mcmc\n  - /dataset: colmap\n  - /render: b\n  - _self_\n"
                         "dataset:\n  downsample_factor: 4\n",
        "apps/self_first.yaml": "# @package _global_\ndefaults:\n  - _self_\n  - /base\nn: 99\nextra: 1\n",
    }
    for name, text in files.items():
        os.makedirs(os.path.dirname(os.path.join(root, name)) or root, exist_ok=True)
        with open(os.path.join(root, name), "w") as f:
            f.write(text)


def test_config_composition(tmp_path):
    _write_tree(tmp_path)
    c = config.load(str(tmp_path), "apps/app.yaml", overrides=["path=/data/scene", "lr.a=0.01", "+extra.deep=1e-3", "name=42"])
    assert c["strategy"] == {"method": "MCMCStrategy", "freq": 100}      # override /strategy inside the nested base
    assert c["dataset"] == {"type": "colmap", "downsample_factor": 4}     # group package, then the app's own keys
    assert c["render"]["method"] == "b" and c["render"]["k"] == 2 and c["render"]["only_a"] is True  # relative default `a`
    assert c["render"]["bwd"] == "refBwd" and c["render"]["ref_n"] == 20  # concatenation; ${n} after base_mcmc's n
    assert c["lr"]["b"] == pytest.approx(0.01 / 20) and c["checkpoint"]["iterations"] == [7, 30]
    assert c["extra"] == {"deep": 1e-3} and c["name"] == 42 and c["path"] == "/data/scene"
    assert "hydra" not in c and "defaults" not in c
    first = config.load(str(tmp_path), "apps/self_first.yaml")
    assert first["n"] == 10 and first["extra"] == 1                       # _self_ first: the base overrides n
    with pytest.raises(KeyError, match="nope"):
        config.load(str(tmp_path), "apps/app.yaml", overrides=["nope=1"])
    with pytest.raises(KeyError, match="lr.c"):
        config.load(str(tmp_path), "apps/app.yaml", overrides=["lr.c=1"])
    # the same dict from the parsed.yaml a run writes
    path = tmp_path / "parsed.yaml"
    with open(path, "w") as f:
        yaml.safe_dump(c, f, sort_keys=False)
    assert config.load(config_file=str(path)) == c


def test_config_file_unresolved(tmp_path):
    path = tmp_path / "p.yaml"
    path.write_text("a:\n  lr: 0.5\n  half: ${div:${a.lr},2}\nviews: ${int_list:[1, 2]}\ns: x${a.lr}y\n")
    c = config.load(config_file=str(path), overrides=["a.lr=1"])
    assert c == {"a": {"lr": 1, "half": 0.5}, "views": [1, 2], "s": "x1y"}


# ---- NeRF-synthetic -----------------------------------------------------------------------------------------------------------------

def _restated_read(img_u8, bg):
    """dataset_nerf.py __read_image, restated with numpy."""
    img = img_u8.astype(np.float32) / 255.0
    if bg == "black":
        img = img[..., :3] * img[..., -1:]
    elif bg == "white":
        img = img[..., :3] * img[..., -1:] + (1 - img[..., -1:])
    return (img * 255.0).astype(np.uint8)


def _nerf_frames(rng, n, w=12, h=10, masks=False):
    out = []
    for i in range(n):
        eye = rng.normal(size=3) * 0.3 + np.array([3.0 + i, 0.5 * i, 1.0])
        c2w = np.linalg.inv(look_at_w2c(eye)).astype(np.float32)
        c2w[:, 1:3] *= -1  # the file stores right-up-back
        img = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        mask = (rng.uniform(size=(h, w)) * 255).astype(np.uint8) if masks else None
        out.append((c2w, img, mask))
    return out


@pytest.mark.parametrize("bg", ["black", "white"])
@pytest.mark.parametrize("ext, suffix", [(".png", ""), (".png", ".png")])
def test_nerf_reader(tmp_path, bg, ext, suffix):
    rng = np.random.default_rng(0)
    frames = {"train": _nerf_frames(rng, 5, masks=True), "val": _nerf_frames(rng, 2), "test": _nerf_frames(rng, 3)}
    write_nerf(tmp_path, frames, camera_angle_x=0.69, ext=ext, path_suffix=suffix)
    conf = {"path": str(tmp_path), "dataset": {"type": "nerf"}, "model": {"background": {"color": bg}}}
    sc = scene_data.SceneData(conf, load_images=False)
    assert (len(sc.train), len(sc.val), len(sc.test)) == (5, 2, 3)
    cam = sc.train.cameras[0]
    assert cam.params["fx"] == pytest.approx(0.5 * 12 / np.tan(0.5 * 0.69)) and (cam.params["cx"], cam.params["cy"]) == (6.0, 5.0)
    for i, (c2w, img, mask) in enumerate(frames["train"]):
        want = c2w.copy()
        want[:, 1:3] *= -1
        np.testing.assert_array_equal(sc.train.c2w[i], want)
        np.testing.assert_array_equal(scene_data.read_image(sc.train.image_paths[i], bg), _restated_read(img, bg))
        np.testing.assert_array_equal(scene_data.read_mask(sc.train.mask_paths[i]), (mask.astype(np.float32) / 255.0 > 0.5).astype(np.float32))
    centres = sc.train.c2w[:, :3, 3]
    med = np.median(centres, axis=0)
    assert sc.scene_extent == pytest.approx(1.1 * np.median(np.linalg.norm(centres - med, axis=1)))
    np.testing.assert_array_equal(sc.observer_points, centres)
    assert scene_data.read_mask(sc.val.mask_paths[0]) is None


def test_nerf_random_background_is_refused_for_rgba(tmp_path):
    rng = np.random.default_rng(1)
    write_nerf(tmp_path, {"train": _nerf_frames(rng, 1)}, 0.69)
    with pytest.raises(ValueError, match="random"):
        scene_data.read_image(str(tmp_path / "train" / "r_0.png"), "random")


# ---- COLMAP -------------------------------------------------------------------------------------------------------------------------

W_FULL, H_FULL = 64, 48
CAMERAS = {
    "SIMPLE_PINHOLE": [50.0, 31.5, 24.5],
    "PINHOLE": [52.0, 49.0, 32.5, 23.0],
    "SIMPLE_RADIAL": [50.0, 32.0, 24.0, -0.05],
    "RADIAL": [50.0, 31.0, 25.0, -0.04, 0.01],
    "OPENCV": [51.0, 49.5, 32.2, 24.3, -0.06, 0.012, 0.001, -0.0015],
    "FULL_OPENCV": [51.0, 49.5, 32.2, 24.3, -0.06, 0.012, 0.001, -0.0015, 0.002, 0.01, -0.02, 0.003],
    "OPENCV_FISHEYE": [30.0, 30.5, 32.4, 23.6, 0.03, -0.01, 0.002, -0.0005],
}


def _colmap_scene(root, models, factor, binary, n_frames=7, rng=None, names=None):
    rng = rng or np.random.default_rng(3)
    cams = {cid: (m, W_FULL, H_FULL, CAMERAS[m]) for cid, m in zip(range(1, len(models) + 1), models)}
    pts = rng.uniform(-0.6, 0.6, (300, 3))
    images = []
    for i in range(n_frames):
        cid = 1 + i % len(models)
        eye = np.array([3.0 * np.cos(0.7 * i), 3.0 * np.sin(0.7 * i), 0.8 + 0.1 * i])
        w2c = look_at_w2c(eye)
        name = (f"{names[cid - 1]}/" if names else "") + f"img_{i:03d}.png"
        images.append(dict(id=i + 1, qvec=rotmat_to_qvec(w2c[:3, :3]), tvec=w2c[:3, 3], camera_id=cid, name=name, xys=np.zeros((0, 2)),
                           point3D_ids=np.zeros(0, np.int64)))
        uv, ok = colmap_project(cams[cid][0], cams[cid][3], pts @ w2c[:3, :3].T + w2c[:3, 3])
        ok &= (uv[:, 0] > 0) & (uv[:, 0] < W_FULL) & (uv[:, 1] > 0) & (uv[:, 1] < H_FULL)
        images[-1]["xys"], images[-1]["point3D_ids"] = uv[ok], np.where(ok)[0]
        folder = "images" if factor == 1 else f"images_{factor}"
        from scene_fixtures import write_png

        write_png(os.path.join(root, folder, name), rng.integers(0, 256, (H_FULL // factor, W_FULL // factor, 3), dtype=np.uint8))
    write_colmap(root, cams, images, binary=binary)
    return cams, images, pts


def colmap_project(model, params, X):
    """COLMAP's own camera models (colmap/src/colmap/sensor/models.h), in its parameter layout, float64: (pixels [M,2], in front [M]).
    Written independently of the loader, so the stored observations check its mapping of every parameter."""
    p = [float(v) for v in params]
    u, v = X[:, 0] / X[:, 2], X[:, 1] / X[:, 2]
    if model in ("SIMPLE_PINHOLE", "SIMPLE_RADIAL", "RADIAL"):
        fx = fy = p[0]
        cx, cy, extra = p[1], p[2], p[3:]
    else:
        fx, fy, cx, cy, extra = p[0], p[1], p[2], p[3], p[4:]
    r2 = u * u + v * v
    if model == "SIMPLE_RADIAL":
        radial = extra[0] * r2
        u, v = u + u * radial, v + v * radial
    elif model == "RADIAL":
        radial = extra[0] * r2 + extra[1] * r2 * r2
        u, v = u + u * radial, v + v * radial
    elif model == "OPENCV":
        k1, k2, p1, p2 = extra
        radial = k1 * r2 + k2 * r2 * r2
        u, v = (u + u * radial + 2 * p1 * u * v + p2 * (r2 + 2 * u * u), v + v * radial + 2 * p2 * u * v + p1 * (r2 + 2 * v * v))
    elif model == "FULL_OPENCV":
        k1, k2, p1, p2, k3, k4, k5, k6 = extra
        radial = (1 + k1 * r2 + k2 * r2 ** 2 + k3 * r2 ** 3) / (1 + k4 * r2 + k5 * r2 ** 2 + k6 * r2 ** 3)
        u, v = (u * radial + 2 * p1 * u * v + p2 * (r2 + 2 * u * u), v * radial + 2 * p2 * u * v + p1 * (r2 + 2 * v * v))
    elif model == "OPENCV_FISHEYE":
        k1, k2, k3, k4 = extra
        r = np.sqrt(r2)
        th = np.arctan(r)
        t2 = th * th
        s = np.where(r > 0, th * (1 + k1 * t2 + k2 * t2 ** 2 + k3 * t2 ** 3 + k4 * t2 ** 4) / np.maximum(r, 1e-30), 1.0)
        u, v = u * s, v * s
    return np.stack([fx * u + cx, fy * v + cy], -1), X[:, 2] > 0


@pytest.mark.parametrize("binary", [True, False])
@pytest.mark.parametrize("factor", [1, 2])
def test_colmap_reader_reprojects_every_observation(tmp_path, binary, factor):
    models = list(CAMERAS)
    cams, images, pts = _colmap_scene(str(tmp_path), models, factor, binary, n_frames=14)
    train, val, extent, ids, loaded = scene_data.colmap_scene(str(tmp_path), factor=factor, test_split_interval=0)
    assert len(train) == len(val) == 14 and ids == sorted(cams)
    for i, im in enumerate(sorted(images, key=lambda m: m["name"])):
        cam = train.cameras[train.camera_of[i]]
        assert ids[train.camera_of[i]] == im["camera_id"] and (cam.width, cam.height) == (W_FULL // factor, H_FULL // factor)
        c2w = train.c2w[i].astype(np.float64)
        cam_pts = (pts[im["point3D_ids"]] - c2w[:3, 3]) @ c2w[:3, :3]
        uv, ok = project(cam.params, cam.kind, cam_pts)
        assert ok.all()
        np.testing.assert_allclose(uv, im["xys"] / factor, atol=1e-3, rtol=0)


@pytest.mark.parametrize("model", list(CAMERAS))
def test_colmap_rays_land_on_pixel_centres(model):
    cam = scene_data.colmap_camera(model, np.asarray(CAMERAS[model]), W_FULL, H_FULL, 1)
    _, d = cam.host_rays()
    d = d[0].reshape(-1, 3).astype(np.float64)
    uv, ok = project(cam.params, cam.kind, d)
    v, u = np.meshgrid(np.arange(H_FULL), np.arange(W_FULL), indexing="ij")
    centres = np.stack([u.ravel() + 0.5, v.ravel() + 0.5], -1)
    assert ok.mean() > 0.9
    np.testing.assert_allclose(uv[ok], centres[ok], atol=1e-3, rtol=0)
    assert np.allclose(np.linalg.norm(d, axis=1), 1.0, atol=1e-6)


def test_colmap_unknown_model_is_named():
    with pytest.raises(NotImplementedError, match="FOV"):
        scene_data.colmap_camera("FOV", np.ones(5), W_FULL, H_FULL, 1)


def test_colmap_split_extent_and_filters(tmp_path):
    cams, images, _ = _colmap_scene(str(tmp_path), ["PINHOLE", "OPENCV"], 1, True, n_frames=7, names=["left", "right"])
    train, val, extent, ids, _ = scene_data.colmap_scene(str(tmp_path), test_split_interval=3)
    assert len(val) == 3 and len(train) == 4
    allc = np.concatenate([train.c2w, val.c2w])[:, :3, 3]
    ordered = sorted(images, key=lambda m: m["name"])
    centres = []
    for im in ordered:
        w2c = np.eye(4, dtype=np.float32)
        w2c[:3, :3], w2c[:3, 3] = scene_data.qvec_to_so3(im["qvec"]), im["tvec"]
        centres.append(np.linalg.inv(w2c)[:3, 3])
    centres = np.array(centres)
    np.testing.assert_array_equal(val.c2w[:, :3, 3], centres[[0, 3, 6]])
    np.testing.assert_array_equal(train.c2w[:, :3, 3], centres[[1, 2, 4, 5]])
    med = np.median(centres, axis=0)
    assert extent == pytest.approx(1.1 * np.median(np.linalg.norm(centres - med, axis=1)))  # all frames, before the split
    assert sorted(map(tuple, allc)) == sorted(map(tuple, centres))
    only2, _, _, ids2, _ = scene_data.colmap_scene(str(tmp_path), test_split_interval=0, camera_ids=[2])
    assert ids2 == [2] and len(only2) == 3 and all("right" in p for p in only2.image_paths)
    left, _, _, ids3, _ = scene_data.colmap_scene(str(tmp_path), test_split_interval=0, camera_names=["left"])
    assert ids3 == [1] and len(left) == 4
    with pytest.raises(ValueError, match="camera_ids"):
        scene_data.colmap_scene(str(tmp_path), camera_ids=[9])


# ---- view stream --------------------------------------------------------------------------------------------------------------------

def _stream_rank(rank, world, port, out):
    import torch.distributed as dist

    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    stream = trainer.ViewStream(10, 42)
    mine = [stream.step_views(s, world)[rank] for s in range(25)]
    gathered = [None] * world
    dist.all_gather_object(gathered, mine)
    if rank == 0:
        out.put(gathered)
    dist.destroy_process_group()


def test_view_stream_two_ranks_cover_each_epoch():
    import socket

    import torch.multiprocessing as mp

    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_stream_rank, args=(r, 2, port, q)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        gathered = q.get(timeout=120)
        for p in procs:
            p.join(timeout=60)
    finally:
        for p in procs:  # a rank that hangs must not outlive the test
            if p.is_alive():
                p.terminate()
                p.join(timeout=10)
    stream = [v for s in range(25) for v in (gathered[0][s], gathered[1][s])]  # 50 elements = 5 epochs of 10
    for e in range(5):
        assert sorted(stream[10 * e:10 * e + 10]) == list(range(10))
        assert stream[10 * e:10 * e + 10] == trainer.epoch_permutation(10, 42, e).tolist()
    restarted = trainer.ViewStream(10, 42)
    assert [restarted.step_views(s, 2) for s in range(13, 25)] == [[gathered[0][s], gathered[1][s]] for s in range(13, 25)]


# ---- PLY ----------------------------------------------------------------------------------------------------------------------------

def test_ply_round_trip(tmp_path):
    g = torch.Generator().manual_seed(0)
    n = 37
    params = {"positions": torch.randn(n, 3, generator=g), "density": torch.randn(n, 1, generator=g), "rotation": torch.randn(n, 4, generator=g),
              "scale": torch.randn(n, 3, generator=g), "features_albedo": torch.randn(n, 3, generator=g),
              "features_specular": torch.randn(n, 45, generator=g)}
    path = str(tmp_path / "x.ply")
    trainer.export_ply(params, path)
    back = initialization.read_gaussian_ply(path)
    for k, v in params.items():
        assert np.array_equal(back[k], v.numpy()), k
    with open(path, "rb") as f:
        header = f.read(4096).split(b"end_header")[0].decode()
    props = [ln.split()[-1] for ln in header.splitlines() if ln.startswith("property")]
    assert props == (["x", "y", "z", "nx", "ny", "nz", "f_dc_0", "f_dc_1", "f_dc_2"] + [f"f_rest_{i}" for i in range(45)]
                     + ["opacity", "scale_0", "scale_1", "scale_2", "rot_0", "rot_1", "rot_2", "rot_3"])
    assert "binary_little_endian" in header
    v = initialization.read_ply_vertices(path)
    assert np.all(v["nz"] == 1) and np.all(v["nx"] == 0)
    spec = params["features_specular"].numpy().reshape(n, 15, 3)
    assert np.array_equal(v["f_rest_1"], spec[:, 1, 0]) and np.array_equal(v["f_rest_15"], spec[:, 0, 1])  # channel-major


# ---- refusals -----------------------------------------------------------------------------------------------------------------------

REFUSED = [("dataset.type", "scannetpp"), ("dataset.normalize_world_space", True), ("dataset.gsplat_image_downscale", True),
           ("loss.use_l2", True), ("strategy.densify.params", "features_albedo"), ("strategy.density_decay.start_iteration", 500),
           ("strategy.prune_weight.start_iteration", 0), ("strategy.prune_scale.start_iteration", 10), ("model.optimize_rotation", False),
           ("model.optimize_density", False), ("export_usd.enabled", True), ("with_gui", True), ("with_viser_gui", True),
           ("post_processing.method", "ppisp"), ("render.method", "3dgrut")]


def _base_conf(path):
    return {"path": str(path), "dataset": {"type": "nerf"}, "render": {"method": "3dgut"}, "model": {"feature_type": "sh"},
            "loss": {"use_l2": False}, "export_usd": {"enabled": False}, "post_processing": {"method": None},
            "strategy": {"method": "GSStrategy", "densify": {"params": "positions"}, "density_decay": {"start_iteration": -1},
                         "prune_weight": {"start_iteration": -1}, "prune_scale": {"start_iteration": -1}}}


@pytest.mark.parametrize("key, value", REFUSED)
def test_refusals_name_the_key_before_reading_images(tmp_path, monkeypatch, key, value):
    conf = _base_conf(tmp_path / "missing")  # no scene on disk: a refusal must come before any file is opened
    node = conf
    *parents, leaf = key.split(".")
    for p in parents:
        node = node.setdefault(p, {})
    node[leaf] = value
    monkeypatch.setattr(scene_data, "read_image", lambda *a, **k: pytest.fail("an image was read"))
    with pytest.raises(NotImplementedError, match=re.escape(key)):
        trainer.train(conf, device="cpu")


def test_strategy_configs_follow_the_shipped_keys():
    gs = {"method": "GSStrategy", "densify": {"params": "positions", "frequency": 7, "start_iteration": 3, "end_iteration": 50,
                                              "clone_grad_threshold": 1e-3, "split_grad_threshold": 2e-3, "relative_size_threshold": 0.05,
                                              "split": {"n_gaussians": 3}},
          "prune": {"frequency": 5, "start_iteration": 2, "end_iteration": 40, "density_threshold": 0.01},
          "reset_density": {"frequency": 11, "start_iteration": 1, "end_iteration": 50, "new_max_density": 0.02},
          "density_decay": {"gamma": 0.9, "start_iteration": -1}}
    c = step_config.strategy_config({"strategy": gs})
    assert (c.densify_frequency, c.densify_start, c.densify_end, c.clone_grad_threshold, c.split_grad_threshold, c.relative_size_threshold,
            c.split_n_gaussians, c.prune_frequency, c.prune_start, c.prune_end, c.prune_density_threshold, c.reset_frequency, c.reset_start,
            c.new_max_density, c.density_decay_gamma) == (7, 3, 50, 1e-3, 2e-3, 0.05, 3, 5, 2, 40, 0.01, 11, 1, 0.02, 0.9)
    m = step_config.strategy_config({"strategy": {"method": "MCMCStrategy", "binom_n_max": 9, "opacity_threshold": 0.1,
                                                  "relocate": {"start_iteration": 1, "end_iteration": 2, "frequency": 3},
                                                  "add": {"start_iteration": 4, "end_iteration": 5, "frequency": 6, "max_n_gaussians": 7},
                                                  "perturb": {"start_iteration": 8, "end_iteration": 9, "frequency": 10, "noise_lr": 11.0}}})
    assert (m.binom_n_max, m.opacity_threshold, m.relocate_start, m.relocate_end, m.relocate_frequency, m.add_start, m.add_end,
            m.add_frequency, m.max_n_gaussians, m.perturb_start, m.perturb_end, m.perturb_frequency, m.noise_lr) == \
        (9, 0.1, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11.0)

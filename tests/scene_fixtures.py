"""Small scenes on disk for the dataset and training-loop tests: NeRF-synthetic folders and COLMAP sparse models (.bin or .txt) with the
images the caller supplies, plus a float64 restatement of the 3DGUT projections (gut_project.cu project_pinhole / project_fisheye)."""
from __future__ import annotations

import json
import os
import struct

import numpy as np

MODEL_IDS = {"SIMPLE_PINHOLE": 0, "PINHOLE": 1, "SIMPLE_RADIAL": 2, "RADIAL": 3, "OPENCV": 4, "OPENCV_FISHEYE": 5, "FULL_OPENCV": 6,
             "FOV": 7}


def write_png(path, arr):
    from PIL import Image

    os.makedirs(os.path.dirname(path), exist_ok=True)
    Image.fromarray(np.ascontiguousarray(arr)).save(path)


def write_nerf(root, frames: dict, camera_angle_x: float, ext: str = ".png", path_suffix: str = ""):
    """frames: split -> [(c2w in NeRF's right-up-back convention [4,4], image uint8 [H,W,3|4], mask uint8 [H,W] or None)].  The json's
    file_path carries `path_suffix` (the reader probes "", ".png", ".jpg")."""
    for split, rows in frames.items():
        out = []
        for i, (c2w, img, mask) in enumerate(rows):
            rel = f"./{split}/r_{i}"
            write_png(os.path.join(root, rel + ext), img)
            if mask is not None:
                write_png(os.path.join(root, rel + "_mask.png"), mask)
            out.append({"file_path": rel + path_suffix, "transform_matrix": np.asarray(c2w, np.float64).tolist()})
        with open(os.path.join(root, f"transforms_{split}.json"), "w") as f:
            json.dump({"camera_angle_x": camera_angle_x, "frames": out}, f)


def rotmat_to_qvec(R):
    """COLMAP's (w, x, y, z) quaternion of a rotation matrix (rotmat2qvec, colmap/scripts/python/read_write_model.py)."""
    R = np.asarray(R, np.float64)
    K = np.array([[R[0, 0] - R[1, 1] - R[2, 2], 0, 0, 0], [R[1, 0] + R[0, 1], R[1, 1] - R[0, 0] - R[2, 2], 0, 0],
                  [R[2, 0] + R[0, 2], R[2, 1] + R[1, 2], R[2, 2] - R[0, 0] - R[1, 1], 0],
                  [R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1], R[0, 0] + R[1, 1] + R[2, 2]]]) / 3.0
    vals, vecs = np.linalg.eigh(K)
    q = vecs[[3, 0, 1, 2], np.argmax(vals)]
    return -q if q[0] < 0 else q


def write_colmap(root, cameras: dict, images: list, binary: bool = True, points=None):
    """cameras: id -> (model, width, height, params); images: [dict(id, qvec, tvec, camera_id, name, xys [M,2], point3D_ids [M])].
    points: optional (xyz [P,3], rgb [P,3] uint8) written as points3D."""
    sparse = os.path.join(root, "sparse/0")
    os.makedirs(sparse, exist_ok=True)
    if binary:
        with open(os.path.join(sparse, "cameras.bin"), "wb") as f:
            f.write(struct.pack("<Q", len(cameras)))
            for cid, (model, w, h, params) in cameras.items():
                f.write(struct.pack("<iiQQ", cid, MODEL_IDS[model], w, h) + struct.pack(f"<{len(params)}d", *params))
        with open(os.path.join(sparse, "images.bin"), "wb") as f:
            f.write(struct.pack("<Q", len(images)))
            for im in images:
                f.write(struct.pack("<idddddddi", im["id"], *im["qvec"], *im["tvec"], im["camera_id"]) + im["name"].encode() + b"\x00")
                f.write(struct.pack("<Q", len(im["xys"])))
                for (x, y), pid in zip(im["xys"], im["point3D_ids"]):
                    f.write(struct.pack("<ddq", x, y, int(pid)))
        if points is not None:
            xyz, rgb = points
            with open(os.path.join(sparse, "points3D.bin"), "wb") as f:
                f.write(struct.pack("<Q", len(xyz)))
                for i, (p, c) in enumerate(zip(xyz, rgb)):
                    f.write(struct.pack("<Q3d3BdQ", i, *p, *c, 0.0, 0))
    else:
        with open(os.path.join(sparse, "cameras.txt"), "w") as f:
            f.write("# camera list\n")
            for cid, (model, w, h, params) in cameras.items():
                f.write(f"{cid} {model} {w} {h} " + " ".join(repr(float(p)) for p in params) + "\n")
        with open(os.path.join(sparse, "images.txt"), "w") as f:
            f.write("# image list\n")
            for im in images:
                f.write(" ".join(str(v) for v in [im["id"], *(repr(float(q)) for q in im["qvec"]), *(repr(float(t)) for t in im["tvec"]),
                                                  im["camera_id"], im["name"]]) + "\n")
                f.write(" ".join(f"{float(x)!r} {float(y)!r} {int(p)}" for (x, y), p in zip(im["xys"], im["point3D_ids"])) + "\n")
        if points is not None:
            xyz, rgb = points
            with open(os.path.join(sparse, "points3D.txt"), "w") as f:
                for i, (p, c) in enumerate(zip(xyz, rgb)):
                    f.write(f"{i} {float(p[0])!r} {float(p[1])!r} {float(p[2])!r} {c[0]} {c[1]} {c[2]} 0.0\n")


def project(params: dict, kind: str, pts_cam: np.ndarray):
    """float64 restatement of project_pinhole / project_fisheye on camera-space points [M,3]: (uv [M,2], valid [M])."""
    x, y, z = pts_cam[:, 0], pts_cam[:, 1], pts_cam[:, 2]
    fx, fy, cx, cy = params["fx"], params["fy"], params["cx"], params["cy"]
    if kind == "fisheye":
        k = [float(v) for v in params["radial"][:4]]
        rho = np.maximum(np.hypot(x, y), 1.1920929e-07)
        th = np.minimum(np.arctan2(rho, z), params["max_angle"])
        t2 = th * th
        delta = th * (1 + t2 * (k[0] + t2 * (k[1] + t2 * (k[2] + t2 * k[3])))) / rho
        return np.stack([fx * x * delta + cx, fy * y * delta + cy], -1), np.arctan2(rho, z) < params["max_angle"]
    u, v = x / z, y / z
    k = [float(c) for c in params.get("radial", np.zeros(6))]
    p = [float(c) for c in params.get("tangential", np.zeros(2))]
    s = [float(c) for c in params.get("thin_prism", np.zeros(4))]
    r2 = u * u + v * v
    icd = (1 + r2 * (k[0] + r2 * (k[1] + r2 * k[2]))) / (1 + r2 * (k[3] + r2 * (k[4] + r2 * k[5])))
    dx = p[0] * 2 * u * v + p[1] * (r2 + 2 * u * u) + r2 * (s[0] + r2 * s[1])
    dy = p[0] * (r2 + 2 * v * v) + p[1] * 2 * u * v + r2 * (s[2] + r2 * s[3])
    return np.stack([(icd * u + dx) * fx + cx, (icd * v + dy) * fy + cy], -1), (z > 0) & (icd > 0.8) & (icd < 1.2)


def look_at_w2c(eye, target=(0.0, 0.0, 0.0)):
    """World -> camera [R | t] of a camera at `eye` looking at `target` ([right, down, front])."""
    import scenes

    c2w = scenes.look_at_c2w(eye, target)
    return np.linalg.inv(c2w)


def run_conf(path, out_dir, *, dataset="nerf", method="3dgut", strategy="gs", feature_type="sh", n_iterations=40, **extra):
    """A run configuration with the reference's keys (configs/base_gs.yaml and its groups) at small sizes."""
    conf = {
        "path": path, "out_dir": out_dir, "experiment_name": "t", "seed_initialization": 42, "n_iterations": n_iterations, "resume": "",
        "val_frequency": 999999, "validate_first": False, "test_last": True, "log_frequency": 10, "with_gui": False, "with_viser_gui": False,
        "checkpoint": {"iterations": [n_iterations // 2]}, "export_ply": {"enabled": feature_type == "sh", "path": ""},
        "import_ply": {"enabled": False, "path": "", "init_global_step": 0}, "export_usd": {"enabled": False},
        "dataset": {"type": dataset} if dataset == "nerf" else {"type": "colmap", "downsample_factor": 1, "test_split_interval": 8,
                                                                "normalize_world_space": False, "gsplat_image_downscale": False},
        "initialization": {"method": "random", "num_gaussians": 2000, "xyz_min": -1.5, "xyz_max": 1.5} if dataset == "nerf" else
        {"method": "colmap", "observation_scale_factor": 0.01, "use_observation_points": False},
        "render": {"method": method, "particle_kernel_degree": 2 if method == "3dgut" else 4, "particle_kernel_density_clamping": method == "3dgrt",
                   "particle_kernel_min_response": 0.0113, "min_transmittance": 0.0001 if method == "3dgut" else 0.001,
                   "max_consecutive_bvh_update": 15, "primitive_type": "instances"},
        "model": {"feature_type": feature_type, "default_density": 0.1 if strategy == "gs" else 0.5,
                  "default_scale_factor": 1.0 if strategy == "gs" else 0.1, "background": {"color": "black"},
                  "progressive_training": {"init_n_features": 0, "max_n_features": 3, "increase_frequency": 10, "increase_step": 1},
                  "nht_decoder": {"hidden_dim": 128, "num_layers": 3, "sh_scale": 3.0, "learning_rate": 0.00068, "color_refine_steps": 5,
                                  "scheduler": {"type": "cosine", "decay_final": 0.1, "max_steps": n_iterations}, "ema_decay": 0.95}},
        "optimizer": {"type": "adam", "eps": 1e-15},
        "scheduler": {"positions": {"type": "exp", "lr_init": 0.00016, "lr_final": 0.0000016, "max_steps": n_iterations},
                      "features": {"type": "cosine", "decay_final": 0.1, "max_steps": n_iterations}},
        "loss": {"use_l1": True, "lambda_l1": 0.8, "use_ssim": True, "lambda_ssim": 0.2, "use_opacity": strategy == "mcmc",
                 "lambda_opacity": 0.01, "use_scale": strategy == "mcmc", "lambda_scale": 0.01},
        "post_processing": {"method": None},
        "strategy": {"method": "GSStrategy", "densify": {"params": "positions", "frequency": 6, "start_iteration": 4, "end_iteration": 10000,
                                                         "clone_grad_threshold": 0.00005, "split_grad_threshold": 0.00005,
                                                         "relative_size_threshold": 0.01, "split": {"n_gaussians": 2}},
                     "prune": {"frequency": 5, "start_iteration": 4, "end_iteration": 10000, "density_threshold": 0.05},
                     "reset_density": {"frequency": 3000, "start_iteration": 0, "end_iteration": 10000, "new_max_density": 0.01},
                     "density_decay": {"start_iteration": -1}, "prune_weight": {"start_iteration": -1}, "prune_scale": {"start_iteration": -1}}
        if strategy == "gs" else
        {"method": "MCMCStrategy", "binom_n_max": 51, "opacity_threshold": 0.005,
         "relocate": {"start_iteration": 4, "end_iteration": 10000, "frequency": 5},
         "add": {"start_iteration": 4, "end_iteration": 10000, "frequency": 5, "max_n_gaussians": 3000},
         "perturb": {"start_iteration": 0, "end_iteration": 10000, "frequency": 1, "noise_lr": 500000.0}},
    }
    for k, v in extra.items():
        conf[k] = v
    return conf

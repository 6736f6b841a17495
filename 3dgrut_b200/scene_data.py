"""Scenes on disk as the training steps take them: the reference's NeRF-synthetic and COLMAP datasets (threedgrut/datasets/
dataset_nerf.py, dataset_colmap.py, __init__.py:68-81,203-210) reduced to what a training run reads.

A split yields **views** in the argument tuples of the steps' `step()` / `render()` -- 3DGUT `(rays_o, rays_d, sensor, pose7)`, 3DGRT
`(rays_o, rays_d, T_to_world)` -- with the float [H,W,3] target and an optional [H,W] mask.  Rays are in camera space through pixel centres
(u+0.5, v+0.5) and are computed once per camera; the sensor and the 3DGUT pose are built by threedgut_tracer's own
`Tracer._create_camera_parameters` from the frame's camera-to-world matrix, as the reference tracer builds them from a batch.  Images are
decoded once, at start-up, on host threads, and kept on the device as uint8 [H,W,3]; a step's target is one conversion into a buffer
allocated once per resolution (`target`).

The reference gets the rays of distorted and fisheye COLMAP cameras from `ncore`, which is not a dependency.  Here they are the inverse of
this repository's projection (gut_project.cu project_pinhole / project_fisheye): undistorted pinholes through scenes.pinhole_rays, fisheye
through scenes.fisheye_rays, and the distorted OpenCV pinhole through `opencv_pinhole_rays`, a float64 Newton inversion of the forward
model.  Projecting a pixel's ray lands on its pixel centre."""
from __future__ import annotations

import json
import os
import struct
from collections.abc import Sequence
from concurrent.futures import ThreadPoolExecutor
from types import SimpleNamespace

import numpy as np
import torch

import scenes
from b200_native import cfg_get

DATASET_TYPES = ("nerf", "colmap")
# COLMAP camera models: id -> (name, number of parameters) (colmap/src/colmap/sensor/models.h)
COLMAP_MODELS = {0: ("SIMPLE_PINHOLE", 3), 1: ("PINHOLE", 4), 2: ("SIMPLE_RADIAL", 4), 3: ("RADIAL", 5), 4: ("OPENCV", 8),
                 5: ("OPENCV_FISHEYE", 8), 6: ("FULL_OPENCV", 12), 7: ("FOV", 5), 8: ("SIMPLE_RADIAL_FISHEYE", 4), 9: ("RADIAL_FISHEYE", 5),
                 10: ("THIN_PRISM_FISHEYE", 12)}
DISTORTED_PINHOLES = ("SIMPLE_RADIAL", "RADIAL", "OPENCV", "FULL_OPENCV")


def check_dataset_config(conf) -> str:
    """dataset.type, with the dataset settings that are not built refused (NotImplementedError naming the key)."""
    kind = cfg_get(conf, "dataset.type", None)
    if kind not in DATASET_TYPES:
        raise NotImplementedError(f"dataset.type={kind!r}: the datasets built are {', '.join(DATASET_TYPES)}")
    for key in ("dataset.normalize_world_space", "dataset.gsplat_image_downscale"):
        if bool(cfg_get(conf, key, False)):
            raise NotImplementedError(f"{key}=true is not built (the GSplat-style COLMAP preprocessing)")
    return kind


# ---- rays ---------------------------------------------------------------------------------------------------------------------------

def opencv_pinhole_rays(height: int, width: int, focal, principal, radial, tangential, thin_prism, iterations: int = 20):
    """Camera-space unit rays of a distorted OpenCV pinhole through the pixel centres: for each pixel, the undistorted (x, y) whose
    project_pinhole image is (u+0.5, v+0.5), by float64 Newton iterations from the distorted point.  Returns ([1,H,W,3] zeros, [1,H,W,3])
    float32."""
    k = [float(v) for v in radial]
    p = [float(v) for v in tangential]
    s = [float(v) for v in thin_prism]
    v, u = np.meshgrid(np.arange(height, dtype=np.float64), np.arange(width, dtype=np.float64), indexing="ij")
    xd = (u + 0.5 - float(principal[0])) / float(focal[0])
    yd = (v + 0.5 - float(principal[1])) / float(focal[1])
    x, y = xd.copy(), yd.copy()
    for _ in range(iterations):
        r2 = x * x + y * y
        num = 1 + r2 * (k[0] + r2 * (k[1] + r2 * k[2]))
        den = 1 + r2 * (k[3] + r2 * (k[4] + r2 * k[5]))
        icd = num / den
        g = ((k[0] + r2 * (2 * k[1] + 3 * r2 * k[2])) * den - num * (k[3] + r2 * (2 * k[4] + 3 * r2 * k[5]))) / (den * den)  # d icd / d r2
        hx, hy = s[0] + 2 * r2 * s[1], s[2] + 2 * r2 * s[3]  # d (r2 (s0 + r2 s1)) / d r2
        fx_ = icd * x + p[0] * 2 * x * y + p[1] * (r2 + 2 * x * x) + r2 * (s[0] + r2 * s[1]) - xd
        fy_ = icd * y + p[0] * (r2 + 2 * y * y) + p[1] * 2 * x * y + r2 * (s[2] + r2 * s[3]) - yd
        a = icd + 2 * x * x * g + 2 * p[0] * y + 6 * p[1] * x + 2 * x * hx
        b = 2 * x * y * g + 2 * p[0] * x + 2 * p[1] * y + 2 * y * hx
        c = 2 * x * y * g + 2 * p[0] * x + 2 * p[1] * y + 2 * x * hy
        d = icd + 2 * y * y * g + 6 * p[0] * y + 2 * p[1] * x + 2 * y * hy
        det = a * d - b * c
        det = np.where(np.abs(det) > 1e-300, det, 1e-300)
        x, y = x - (d * fx_ - b * fy_) / det, y - (a * fy_ - c * fx_) / det
    dirs = np.stack([x, y, np.ones_like(x)], -1)
    dirs /= np.linalg.norm(dirs, axis=-1, keepdims=True)
    return np.zeros((1, height, width, 3), np.float32), dirs[None].astype(np.float32)


def fisheye_max_angle(width: int, height: int, focal, principal) -> float:
    """create_fisheye_camera's valid cone (dataset_colmap.py:403-408, utils.py:195-214): half the larger field of view spanned by the
    largest distance from the principal point to the image borders."""
    def border(size, pp):
        return pp if pp > 0.5 * size else size - pp
    focal = np.asarray(focal, np.float32)
    radius = float(np.linalg.norm(np.array([border(float(width), float(principal[0])), border(float(height), float(principal[1]))])))
    return float(np.max([2.0 * radius / focal[0], 2.0 * radius / focal[1]]) / 2.0)


# ---- cameras and splits --------------------------------------------------------------------------------------------------------------

class Camera:
    """One camera model at one resolution: `kind` pinhole / opencv_pinhole / fisheye, its intrinsics `params` and, once `to(device)`
    has run, its rays on the device."""

    def __init__(self, kind: str, width: int, height: int, params: dict):
        self.kind, self.width, self.height, self.params = kind, int(width), int(height), params
        self.rays = None

    def batch_intrinsics(self) -> dict:
        """The batch attribute the reference tracer reads the sensor from (tracer.py:383-488)."""
        p = self.params
        if self.kind == "pinhole" and p.get("nerf"):
            return {"intrinsics": [p["fx"], p["fy"], p["cx"], p["cy"]]}
        resolution = np.array([self.width, self.height], dtype=np.uint64)
        if self.kind == "fisheye":
            return {"intrinsics_OpenCVFisheyeCameraModelParameters": dict(
                resolution=resolution, shutter_type=4, principal_point=np.float32([p["cx"], p["cy"]]), focal_length=np.float32([p["fx"], p["fy"]]),
                radial_coeffs=np.float32(p["radial"][:4]), max_angle=p["max_angle"])}
        return {"intrinsics_OpenCVPinholeCameraModelParameters": dict(
            resolution=resolution, shutter_type=4, principal_point=np.float32([p["cx"], p["cy"]]), focal_length=np.float32([p["fx"], p["fy"]]),
            radial_coeffs=np.float32(p.get("radial", np.zeros(6))), tangential_coeffs=np.float32(p.get("tangential", np.zeros(2))),
            thin_prism_coeffs=np.float32(p.get("thin_prism", np.zeros(4))))}

    def host_rays(self):
        p, h, w = self.params, self.height, self.width
        if self.kind == "fisheye":
            return scenes.fisheye_rays(h, w, p["fx"], p["fy"], p["cx"], p["cy"], p["radial"][:4])
        if self.kind == "opencv_pinhole":
            return opencv_pinhole_rays(h, w, (p["fx"], p["fy"]), (p["cx"], p["cy"]), p["radial"], p["tangential"], p["thin_prism"])
        return scenes.pinhole_rays(h, w, p["fx"], p["fy"], p["cx"], p["cy"])

    def to(self, device):
        o, d = self.host_rays()
        self.rays = (torch.from_numpy(o).to(device), torch.from_numpy(d).to(device))
        return self


class Split:
    """The frames of one split.  Construct with the host data; `load(device)` decodes the images and puts images, masks and rays on the
    device.  Frame i: `view(i, method)`, `target(i)`, `mask(i)`, `c2w[i]`."""

    def __init__(self, cameras: list, camera_of: list, c2w: np.ndarray, image_paths: list, background=None, rgba_ok: bool = True):
        self.cameras, self.camera_of = cameras, [int(c) for c in camera_of]
        self.c2w = np.asarray(c2w, np.float32).reshape(-1, 4, 4)
        self.image_paths = list(image_paths)
        self.mask_paths = [os.path.splitext(p)[0] + "_mask.png" for p in self.image_paths]
        self.background = background   # nerf: model.background.color that RGBA images are composited onto
        self.images = self.masks = None
        self._sensors, self._poses, self._targets = {}, {}, {}

    def __len__(self):
        return len(self.image_paths)

    @property
    def camera_centers(self) -> np.ndarray:
        return self.c2w[:, :3, 3]

    def load(self, device, threads: int | None = None):
        """Decode every image and mask (PIL, host threads) and place them, and every camera's rays, on `device`."""
        with ThreadPoolExecutor(max_workers=threads or min(32, os.cpu_count() or 1)) as pool:
            images = list(pool.map(lambda p: read_image(p, self.background), self.image_paths))
            masks = list(pool.map(read_mask, self.mask_paths))
        for i, img in enumerate(images):
            cam = self.cameras[self.camera_of[i]]
            if img.shape[:2] != (cam.height, cam.width):
                raise ValueError(f"{self.image_paths[i]}: {img.shape[1]}x{img.shape[0]} image for a {cam.width}x{cam.height} camera")
        self.images = [torch.from_numpy(img).to(device) for img in images]
        self.masks = [None if m is None else torch.from_numpy(m).to(device) for m in masks]
        for cam in self.cameras:
            if cam.rays is None:
                cam.to(device)
        return self

    def _camera_parameters(self, i: int):
        from threedgut_tracer.tracer import Tracer

        if i not in self._sensors:
            cam = self.cameras[self.camera_of[i]]
            batch = SimpleNamespace(T_to_world=torch.from_numpy(self.c2w[i][None].copy()), **cam.batch_intrinsics())
            sensor, poses = Tracer._create_camera_parameters(batch)
            self._sensors[i] = (sensor, poses.T_world_sensors[0])
        return self._sensors[i]

    def view(self, i: int, method: str = "3dgut") -> tuple:
        """The render arguments of frame i: 3dgut (rays_o, rays_d, sensor, pose7) or 3dgrt (rays_o, rays_d, T_to_world [1,4,4] host tensor)."""
        rays_o, rays_d = self.cameras[self.camera_of[i]].rays
        if method == "3dgrt":
            key = ("T", i)
            if key not in self._poses:
                self._poses[key] = torch.from_numpy(np.ascontiguousarray(self.c2w[i][None]))  # a host tensor: no device read-back
            return rays_o, rays_d, self._poses[key]
        sensor, pose = self._camera_parameters(i)
        return rays_o, rays_d, sensor, pose

    def target(self, i: int) -> torch.Tensor:
        """Frame i's image as float [H,W,3] in [0,1], written into one buffer per resolution (the next call overwrites it)."""
        img = self.images[i]
        key = tuple(img.shape)
        buf = self._targets.get(key)
        if buf is None:
            buf = self._targets[key] = torch.empty(key, dtype=torch.float32, device=img.device)
        return torch.div(img, 255, out=buf)

    def mask(self, i: int):
        return self.masks[i]

    def views(self, method: str = "3dgut", device=None) -> "Views":
        """The (render_args, target) of every frame, for evaluate.evaluate / validate: a sequence whose items are made when read, each
        target a float tensor of its own, so a pass holds one float image at a time.  The split is loaded on `device` (default: the
        current CUDA device) first if it is not yet."""
        if self.images is None:
            self.load(torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device))
        return Views(self, method)


class Views(Sequence):
    """Split.views(): item i is (split.view(i, method), frame i's image as a new float [H,W,3] tensor)."""

    def __init__(self, split: Split, method: str):
        self.split, self.method = split, method

    def __len__(self):
        return len(self.split)

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self[j] for j in range(*i.indices(len(self)))]
        if not -len(self) <= i < len(self):
            raise IndexError(i)
        i %= len(self)
        return self.split.view(i, self.method), torch.div(self.split.images[i], 255)


# ---- images -------------------------------------------------------------------------------------------------------------------------

def read_image(path: str, background=None) -> np.ndarray:
    """uint8 [H,W,3] as the reference stores it (dataset_nerf.py:416-445): RGBA composited onto black or white in float32, then
    truncated with (img * 255).astype(uint8).  RGB images take the same float round trip.  "random" with an RGBA image raises
    ValueError, as the reference asserts."""
    from PIL import Image

    with Image.open(path) as im:
        arr = np.asarray(im)
    if arr.ndim == 2:
        arr = np.repeat(arr[..., None], 3, axis=-1)
    img = arr.astype(np.float32) / 255.0
    if img.shape[2] == 4:
        if background is None:
            img = img[..., :3]
        elif background == "black":
            img = img[..., :3] * img[..., -1:]
        elif background == "white":
            img = img[..., :3] * img[..., -1:] + (1 - img[..., -1:])
        else:
            raise ValueError(f"model.background.color={background!r} with RGBA images: the reference composites RGBA images onto black "
                             f"or white only (dataset_nerf.py:431)")
    return np.ascontiguousarray((img[..., :3] * 255.0).astype(np.uint8))


def read_mask(path: str):
    """float32 [H,W] of `<image>_mask.png` thresholded at > 0.5 after dividing by 255 (dataset_nerf.py:249-280), None when absent."""
    if not os.path.exists(path):
        return None
    from PIL import Image

    with Image.open(path) as im:
        m = np.asarray(im)
    if m.ndim == 3:
        m = m[..., 0]
    return ((m.astype(np.float32) / 255.0) > 0.5).astype(np.float32)


def center_and_diag(centers: np.ndarray):
    """utils.py:155-160: the median camera centre and the median distance from it."""
    center = np.median(centers, axis=0, keepdims=True)
    return center.flatten(), float(np.median(np.linalg.norm(centers - center, axis=1, keepdims=True)))


# ---- NeRF-synthetic ------------------------------------------------------------------------------------------------------------------

def nerf_split(root: str, split: str, background) -> Split:
    """transforms_{split}.json of a NeRF-synthetic scene (dataset_nerf.py:100-170)."""
    with open(os.path.join(root, "transforms_train.json")) as f:
        meta = json.load(f)
    first = os.path.join(root, meta["frames"][0]["file_path"])
    suffix = next((s for s in ("", ".png", ".jpg") if os.path.exists(first + s)), None)
    if suffix is None:
        raise FileNotFoundError(f"Image path {first} does not exist.")
    from PIL import Image

    with Image.open(first + suffix) as im:
        w, h = im.width, im.height
    fx = float(0.5 * w / np.tan(0.5 * meta["camera_angle_x"]))
    with open(os.path.join(root, f"transforms_{split}.json")) as f:
        frames = json.load(f)["frames"]
    c2w = []
    for fr in frames:
        m = np.array(fr["transform_matrix"], dtype=np.float32)
        m[:, 1:3] *= -1  # [right up back] to [right down front]
        c2w.append(m)
    cam = Camera("pinhole", w, h, {"fx": fx, "fy": fx, "cx": w / 2, "cy": h / 2, "nerf": True})
    paths = [os.path.join(root, fr["file_path"]) + suffix for fr in frames]
    return Split([cam], [0] * len(frames), np.stack(c2w), paths, background=background)


# ---- COLMAP -------------------------------------------------------------------------------------------------------------------------

def read_colmap_cameras(path: str) -> dict:
    """cameras.bin / cameras.txt -> {camera_id: (model name, width, height, params float64)}."""
    out = {}
    if path.endswith(".bin"):
        with open(path, "rb") as f:
            data = f.read()
        (n,), off = struct.unpack_from("<Q", data, 0), 8
        for _ in range(n):
            cid, mid, w, h = struct.unpack_from("<iiQQ", data, off)
            off += 24
            name, k = COLMAP_MODELS.get(mid, (f"model id {mid}", 0))
            if k == 0:
                raise NotImplementedError(f"COLMAP camera {name} is not a known model")
            out[cid] = (name, int(w), int(h), np.array(struct.unpack_from(f"<{k}d", data, off), np.float64))
            off += 8 * k
        return out
    with open(path) as f:
        for line in f:
            t = line.split()
            if t and not t[0].startswith("#"):
                out[int(t[0])] = (t[1], int(t[2]), int(t[3]), np.array([float(v) for v in t[4:]], np.float64))
    return out


def read_colmap_images(path: str) -> list:
    """images.bin / images.txt -> [dict(id, qvec, tvec, camera_id, name, xys, point3D_ids)] sorted by name (utils.py:440-560)."""
    images = []
    if path.endswith(".bin"):
        with open(path, "rb") as f:
            data = f.read()
        (n,), off = struct.unpack_from("<Q", data, 0), 8
        for _ in range(n):
            iid, *qt, cid = struct.unpack_from("<idddddddi", data, off)
            off += 64
            end = data.index(b"\x00", off)
            name = data[off:end].decode("utf-8")
            off = end + 1
            (m,) = struct.unpack_from("<Q", data, off)
            off += 8
            pts = np.frombuffer(data, dtype=np.dtype([("x", "<f8"), ("y", "<f8"), ("id", "<i8")]), count=m, offset=off)
            off += 24 * m
            images.append(dict(id=iid, qvec=np.array(qt[:4]), tvec=np.array(qt[4:7]), camera_id=cid, name=name,
                               xys=np.stack([pts["x"], pts["y"]], -1), point3D_ids=pts["id"].astype(np.int64)))
    else:
        with open(path) as f:
            lines = [ln.strip() for ln in f if not ln.strip().startswith("#")]
        i = 0
        while i < len(lines):
            if not lines[i]:
                i += 1
                continue
            t = lines[i].split()
            pts = np.array([float(v) for v in lines[i + 1].split()], np.float64).reshape(-1, 3) if i + 1 < len(lines) else np.zeros((0, 3))
            images.append(dict(id=int(t[0]), qvec=np.array([float(v) for v in t[1:5]]), tvec=np.array([float(v) for v in t[5:8]]),
                               camera_id=int(t[8]), name=" ".join(t[9:]), xys=pts[:, :2], point3D_ids=pts[:, 2].astype(np.int64)))
            i += 2
    return sorted(images, key=lambda im: im["name"])


def qvec_to_so3(q) -> np.ndarray:
    """utils.py:413-432."""
    w, x, y, z = (float(v) for v in q)
    return np.array([[1 - 2 * y * y - 2 * z * z, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
                     [2 * x * y + 2 * w * z, 1 - 2 * x * x - 2 * z * z, 2 * y * z - 2 * w * x],
                     [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x * x - 2 * y * y]])


def colmap_camera(model: str, params: np.ndarray, width: int, height: int, factor: int) -> Camera:
    """The Camera of a COLMAP model at the image size, its intrinsics divided by the scaling factor (dataset_colmap.py:83-113, 476-535)."""
    p = np.asarray(params, np.float64)
    if model == "SIMPLE_PINHOLE":
        return Camera("pinhole", width, height, {"fx": p[0] / factor, "fy": p[0] / factor, "cx": p[1] / factor, "cy": p[2] / factor})
    if model == "PINHOLE":
        return Camera("pinhole", width, height, {"fx": p[0] / factor, "fy": p[1] / factor, "cx": p[2] / factor, "cy": p[3] / factor})
    if model in DISTORTED_PINHOLES:
        q = p.astype(np.float32)  # _opencv_pinhole_intrinsics_from_colmap works in float32
        radial, tangential = np.zeros(6, np.float32), np.zeros(2, np.float32)
        if model in ("SIMPLE_RADIAL", "RADIAL"):
            focal, principal = np.float32([q[0], q[0]]) / factor, q[1:3] / factor
            radial[:len(q) - 3] = q[3:]
        elif model == "OPENCV":
            focal, principal = q[:2] / factor, q[2:4] / factor
            radial[:2], tangential[:] = q[4:6], q[6:8]
        else:
            focal, principal = q[:2] / factor, q[2:4] / factor
            radial[:], tangential[:] = q[[4, 5, 8, 9, 10, 11]], q[6:8]
        return Camera("opencv_pinhole", width, height, {"fx": float(focal[0]), "fy": float(focal[1]), "cx": float(principal[0]),
                                                         "cy": float(principal[1]), "radial": radial, "tangential": tangential,
                                                         "thin_prism": np.zeros(4, np.float32)})
    if model == "OPENCV_FISHEYE":
        q = p.copy()
        q[:4] = q[:4] / factor
        focal, principal = q[0:2].astype(np.float32), q[2:4].astype(np.float32)
        return Camera("fisheye", width, height, {"fx": float(focal[0]), "fy": float(focal[1]), "cx": float(principal[0]), "cy": float(principal[1]),
                                                  "radial": q[4:8].astype(np.float32), "max_angle": fisheye_max_angle(width, height, focal, principal)})
    raise NotImplementedError(f"COLMAP camera model {model!r} is not built (PINHOLE, SIMPLE_PINHOLE, SIMPLE_RADIAL, RADIAL, OPENCV, "
                              f"FULL_OPENCV and OPENCV_FISHEYE are)")


def _image_size(path: str):
    from PIL import Image

    with Image.open(path) as im:
        return im.size


def colmap_scene(root: str, factor: int = 1, test_split_interval: int = 8, camera_names=None, camera_ids=None):
    """(train Split, val Split, scene extent, camera ids in index order) of a COLMAP scene (dataset_colmap.py:148-240, 302-570)."""
    sparse = os.path.join(root, "sparse/0")
    ext = ".bin" if os.path.isfile(os.path.join(sparse, "images.bin")) and os.path.isfile(os.path.join(sparse, "cameras.bin")) else ".txt"
    intrinsics = read_colmap_cameras(os.path.join(sparse, "cameras" + ext))
    images = read_colmap_images(os.path.join(sparse, "images" + ext))
    # camera filters (dataset_colmap.py:236-300)
    selected = set(intrinsics)
    names = {cid: f"camera_{i}" for i, cid in enumerate(sorted(intrinsics))}
    for im in images:
        if os.path.dirname(im["name"]):
            names[im["camera_id"]] = os.path.dirname(im["name"])
    if camera_ids is not None:
        missing = sorted(set(camera_ids) - selected)
        if missing:
            raise ValueError(f"COLMAP camera_ids {missing} not found. Available camera_ids: {sorted(selected)}")
        selected &= set(camera_ids)
    if camera_names is not None:
        by_name = {}
        for cid, name in names.items():
            by_name.setdefault(name, set()).add(cid)
        missing = sorted(set(camera_names) - set(by_name))
        if missing:
            raise ValueError(f"COLMAP camera_names {missing} not found. Available camera_names: {sorted(by_name)}")
        selected &= set().union(*(by_name[n] for n in camera_names))
    images = [im for im in images if im["camera_id"] in selected]
    if not images:
        raise ValueError("COLMAP camera selection has no frames.")
    intrinsics = {cid: v for cid, v in intrinsics.items() if cid in selected}
    folder = "images" if factor == 1 else f"images_{factor}"
    index = {cid: i for i, cid in enumerate(sorted(intrinsics))}
    last_image = {im["camera_id"]: im["name"] for im in images}
    cameras = [None] * len(index)
    for cid, (model, full_w, full_h, params) in intrinsics.items():
        if cid not in last_image:
            continue
        width, height = _image_size(os.path.join(root, folder, last_image[cid]))
        scale = int(round(full_h / height))
        if abs(full_w / scale - width) > 1 or abs(full_h / scale - height) > 1:
            raise ValueError(f"Scaled image dimension {full_w / scale}x{full_h / scale} (factor {scale}x) does not match the actual image "
                             f"dimensions {width}x{height}")
        cameras[index[cid]] = colmap_camera(model, params, width, height, scale)
    c2w = []
    for im in images:
        w2c = np.eye(4, dtype=np.float32)
        w2c[:3, :3], w2c[:3, 3] = qvec_to_so3(im["qvec"]), im["tvec"]
        c2w.append(np.linalg.inv(w2c))
    c2w = np.stack(c2w).astype(np.float32)
    _, diag = center_and_diag(c2w[:, :3, 3])  # all frames, before the split (dataset_colmap.py:568-570)
    extent = diag * 1.1
    idx = np.arange(len(images))
    train = (idx % test_split_interval != 0) if test_split_interval > 0 else np.ones(len(images), bool)
    val = (idx % test_split_interval == 0) if test_split_interval > 0 else np.ones(len(images), bool)
    paths = [os.path.join(root, folder, im["name"]) for im in images]
    cam_of = [index[im["camera_id"]] for im in images]

    def split(sel):
        where = np.where(sel)[0]
        return Split(cameras, [cam_of[i] for i in where], c2w[where], [paths[i] for i in where])

    return split(train), split(val), extent, sorted(intrinsics), images


# ---- a scene -------------------------------------------------------------------------------------------------------------------------

class SceneData:
    """What a training run reads from a dataset: `train`, `val` and `test` Splits, `scene_extent`, `observer_points` (the training
    cameras' centres, get_observer_points), `points_transform` (None: no world normalisation is built) and `path`."""

    def __init__(self, conf, device=None, load_images: bool = True):
        kind = check_dataset_config(conf)
        self.path = str(cfg_get(conf, "path", ""))
        if kind == "nerf":
            bg = str(cfg_get(conf, "model.background.color", "black"))
            self.train = nerf_split(self.path, "train", bg)
            self.val = nerf_split(self.path, "val", bg)
            self.test = nerf_split(self.path, "test", bg)
            _, diag = center_and_diag(self.train.camera_centers)  # dataset_nerf.py:162-164
            self.scene_extent = diag * 1.1
        else:
            self.train, self.val, self.scene_extent, self.camera_ids, _ = colmap_scene(
                self.path, int(cfg_get(conf, "dataset.downsample_factor", 1)), int(cfg_get(conf, "dataset.test_split_interval", 8)),
                cfg_get(conf, "dataset.camera_names", None), cfg_get(conf, "dataset.camera_ids", None))
            self.test = self.val  # make_test builds the colmap "val" split (datasets/__init__.py:203-215)
        self.scene_extent = float(self.scene_extent)
        self.observer_points = np.ascontiguousarray(self.train.camera_centers, np.float32)
        self.points_transform = None
        if load_images:
            self.load(device)

    def load(self, device=None):
        """Decode the training split onto the device.  The val and test splits are decoded when they are first evaluated
        (Split.views), so a run that never validates holds only the training images."""
        self.train.load(torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device))
        return self

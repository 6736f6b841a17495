"""The start of a run: the reference's Gaussian initialisations (threedgrut/model/model.py:416-611 and :708-780, Trainer.setup_training,
trainer.py:326-401), producing the `params` dict every training step takes.

Every initialisation returns contiguous float32 raw leaf tensors on the device: schedule.SH_GROUPS with features_albedo [N,3] and
features_specular [N,45] for SH, schedule.NHT_GROUPS with features [N,48] for NHT.  The starting scales come from an exact k-nearest-
neighbour search on the GPU (gutb200_knn, DESIGN.md section 19) instead of the reference's scikit-learn KD-tree on the CPU; the distances
are recomputed from its indices with the reference's own expressions, so the same neighbours give the same bits.  There is no CPU path.

Datasets stay outside: the caller passes what the dataset would give (observer points, the dataset's world transform, lidar points).
Readers for COLMAP points3D.bin / .txt and vertex PLY files are here because the reference's `plyfile` is not a dependency."""
from __future__ import annotations

import os
import struct

import numpy as np
import torch

import b200_native as nat
import schedule
from b200_native import cfg_get

C0 = 0.28209479177387814  # SH band-0 constant (threedgrut/utils/render.py RGB2SH)
METHODS = ("colmap", "fused_point_cloud", "point_cloud", "random", "checkpoint", "lidar")
SPECULAR_DIM = 45         # sh_degree_to_specular_dim(3): the steps store 16 SH coefficients
# the reference's defaults (configs/base_gs.yaml, configs/initialization/*.yaml) for keys a conf leaves out
DEFAULTS = {"seed_initialization": 42, "model.default_density": 0.1, "model.default_scale_factor": 1.0,
            "initialization.observation_scale_factor": 0.01, "initialization.use_observation_points": True,
            "initialization.num_gaussians": 100_000, "initialization.xyz_min": -1.5, "initialization.xyz_max": 1.5,
            "initialization.num_points": 1_000_000, "model.nht_features.init_min": -5.0, "model.nht_features.init_max": 5.0}


def _get(conf, key):
    return cfg_get(conf, key, DEFAULTS.get(key))


def _device(device) -> torch.device:
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    if dev.type != "cuda":
        raise ValueError(f"device={dev}: the initialisation runs on a CUDA device (there is no CPU path)")
    return dev


# ---- k nearest neighbours ----------------------------------------------------------------------------------------------------------

def _points_arg(name: str, t) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or t.ndim != 2 or t.shape[1] != 3:
        raise ValueError(f"{name} must be a [N,3] tensor, got {type(t).__name__} {tuple(getattr(t, 'shape', ()))}")
    if t.device.type != "cuda":
        raise ValueError(f"{name} is on {t.device}: the search runs on a CUDA device (there is no CPU path)")
    t = t.detach().to(torch.float32).contiguous()
    if not bool(torch.isfinite(t).all()):
        raise ValueError(f"{name} holds non-finite coordinates")
    return t


def nearest_neighbors(points: torch.Tensor, k: int = 1, targets: torch.Tensor | None = None):
    """The k nearest neighbours of each row of `points` ([N,3], CUDA), exactly: among `targets` ([M,3]) when given, else among the other
    points (row i excludes point i and only it; duplicates are neighbours at distance 0).  Rows ascend by float32 squared distance, ties
    by the lower index.  Returns (dist [N,k] float32 squared distances, idx [N,k] int64).  1 <= k <= 4; the same inputs give the same
    bits on every run.  Non-finite coordinates raise ValueError."""
    pts = _points_arg("points", points)
    tgt = pts if targets is None else _points_arg("targets", targets)
    if tgt.device != pts.device:
        raise ValueError(f"targets are on {tgt.device} and points on {pts.device}")
    n, m, k = int(pts.shape[0]), int(tgt.shape[0]), int(k)
    lib = nat.load()
    dist = torch.empty((n, max(k, 0)), dtype=torch.float32, device=pts.device)
    idx = torch.empty((n, max(k, 0)), dtype=torch.int32, device=pts.device)
    with torch.cuda.device(pts.device):
        ws = torch.empty(max(int(lib.gutb200_knn_workspace_bytes(m)), 1), dtype=torch.uint8, device=pts.device)
        rc = lib.gutb200_knn(torch.cuda.current_stream(pts.device).cuda_stream, m, tgt.data_ptr(), n,
                             None if targets is None else pts.data_ptr(), k, ws.data_ptr(), ws.numel(), idx.data_ptr(), dist.data_ptr())
    if rc != 0:
        raise ValueError(lib.gutb200_last_error(None).decode())
    return dist, idx.long()


# ---- initialisation from points (default_initialize_from_points) -------------------------------------------------------------------

def _feature_type(conf) -> str:
    """'sh' or 'nht'; NotImplementedError naming the key for a setting the steps do not train."""
    for key, want in (("model.density_activation", "sigmoid"), ("model.scale_activation", "exp")):
        got = cfg_get(conf, key, want)
        if str(got) != want:
            raise NotImplementedError(f"{key}={got!r}: the training steps' activations are fixed ({key}={want!r})")
    nht = nat.nht_feature_config(conf, "initialization") is not None
    if not nht:
        got = cfg_get(conf, "model.progressive_training.max_n_features", 3)
        if int(got) != 3:
            raise NotImplementedError(f"model.progressive_training.max_n_features={got!r}: the build stores 16 SH coefficients (degree 3)")
    return "nht" if nht else "sh"


def _inverse_sigmoid(x):
    return torch.log(x / (1 - x))  # threedgrut/utils/misc.py inverse_sigmoid


def from_points(points, colors=None, observers=None, conf=None, *, use_observer_pts: bool | None = None) -> dict:
    """default_initialize_from_points (model.py:708-780) on `points` [N,3] (CUDA): positions = the points, random rotations, constant
    density, scales from the neighbours, features from `colors` ([N,3] uint8; drawn when None).  use_observer_pts: None reads
    initialization.use_observation_points; true scales each Gaussian by its distance to the nearest of `observers` [M,3], false by the
    mean squared distance to its 3 nearest other points.  Draws come from a generator on the device seeded seed_initialization, in the
    reference's order: rotations, colours (when absent), NHT features."""
    ft = _feature_type(conf)
    if use_observer_pts is None:
        use_observer_pts = bool(_get(conf, "initialization.use_observation_points"))
    pts = _points_arg("points", points)
    dev, dtype, n = pts.device, torch.float32, int(pts.shape[0])
    rng = torch.Generator(device=dev).manual_seed(int(_get(conf, "seed_initialization")))
    rots = torch.rand((n, 4), dtype=dtype, device=dev, generator=rng)
    if use_observer_pts:
        if observers is None:
            raise ValueError("initialization.use_observation_points is true but no observer points were given")
        obs = _points_arg("observers", torch.as_tensor(observers, dtype=dtype, device=dev))
        _, idx = nearest_neighbors(pts, 1, targets=obs)
        dist = torch.clamp_min(torch.linalg.norm(pts - obs[idx[:, 0], :], dim=-1), 1e-7)
        scale = dist * float(_get(conf, "initialization.observation_scale_factor"))
    else:
        _, idx = nearest_neighbors(pts, 3)
        # scikit-learn's float64 distances, cast back to the points' dtype (geometry.py k_nearest_neighbors: `.to(x)`)
        d = torch.linalg.norm(pts.double()[:, None, :] - pts.double()[idx], dim=-1).to(pts)
        scale = torch.sqrt((d ** 2).mean(dim=-1))
    scale = scale * float(_get(conf, "model.default_scale_factor"))
    scales = torch.log(scale)[:, None].repeat(1, 3)
    density = _inverse_sigmoid(torch.full((n, 1), fill_value=float(_get(conf, "model.default_density")), dtype=dtype, device=dev))
    if colors is None:
        colors = torch.randint(0, 256, (n, 3), dtype=torch.uint8, device=dev, generator=rng)
    else:
        colors = torch.as_tensor(colors)
        if colors.dtype != torch.uint8 or tuple(colors.shape) != (n, 3):
            raise ValueError(f"colors must be [N,3] uint8 (N = {n}), got {colors.dtype} {tuple(colors.shape)}")
    out = {"positions": pts.clone(), "density": density, "rotation": rots, "scale": scales}
    if ft == "sh":
        # colours / 255 where the colours are, then RGB2SH on the host in float32, as the reference's numpy path computes it
        rgb = (colors.float() / 255.0).cpu().numpy()
        out["features_albedo"] = torch.from_numpy((rgb - 0.5) / C0).to(dev)
        out["features_specular"] = torch.zeros((n, SPECULAR_DIM), dtype=dtype, device=dev)
    else:
        lo, hi = float(_get(conf, "model.nht_features.init_min")), float(_get(conf, "model.nht_features.init_max"))
        out["features"] = torch.rand((n, nat.NHT_FEATURE_DIM), dtype=dtype, device=dev, generator=rng) * (hi - lo) + lo
    return _leaves(out, ft)


def _leaves(out: dict, ft: str) -> dict:
    groups = schedule.NHT_GROUPS if ft == "nht" else schedule.SH_GROUPS
    return {k: out[k].detach().to(torch.float32).contiguous() for k in groups}


def random_point_cloud(num_gaussians: int = 100_000, xyz_min: float = -1.5, xyz_max: float = 1.5, conf=None, device=None,
                       generator: torch.Generator | None = None) -> dict:
    """init_from_random_point_cloud (model.py:553-611): uniform positions in [xyz_min, xyz_max)^3, albedo = a uniform colour / 255 (no
    RGB2SH), scale = log(max(nearest-neighbour distance, 1e-3) x default_scale_factor), rotations uniform with column 0 set to 1.  Draws
    come from torch's default generator on the device (as the reference's), or from `generator`, in the order positions, colours, NHT
    features, rotations."""
    ft = _feature_type(conf)
    dev = _device(device) if generator is None else generator.device
    n, dtype = int(num_gaussians), torch.float32
    g = {} if generator is None else {"generator": generator}
    pts = torch.rand((n, 3), dtype=dtype, device=dev, **g) * (xyz_max - xyz_min) + xyz_min
    color = torch.rand((n, 3), dtype=dtype, device=dev, **g) / 255.0
    out = {}
    if ft == "sh":
        out["features_albedo"] = color.contiguous()
        out["features_specular"] = torch.zeros((n, SPECULAR_DIM), dtype=dtype, device=dev)
    else:
        lo, hi = float(_get(conf, "model.nht_features.init_min")), float(_get(conf, "model.nht_features.init_max"))
        out["features"] = torch.rand((n, nat.NHT_FEATURE_DIM), dtype=dtype, device=dev, **g) * (hi - lo) + lo
    _, idx = nearest_neighbors(pts, 1)
    dist = torch.clamp_min(torch.linalg.norm(pts - pts[idx[:, 0], :], dim=-1), 1e-3)
    scales = torch.log(dist * float(_get(conf, "model.default_scale_factor")))[..., None].repeat(1, 3)
    rots = torch.rand((n, 4), device=dev, **g)
    rots[:, 0] = 1
    density = _inverse_sigmoid(float(_get(conf, "model.default_density")) * torch.ones((n, 1), dtype=dtype, device=dev))
    out.update(positions=pts, rotation=rots, scale=scales, density=density)
    return _leaves(out, ft)


def apply_points_transform(points: torch.Tensor, transform) -> torch.Tensor:
    """The 4x4 affine `transform` applied to points [N,3] (geometry.py:24-39): p @ T[:3,:3].T + T[:3,3]; None returns the points."""
    if transform is None:
        return points
    if points.ndim != 2 or points.shape[1] != 3:
        raise ValueError(f"points must have shape (N, 3), got {tuple(points.shape)}")
    t = torch.as_tensor(transform, dtype=points.dtype, device=points.device)
    if tuple(t.shape) != (4, 4):
        raise ValueError(f"transform must have shape (4, 4), got {tuple(t.shape)}")
    if not bool(torch.isfinite(t).all()):
        raise ValueError("transform must contain only finite values")
    return points @ t[:3, :3].T + t[:3, 3]


# ---- readers -----------------------------------------------------------------------------------------------------------------------

def read_colmap_points3d_bin(path: str):
    """COLMAP points3D.bin -> (xyz float64 [N,3], rgb uint8 [N,3]).  A record is id u64, xyz 3 x f64, rgb 3 x u8, error f64, track
    length u64 and that many (image, point2D) int32 pairs; the record offsets are chained through the track lengths, so they are walked
    with one small read per point, and the fields are then gathered with numpy."""
    buf = np.fromfile(path, dtype=np.uint8)
    data = buf.tobytes()
    if len(data) < 8:
        raise ValueError(f"{path}: truncated points3D.bin")
    n = struct.unpack_from("<Q", data, 0)[0]
    if 8 + 51 * n > len(data):
        raise ValueError(f"{path}: {n} points do not fit in {len(data)} bytes")
    offs = np.empty(n, dtype=np.int64)
    unpack, off = struct.Struct("<Q").unpack_from, 8
    try:
        for i in range(n):
            offs[i] = off
            off += 51 + 8 * unpack(data, off + 43)[0]
    except struct.error:
        raise ValueError(f"{path}: truncated after {i} of {n} points") from None
    if off > len(data):
        raise ValueError(f"{path}: truncated (records end at byte {off}, the file has {len(data)})")
    xyz = buf[offs[:, None] + np.arange(8, 32)[None, :]].view("<f8").astype(np.float64)
    rgb = buf[offs[:, None] + np.arange(32, 35)[None, :]]
    return xyz, rgb


def read_colmap_points3d_txt(path: str):
    """COLMAP points3D.txt -> (xyz float64 [N,3], rgb uint8 [N,3]); `#` lines are comments."""
    rows = []
    with open(path, "r") as f:
        for line in f:
            line = line.strip()
            if line and line[0] != "#":
                rows.append(line.split()[1:7])
    if not rows:
        return np.zeros((0, 3), np.float64), np.zeros((0, 3), np.uint8)
    xyz = np.array([r[0:3] for r in rows], dtype=np.float64)
    rgb = np.array([r[3:6] for r in rows], dtype=np.int64).astype(np.uint8)
    return xyz, rgb


_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2", "uint16": "u2",
              "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4", "double": "f8", "float64": "f8"}


def _ply_header(f, path):
    if f.readline().strip() != b"ply":
        raise ValueError(f"{path}: not a PLY file")
    fmt, elements = None, []
    while True:
        line = f.readline()
        if not line:
            raise ValueError(f"{path}: PLY header has no end_header")
        tok = line.decode("ascii", "replace").split()
        if not tok or tok[0] in ("comment", "obj_info"):
            continue
        if tok[0] == "end_header":
            return fmt, elements
        if tok[0] == "format":
            fmt = tok[1]
        elif tok[0] == "element":
            elements.append((tok[1], int(tok[2]), []))
        elif tok[0] == "property":
            if tok[1] == "list":
                elements[-1][2].append((tok[4], None, (_PLY_TYPES[tok[2]], _PLY_TYPES[tok[3]])))
            else:
                if tok[1] not in _PLY_TYPES:
                    raise ValueError(f"{path}: unknown PLY property type {tok[1]!r}")
                elements[-1][2].append((tok[2], _PLY_TYPES[tok[1]], None))


def read_ply_vertices(path: str) -> dict:
    """{property name: numpy array [N]} of the `vertex` element of a PLY file in `ascii` or `binary_little_endian` format; other
    elements are skipped.  Any other format raises ValueError naming it."""
    with open(path, "rb") as f:
        fmt, elements = _ply_header(f, path)
        if fmt not in ("ascii", "binary_little_endian"):
            raise ValueError(f"{path}: PLY format {fmt!r} is not read (ascii and binary_little_endian are)")
        for name, count, props in elements:
            if name == "vertex" and any(p[1] is None for p in props):
                raise ValueError(f"{path}: the vertex element has a list property")
            if fmt == "ascii":
                lines = [f.readline() for _ in range(count)]
                if name != "vertex":
                    continue
                table = np.array([ln.split()[: len(props)] for ln in lines], dtype=np.float64).reshape(count, len(props))
                return {p[0]: table[:, j].astype(p[1]) for j, p in enumerate(props)}
            if all(p[1] is not None for p in props):
                dt = np.dtype([(p[0], "<" + p[1]) for p in props])
                raw = f.read(dt.itemsize * count)
                if len(raw) != dt.itemsize * count:
                    raise ValueError(f"{path}: truncated element {name!r}")
                if name == "vertex":
                    rec = np.frombuffer(raw, dtype=dt)
                    return {p[0]: rec[p[0]].copy() for p in props}
                continue
            for _ in range(count):  # an element with list properties (faces): walk its rows
                for _, scalar, lst in props:
                    if scalar is not None:
                        f.read(np.dtype(scalar).itemsize)
                    else:
                        cnt = int(np.frombuffer(f.read(np.dtype(lst[0]).itemsize), dtype="<" + lst[0])[0])
                        f.read(cnt * np.dtype(lst[1]).itemsize)
    raise ValueError(f"{path}: no vertex element")


def read_ply_points(path: str):
    """A vertex PLY -> (xyz float32 [N,3], rgb uint8 [N,3] or None when the file has no red / green / blue)."""
    v = read_ply_vertices(path)
    for key in ("x", "y", "z"):
        if key not in v:
            raise ValueError(f"{path}: the vertex element has no {key!r} property")
    xyz = np.stack([v["x"], v["y"], v["z"]], axis=1).astype(np.float32)
    rgb = np.stack([v["red"], v["green"], v["blue"]], axis=1).astype(np.uint8) if all(c in v for c in ("red", "green", "blue")) else None
    return xyz, rgb


def read_gaussian_ply(path: str) -> dict:
    """A 3DGS Gaussian PLY (init_from_pretrained_point_cloud, model.py:416-550) -> the SH `params` as float32 numpy arrays; the 45
    f_rest_* coefficients are reordered from the file's channel-major (C) layout to the coefficient-major (F) layout the steps store."""
    v = read_ply_vertices(path)
    need = ["x", "y", "z", "opacity", *(f"rot_{i}" for i in range(4)), *(f"scale_{i}" for i in range(3)), *(f"f_dc_{i}" for i in range(3)),
            *(f"f_rest_{i}" for i in range(SPECULAR_DIM))]
    missing = [k for k in need if k not in v]
    if missing:
        raise ValueError(f"{path}: the Gaussian PLY lacks {', '.join(missing)}")
    n = len(v["x"])
    stack = lambda keys: np.stack([v[k] for k in keys], axis=1).astype(np.float32)  # noqa: E731
    spec = stack([f"f_rest_{i}" for i in range(SPECULAR_DIM)]).reshape(n, 3, -1).transpose(0, 2, 1).reshape(n, -1)
    return {"positions": stack(["x", "y", "z"]), "density": v["opacity"].astype(np.float32).reshape(n, 1),
            "rotation": stack([f"rot_{i}" for i in range(4)]), "scale": stack([f"scale_{i}" for i in range(3)]),
            "features_albedo": stack([f"f_dc_{i}" for i in range(3)]), "features_specular": np.ascontiguousarray(spec)}


# ---- dispatch (Trainer.setup_training) ---------------------------------------------------------------------------------------------

def lidar_subsample(n: int, num_points: int, seed: int):
    """The lidar points kept (trainer.py:386-390): all when n <= num_points, else the first num_points of a CPU randperm seeded
    seed_initialization.  Returns None for all."""
    if num_points >= n:
        return None
    return torch.randperm(n, generator=torch.Generator().manual_seed(int(seed)))[:num_points]


def initialize(conf, *, observers=None, points_transform=None, point_cloud=None, device=None) -> dict:
    """The parameters a run starts from, by initialization.method, as Trainer.setup_training computes them (trainer.py:326-401).
    observers: the dataset's get_observer_points() ([M,3]); points_transform: its get_dataset_world_transform (colmap, fused_point_cloud,
    point_cloud); point_cloud: (xyz [N,3], rgb [N,3] uint8 or None) for `lidar`.  Returns the dict of raw leaf tensors the steps take."""
    method = cfg_get(conf, "initialization.method", None)
    if method not in METHODS:
        raise ValueError(f"initialization.method={method!r} is not one of [{', '.join(METHODS)}]")
    ft = _feature_type(conf)
    dev = _device(device)
    use_obs = bool(_get(conf, "initialization.use_observation_points"))
    if method in ("colmap", "lidar") and use_obs and observers is None:
        raise ValueError(f"initialization.method={method!r} with initialization.use_observation_points needs observer points")
    if method == "random":
        return random_point_cloud(int(_get(conf, "initialization.num_gaussians")), float(_get(conf, "initialization.xyz_min")),
                                  float(_get(conf, "initialization.xyz_max")), conf=conf, device=dev)
    if method == "checkpoint":
        import checkpoint

        ckpt = torch.load(cfg_get(conf, "initialization.path", None), map_location=dev, weights_only=False)
        params = checkpoint.from_reference_layout(ckpt, feature_type=ft)["params"]
        return {k: v.detach().to(device=dev, dtype=torch.float32).clone().contiguous() for k, v in params.items()}
    if method == "point_cloud":
        if points_transform is not None:
            raise ValueError("initialization.method='point_cloud' loads complete Gaussian geometry and cannot apply the dataset world "
                             "transform; pass points_transform=None")
        if ft != "sh":
            raise NotImplementedError("model.feature_type='nht': initialization.method='point_cloud' reads SH Gaussians only")
        g = read_gaussian_ply(os.path.join(str(cfg_get(conf, "path", "")), "point_cloud.ply"))
        return {k: torch.from_numpy(g[k]).to(dev).contiguous() for k in schedule.SH_GROUPS}
    obs = None if observers is None else torch.as_tensor(observers, dtype=torch.float32, device=dev)
    if method == "lidar":
        if point_cloud is None:
            raise ValueError("initialization.method='lidar' needs point_cloud=(xyz, rgb)")
        xyz, rgb = point_cloud
        xyz = torch.as_tensor(xyz, dtype=torch.float32)
        rgb = None if rgb is None else torch.as_tensor(rgb)
        keep = lidar_subsample(int(xyz.shape[0]), int(_get(conf, "initialization.num_points")), int(_get(conf, "seed_initialization")))
        if keep is not None:
            xyz = xyz[keep.to(xyz.device)]
            rgb = None if rgb is None else rgb[keep.to(rgb.device)]
        # the colours stay where the caller keeps them: the reference divides them by 255 on the point cloud's device
        return from_points(xyz.to(dev), rgb, obs, conf, use_observer_pts=use_obs)
    if method == "colmap":
        root = str(cfg_get(conf, "path", ""))
        if cfg_get(conf, "dataset.type", None) == "scannetpp":
            xyz, rgb = read_colmap_points3d_txt(os.path.join(root, "colmap", "points3D.txt"))
        else:
            path = os.path.join(root, "sparse/0", "points3D.bin")
            if os.path.isfile(path):
                xyz, rgb = read_colmap_points3d_bin(path)
            else:
                xyz, rgb = read_colmap_points3d_txt(os.path.join(root, "sparse/0", "points3D.txt"))
    else:  # fused_point_cloud
        xyz, rgb = read_ply_points(str(cfg_get(conf, "initialization.fused_point_cloud_path", "")))
        if rgb is None:  # the reference draws these from numpy's unseeded global generator; seeded here so that replicas agree
            rgb = np.random.RandomState(int(_get(conf, "seed_initialization"))).randint(0, 256, size=(len(xyz), 3), dtype=np.uint8)
    pts = apply_points_transform(torch.tensor(xyz, dtype=torch.float32, device=dev), points_transform)
    return from_points(pts, torch.tensor(rgb, dtype=torch.uint8, device=dev), obs, conf, use_observer_pts=use_obs)

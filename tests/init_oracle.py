"""Torch restatement of the reference's two point initialisations, for tests/test_initialization_gpu.py: init_from_random_point_cloud
(threedgrut/model/model.py:553-611) and default_initialize_from_points (:708-780) with the neighbour searches of model/geometry.py.  The
neighbour indices come from scipy's cKDTree in float64 instead of scikit-learn's KD-tree; every other expression is the reference's, on
the same device and with the same generators."""
import numpy as np
import torch
from scipy.spatial import cKDTree

C0 = 0.28209479177387814


def _np(t):
    return t.detach().cpu().numpy().astype(np.float64)


def knn_self(pts, k):
    """[N,k] int64: the k nearest other points (self removed; with duplicates, exactly one index is dropped, as geometry.py does)."""
    p = _np(pts)
    _, nb = cKDTree(p).query(p, k=k + 1)
    nb = nb.reshape(len(p), k + 1)
    mask = nb != np.arange(len(p))[:, None]
    mask[mask.sum(1) == k + 1, -1] = False
    return torch.from_numpy(nb[mask].reshape(len(p), k)).to(pts.device)


def knn_targets(pts, targets):
    _, nb = cKDTree(_np(targets)).query(_np(pts), k=1)
    return torch.from_numpy(np.asarray(nb).reshape(-1)).to(pts.device)


def inverse_sigmoid(x):
    return torch.log(x / (1 - x))


def random_point_cloud(n, xyz_min, xyz_max, default_scale_factor, default_density, nht=False, init_min=-5.0, init_max=5.0, dim=48,
                       device="cuda"):
    dtype = torch.float32
    pts = torch.rand((n, 3), dtype=dtype, device=device) * (xyz_max - xyz_min) + xyz_min
    color = torch.rand((n, 3), dtype=dtype, device=device) / 255.0
    out = {}
    if nht:
        out["features"] = torch.rand((n, dim), dtype=dtype, device=device) * (init_max - init_min) + init_min
    else:
        out["features_albedo"] = color.contiguous()
        out["features_specular"] = torch.zeros((n, 45), dtype=dtype, device=device)
    nb = knn_self(pts, 1)[:, 0]
    dist = torch.clamp_min(torch.linalg.norm(pts - pts[nb, :], dim=-1), 1e-3)
    scales = torch.log(dist * default_scale_factor)[..., None].repeat(1, 3)
    rots = torch.rand((n, 4), device=device)
    rots[:, 0] = 1
    opac = inverse_sigmoid(default_density * torch.ones((n, 1), dtype=dtype, device=device))
    out.update(positions=pts, rotation=rots, scale=scales, density=opac)
    return out, nb[:, None]


def from_points(pts, observer_pts, colors, use_observer_pts, seed, observation_scale_factor, default_scale_factor, default_density, nht=False,
                init_min=-5.0, init_max=5.0, dim=48):
    """Returns (params, the neighbour indices used: [N,1] observers or [N,3] points)."""
    dtype, dev, n = torch.float32, pts.device, pts.shape[0]
    rng = torch.Generator(device=dev).manual_seed(seed)
    rots = torch.rand((n, 4), dtype=dtype, device=dev, generator=rng)
    if use_observer_pts:
        nb = knn_targets(pts, observer_pts)
        dist = torch.clamp_min(torch.linalg.norm(pts - observer_pts[nb, :], dim=-1), 1e-7)
        scale = dist * observation_scale_factor
        nb = nb[:, None]
    else:
        nb = knn_self(pts, 3)
        d = torch.linalg.norm(pts.double()[:, None, :] - pts.double()[nb], dim=-1).to(pts)
        scale = torch.sqrt((d ** 2).mean(dim=-1))
    scale = scale * default_scale_factor
    scales = torch.log(scale)[:, None].repeat(1, 3)
    opac = inverse_sigmoid(torch.full((n, 1), fill_value=default_density, dtype=dtype, device=dev))
    if colors is None:
        colors = torch.randint(0, 256, (n, 3), dtype=torch.uint8, device=dev, generator=rng)
    out = {"positions": pts.clone(), "rotation": rots, "scale": scales, "density": opac}
    if nht:
        out["features"] = torch.rand((n, dim), dtype=dtype, device=dev, generator=rng) * (init_max - init_min) + init_min
    else:
        out["features_albedo"] = torch.from_numpy(((colors.float() / 255.0).cpu().numpy() - 0.5) / C0).to(dev)  # RGB2SH(to_np(...))
        out["features_specular"] = torch.zeros((n, 45), dtype=dtype, device=dev)
    return out, nb

"""Playground: render a trained scene with mirror, glass and diffuse triangle meshes inserted (forward only, DESIGN.md section 22).

Restates the feature set of the reference's Playground v1 (threedgrut_playground/engine.py, src/kernels/cuda/playgroundKernel.cu) on this
library's own tracer: every camera ray alternates a closest hit against an LBVH over the meshes' triangles and the 3DGRT k-nearest walk
over the Gaussians on the segment up to it, and bounces at each surface by the mesh's material (grtb200_trace_playground).

    Mesh      vertices [V,3], faces [F,3], optional vertex normals, a material ("mirror", "glass" with `ior`, "diffuse" with `color`)
              and a 4x4 object-to-world transform; Mesh.sphere / cube / quad / from_obj make one
    Engine    a scene from a `ckpt_*.pt` (ours or the reference's) or an SH Gaussian PLY, the meshes added to it, and render(batch)
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np
import torch

import b200_native as native
from b200_native import cfg_get, ptr

MATERIALS = {"mirror": 0, "glass": 1, "diffuse": 2}  # GRTB200_MATERIAL_* (include/grt_b200.h)

# What a scene is traced with when it does not bring a 3DGRT render section of its own (a 3DGUT checkpoint, a PLY): the reference's
# configs/render/3dgrt.yaml, as load_3dgrt_object applies it
DEFAULT_RENDER = {"method": "3dgrt", "primitive_type": "instances", "particle_kernel_degree": 4, "particle_kernel_min_response": 0.0113,
                  "particle_kernel_max_alpha": 0.99, "particle_kernel_density_clamping": True, "min_transmittance": 0.001,
                  "pipeline_type": "reference", "backward_pipeline_type": "referenceBwd"}


def face_normals(vertices: np.ndarray, faces: np.ndarray) -> np.ndarray:
    """Unit normals [F,3] of the triangles, normalize(cross(v1 - v0, v2 - v0)); zero for a degenerate triangle."""
    v = vertices[faces]
    n = np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])
    ln = np.linalg.norm(n, axis=1, keepdims=True)
    return np.where(ln > 0, n / np.where(ln > 0, ln, 1), 0)


def smooth_normals(vertices: np.ndarray, faces: np.ndarray) -> np.ndarray:
    """Vertex normals [V,3]: the normalised sum of the unit normals of the faces around each vertex."""
    acc = np.zeros_like(vertices, dtype=np.float64)
    fn = face_normals(vertices.astype(np.float64), faces)
    for k in range(3):
        np.add.at(acc, np.asarray(faces)[:, k], fn)
    ln = np.linalg.norm(acc, axis=1, keepdims=True)
    return np.where(ln > 0, acc / np.where(ln > 0, ln, 1), 0)


def read_obj(path: str):
    """A minimal Wavefront OBJ reader: `v`, `vn` and `f` lines (v, v/t, v/t/n or v//n references, 1-based or negative), polygons
    triangulated as fans.  Returns (vertices [V,3] float64, faces [F,3] int64, vertex normals [V,3] or None).  A vertex takes the normal
    its face corners name (the last one read); normals are returned only when every vertex got one."""
    verts, vns, faces, corner_vn = [], [], [], {}
    with open(path) as f:
        for line in f:
            parts = line.split()
            if not parts:
                continue
            if parts[0] == "v":
                verts.append([float(x) for x in parts[1:4]])
            elif parts[0] == "vn":
                vns.append([float(x) for x in parts[1:4]])
            elif parts[0] == "f":
                idx = []
                for ref in parts[1:]:
                    fields = ref.split("/")
                    vi = int(fields[0])
                    vi = vi - 1 if vi > 0 else len(verts) + vi
                    idx.append(vi)
                    if len(fields) > 2 and fields[2]:
                        ni = int(fields[2])
                        corner_vn[vi] = ni - 1 if ni > 0 else len(vns) + ni
                if len(idx) < 3:
                    raise ValueError(f"{path}: a face with {len(idx)} vertices")
                faces.extend([idx[0], idx[k], idx[k + 1]] for k in range(1, len(idx) - 1))
    v = np.asarray(verts, np.float64).reshape(-1, 3)
    fc = np.asarray(faces, np.int64).reshape(-1, 3)
    if fc.size and (fc.min() < 0 or fc.max() >= len(v)):
        raise ValueError(f"{path}: a face names a vertex that does not exist")
    normals = None
    if vns and len(corner_vn) == len(v):
        vn = np.asarray(vns, np.float64)
        normals = vn[[corner_vn[i] for i in range(len(v))]]
    return v, fc, normals


@dataclass
class Mesh:
    """A triangle mesh with one material.  vertices [V,3] and faces [F,3] in object space; normals [V,3] or None (then the smooth normals
    of the faces); material "mirror", "glass" (index of refraction `ior`) or "diffuse" (colour `color`, linear RGB); transform: the 4x4
    object-to-world matrix (normals take its inverse transpose)."""

    vertices: np.ndarray
    faces: np.ndarray
    material: str = "mirror"
    ior: float = 1.33
    color: tuple = (0.8, 0.8, 0.8)
    normals: np.ndarray | None = None
    transform: np.ndarray = field(default_factory=lambda: np.eye(4))

    def __post_init__(self):
        if self.material not in MATERIALS:
            raise NotImplementedError(f"material={self.material!r}: the playground renders {', '.join(MATERIALS)}")
        self.vertices = np.asarray(self.vertices, np.float64).reshape(-1, 3)
        self.faces = np.asarray(self.faces, np.int64).reshape(-1, 3)
        if self.faces.size and (self.faces.min() < 0 or self.faces.max() >= len(self.vertices)):
            raise ValueError("faces name vertices that do not exist")
        if self.normals is not None:
            self.normals = np.asarray(self.normals, np.float64).reshape(-1, 3)
            if self.normals.shape != self.vertices.shape:
                raise ValueError("normals must be [V,3], one per vertex")
        self.transform = np.asarray(self.transform, np.float64).reshape(4, 4)
        self.color = tuple(float(c) for c in self.color)
        self.ior = float(self.ior)

    def world(self):
        """(vertices [V,3], unit vertex normals [V,3]) in world space, float64."""
        m = self.transform
        v = self.vertices @ m[:3, :3].T + m[:3, 3]
        n = self.normals if self.normals is not None else smooth_normals(self.vertices, self.faces)
        n = n @ np.linalg.inv(m[:3, :3])  # (M^-T n^T)^T
        ln = np.linalg.norm(n, axis=1, keepdims=True)
        return v, np.where(ln > 0, n / np.where(ln > 0, ln, 1), 0)

    @classmethod
    def sphere(cls, radius: float = 1.0, stacks: int = 32, slices: int = 64, **kw) -> "Mesh":
        """A UV sphere about the origin: 2 * slices * (stacks - 1) triangles, exact vertex normals."""
        rows = []
        for i in range(stacks + 1):
            th = math.pi * i / stacks
            for j in range(slices):
                ph = 2 * math.pi * j / slices
                rows.append((math.sin(th) * math.cos(ph), math.sin(th) * math.sin(ph), math.cos(th)))
        n = np.asarray(rows)
        faces = []
        for i in range(stacks):
            for j in range(slices):
                a, b = i * slices + j, i * slices + (j + 1) % slices
                c, d = a + slices, b + slices
                if i > 0:
                    faces.append((a, c, b))
                if i < stacks - 1:
                    faces.append((b, c, d))
        return cls(n * radius, np.asarray(faces), normals=kw.pop("normals", n), **kw)

    @classmethod
    def cube(cls, size: float = 1.0, **kw) -> "Mesh":
        """An axis-aligned cube of edge `size` about the origin, 12 triangles, outward winding."""
        h = size / 2
        v = np.array([[x, y, z] for x in (-h, h) for y in (-h, h) for z in (-h, h)], np.float64)
        f = [(0, 1, 3), (0, 3, 2), (4, 6, 7), (4, 7, 5), (0, 4, 5), (0, 5, 1), (2, 3, 7), (2, 7, 6), (0, 2, 6), (0, 6, 4), (1, 5, 7), (1, 7, 3)]
        return cls(v, np.asarray(f), **kw)

    @classmethod
    def quad(cls, size: float = 1.0, **kw) -> "Mesh":
        """A square of edge `size` in the z = 0 plane about the origin, normal +z, 2 triangles."""
        h = size / 2
        v = np.array([[-h, -h, 0], [h, -h, 0], [h, h, 0], [-h, h, 0]], np.float64)
        return cls(v, np.array([(0, 1, 2), (0, 2, 3)]), normals=kw.pop("normals", np.tile([0.0, 0.0, 1.0], (4, 1))), **kw)

    @classmethod
    def from_obj(cls, path: str, **kw) -> "Mesh":
        v, f, n = read_obj(path)
        return cls(v, f, normals=kw.pop("normals", n), **kw)


def pack_meshes(meshes):
    """The arrays grtb200_build_mesh_bvh takes, in numpy: vertices [V,3] f32, vertex normals [V,3] f32, faces [F,3] i32, face material
    [F] i32 (the mesh's index) and the material table [M,8] f32 = (kind, ior, 0, 0, r, g, b, 0)."""
    vs, ns, fs, fm, mats, base = [], [], [], [], [], 0
    for i, m in enumerate(meshes):
        v, n = m.world()
        vs.append(v)
        ns.append(n)
        fs.append(m.faces + base)
        fm.append(np.full(len(m.faces), i))
        mats.append([MATERIALS[m.material], m.ior, 0, 0, *m.color, 0])
        base += len(v)
    cat = lambda xs, shape, dt: np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros(shape), dt)  # noqa: E731
    return (cat(vs, (0, 3), np.float32), cat(ns, (0, 3), np.float32), cat(fs, (0, 3), np.int32), cat(fm, (0,), np.int32),
            np.ascontiguousarray(np.asarray(mats, np.float32).reshape(-1, 8)))


def _plain(conf):
    import evaluate

    return evaluate._plain(conf)


class Engine:
    """A trained scene and the meshes inserted into it.

    source: a `ckpt_*.pt` (ours or the reference's; loaded through evaluate.from_checkpoint) or an SH Gaussian PLY.  A 3DGRT checkpoint is
    traced with its own render section (with evaluation's overrides); anything else with DEFAULT_RENDER.  The background is the
    checkpoint's model.background.color (black for a PLY).  smooth_normals: shade with interpolated vertex normals, else with each
    triangle's own normal.  model.feature_type nht is refused."""

    def __init__(self, source: str, device="cuda", smooth_normals: bool = True):
        background, render = (0.0, 0.0, 0.0), dict(DEFAULT_RENDER)
        if str(source).lower().endswith(".ply"):
            import initialization
            import train_step

            g = {k: torch.from_numpy(v) for k, v in initialization.read_gaussian_ply(source).items()}
            particles, sph, sph_degree = train_step.particle_record(g), torch.cat([g["features_albedo"], g["features_specular"]], 1), 3
        else:
            ckpt = torch.load(source, map_location="cpu", weights_only=False)
            conf = _plain(ckpt.get("config"))
            del ckpt
            ft = str(cfg_get(conf, "model.feature_type", "sh")).lower()
            if ft != "sh":
                raise NotImplementedError(f"model.feature_type={ft!r}: the playground renders SH radiance only")
            import evaluate

            step = evaluate.from_checkpoint(source, device=device)
            if step.background.random:
                raise NotImplementedError("model.background.color='random': the playground composites a fixed background colour")
            particles, sph = step.activated()
            sph_degree, background = int(step.sph_degree), tuple(float(c) for c in step.background.color)
            if str(cfg_get(conf, "render.method", "3dgut")).lower() == "3dgrt":
                render = evaluate.eval_config(conf)["render"]
        self._setup(particles, sph, sph_degree, render, background, device, smooth_normals)

    @classmethod
    def from_gaussians(cls, particles, sph, sph_degree: int = 3, render: dict | None = None, background=(0.0, 0.0, 0.0), device="cuda",
                       smooth_normals: bool = True) -> "Engine":
        """An engine over Gaussians held in memory: particles the activated [N,12] record (pos3, density, quat wxyz, scale3, pad), sph
        [N,48]; render: the 3DGRT render section (DEFAULT_RENDER's keys; missing keys take its values)."""
        eng = cls.__new__(cls)
        eng._setup(torch.as_tensor(particles), torch.as_tensor(sph), sph_degree, {**DEFAULT_RENDER, **(render or {})}, background, device,
                   smooth_normals)
        return eng

    def _setup(self, particles, sph, sph_degree, render, background, device, smooth_normals):
        from threedgrt_tracer.tracer import Tracer

        self.device = torch.device(device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.smooth_normals = bool(smooth_normals)
        self.background = tuple(float(c) for c in background)
        self.sph_degree = int(sph_degree)
        self.conf = {"render": render, "model": {"feature_type": "sh"}}
        with torch.cuda.device(self.device):
            self.tracer = Tracer(self.conf)
            self.particles = particles.detach().to(self.device, torch.float32).contiguous()
            self.sph = sph.detach().to(self.device, torch.float32).contiguous()
            wrapper = self.tracer.tracer_wrapper
            wrapper.set_replay(False, self.device)
            wrapper.build_bvh_packed(self.particles)
            self._ctx = wrapper.native_context(self.device)
            self._bvh = native.MeshBvh(self.device.index)
        self.min_transmittance = self.tracer._min_transmittance
        self.meshes: dict[str, Mesh] = {}
        self._dirty = False

    def add_mesh(self, name: str, mesh: Mesh) -> None:
        """Insert (or replace) the mesh `name`; the mesh BVH is rebuilt before the next render."""
        if not isinstance(mesh, Mesh):
            raise TypeError("add_mesh takes a playground.Mesh")
        self.meshes[name] = mesh
        self._dirty = True

    def remove_mesh(self, name: str) -> None:
        del self.meshes[name]
        self._dirty = True

    def _build_meshes(self):
        v, n, f, fm, mats = pack_meshes(list(self.meshes.values()))
        t = lambda a: torch.from_numpy(a).to(self.device)  # noqa: E731
        v, n, f, fm, mats = t(v), t(n), t(f), t(fm), t(mats)
        stream = torch.cuda.current_stream(self.device).cuda_stream
        self._bvh.build(stream, int(v.shape[0]), ptr(v), ptr(n), int(f.shape[0]), ptr(f), ptr(fm), int(mats.shape[0]), ptr(mats))
        self._dirty = False

    @torch.no_grad()
    def render(self, batch, ray_max_t=None) -> dict:
        """batch: T_to_world [1,4,4] and camera-space rays_ori / rays_dir [1,H,W,3] (what threedgrt_tracer.Tracer.render takes), as
        attributes or dict keys.  ray_max_t: None (1e9) or a [1,H,W] / [1,H,W,1] tensor.  Returns {"rgb": [1,H,W,3], "opacity": [1,H,W,1]},
        composited on the background and clamped to [0, 1]."""
        get = (lambda k: batch[k]) if isinstance(batch, dict) else (lambda k: getattr(batch, k))
        rays_o = get("rays_ori").to(self.device, torch.float32).contiguous()
        rays_d = get("rays_dir").to(self.device, torch.float32).contiguous()
        b, h, w = (int(x) for x in rays_o.shape[:3])
        if b != 1:
            raise ValueError("render takes one view ([1,H,W,3] rays)")
        with torch.cuda.device(self.device):
            if self._dirty:
                self._build_meshes()
            r2w = self.tracer.tracer_wrapper._r2w(get("T_to_world"))
            bg = np.asarray(self.background, np.float32)
            tmax = None if ray_max_t is None else ray_max_t.to(self.device, torch.float32).reshape(b * h * w).contiguous()
            rgb = torch.empty((b, h, w, 3), dtype=torch.float32, device=self.device)
            alpha = torch.empty((b, h, w, 1), dtype=torch.float32, device=self.device)
            n = int(self.particles.shape[0])
            vis = torch.empty((max(n, 1),), dtype=torch.float32, device=self.device)
            stream = torch.cuda.current_stream(self.device).cuda_stream
            self._ctx.trace_playground(stream, self._bvh if self.meshes else None, n, ptr(self.particles), ptr(self.sph), self.sph_degree,
                                       float(self.min_transmittance), b, h, w, ptr(rays_o), ptr(rays_d), r2w.ctypes.data,
                                       None if tmax is None else ptr(tmax), bg.ctypes.data, self.smooth_normals, ptr(rgb), ptr(alpha), ptr(vis))
        return {"rgb": rgb, "opacity": alpha}

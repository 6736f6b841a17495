"""Playground host logic and oracle (no GPU): the oracle's mirror law, Snell refraction and total internal reflection against closed forms,
its brute-force closest hit, the OBJ reader, generated normals, mesh transforms and the refusals."""
import math

import numpy as np
import pytest

import playground as pg
import playground_oracle as po


def _unit(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v)


@pytest.mark.parametrize("angle", [0.0, 0.3, 1.2])
@pytest.mark.parametrize("flip", [False, True])
def test_mirror_law(angle, flip):
    d = np.array([math.sin(angle), 0.0, -math.cos(angle)])
    n = np.array([0.0, 0.0, -1.0 if flip else 1.0])  # either face: the normal is turned against the ray
    r = po.reflect(d, n)
    assert np.allclose(r, [math.sin(angle), 0.0, math.cos(angle)], atol=1e-15)


@pytest.mark.parametrize("ior", [1.33, 1.5, 2.4])
@pytest.mark.parametrize("angle", [0.0, 0.4, 1.0])
def test_snell_refraction_entering_and_leaving(ior, angle):
    n = np.array([0.0, 0.0, 1.0])
    d = np.array([math.sin(angle), 0.0, -math.cos(angle)])  # entering: dot(d, n) < 0
    t, refracted = po.refract(d, n, ior)
    assert refracted
    sin_t = math.sin(angle) * po.N_OUTSIDE / ior
    assert np.allclose(t, [sin_t, 0.0, -math.sqrt(1 - sin_t * sin_t)], atol=1e-12)
    back, refracted = po.refract(-t, n, ior)  # leaving the glass back along the refracted ray retraces it
    assert refracted and np.allclose(back, -d, atol=1e-12)


def test_total_internal_reflection_is_a_mirror_bounce():
    ior = 1.5
    crit = math.asin(po.N_OUTSIDE / ior)
    n = np.array([0.0, 0.0, 1.0])
    for angle, tir in ((crit - 1e-3, False), (crit + 1e-3, True), (1.3, True)):
        d = np.array([math.sin(angle), 0.0, math.cos(angle)])  # inside, heading out: dot(d, n) > 0
        out, refracted = po.refract(d, n, ior)
        assert refracted == (not tir)
        if tir:
            assert np.allclose(out, po.reflect(d, n)) and np.allclose(out, [math.sin(angle), 0.0, -math.cos(angle)])


def test_pass_through_glass_keeps_the_direction():
    d = _unit([0.3, -0.2, -1.0])
    out, refracted = po.refract(d, np.array([0.0, 0.0, 1.0]), po.N_OUTSIDE)
    assert refracted and np.allclose(out, d, atol=1e-12)


def test_brute_force_closest_hit_ties_and_faces():
    # two coincident quads: the lower triangle index wins; the back face counts
    q = pg.Mesh.quad(2.0)
    v = np.concatenate([q.vertices, q.vertices])
    f = np.concatenate([q.faces, q.faces + 4])
    tris = po.packed_triangles(v, f)
    o = np.array([[0.2, 0.3, 1.0], [0.2, 0.3, -1.0], [5.0, 0.0, 1.0]])
    d = np.array([[0.0, 0.0, -1.0], [0.0, 0.0, 1.0], [0.0, 0.0, -1.0]])
    t, u, vv, tri = po.closest_hit(*tris, o, d)
    assert np.allclose(t[:2], 1.0) and tri[0] == tri[1] and tri[0] in (0, 1) and tri[2] == -1 and t[2] == po.T_MAX


def test_obj_reader_fans_polygons_and_reads_normals(tmp_path):
    p = tmp_path / "m.obj"
    p.write_text("# a quad and a triangle\nv 0 0 0\nv 1 0 0\nv 1 1 0\nv 0 1 0\nv 0 0 1\nvn 0 0 1\nvn 1 0 0\n"
                 "f 1//1 2//1 3//1 4//1\nf -5/1/2 -4/1/2 -1/1/2\n")
    v, f, n = pg.read_obj(str(p))
    assert v.shape == (5, 3) and f.tolist() == [[0, 1, 2], [0, 2, 3], [0, 1, 4]]
    assert n is not None and n[4].tolist() == [1, 0, 0] and n[3].tolist() == [0, 0, 1]
    m = pg.Mesh.from_obj(str(p), material="diffuse", color=(1, 0, 0))
    assert m.faces.shape == (3, 3) and m.material == "diffuse"
    p.write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nf 1 2 3\n")
    v, f, n = pg.read_obj(str(p))
    assert n is None and f.tolist() == [[0, 1, 2]]
    p.write_text("v 0 0 0\nv 1 0 0\nf 1 2 7\n")
    with pytest.raises(ValueError):
        pg.read_obj(str(p))


def test_generated_normals():
    q = pg.Mesh.quad(1.0, normals=None)
    assert np.allclose(q.world()[1], [0, 0, 1])
    s = pg.Mesh.sphere(2.0, stacks=24, slices=48, normals=None)
    n = s.world()[1]
    radial = s.vertices / np.linalg.norm(s.vertices, axis=1, keepdims=True)
    assert np.all(np.abs(np.abs((n * radial).sum(1)) - 1) < 2e-2)
    # the normalised sum of unit face normals: a vertex shared by a +z face and a -x face gets (-1, 0, 1) / sqrt(2)
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, -1.0]])
    f = np.array([[0, 1, 2], [0, 2, 3]])
    assert np.allclose(pg.smooth_normals(v, f)[0], _unit([-1, 0, 1]))


def test_mesh_transform_moves_vertices_and_takes_the_inverse_transpose_for_normals():
    th = 0.7
    rot = np.array([[math.cos(th), 0, math.sin(th)], [0, 1, 0], [-math.sin(th), 0, math.cos(th)]])
    m = np.eye(4)
    m[:3, :3] = rot @ np.diag([3.0, 1.0, 0.5])
    m[:3, 3] = [1, 2, 3]
    # a tilted plane z = x: under non-uniform scale its normal is not the rotated-and-scaled normal
    v = np.array([[0, 0, 0], [1, 0, 1], [0, 1, 0.0]])
    mesh = pg.Mesh(v, [[0, 1, 2]], material="mirror", transform=m)
    wv, wn = mesh.world()
    assert np.allclose(wv, v @ m[:3, :3].T + [1, 2, 3])
    e1, e2 = wv[1] - wv[0], wv[2] - wv[0]
    assert np.allclose(wn @ e1, 0, atol=1e-12) and np.allclose(wn @ e2, 0, atol=1e-12)
    assert np.allclose(np.linalg.norm(wn, axis=1), 1)


def test_packing_offsets_faces_and_tabulates_materials():
    a = pg.Mesh.quad(1.0, material="mirror")
    b = pg.Mesh.cube(1.0, material="glass", ior=1.5)
    c = pg.Mesh.cube(1.0, material="diffuse", color=(0.1, 0.2, 0.3))
    v, n, f, fm, mats = pg.pack_meshes([a, b, c])
    assert v.shape == (20, 3) and f.shape == (26, 3) and f.dtype == np.int32 and f[2:14].min() == 4 and f[14:].min() == 12
    assert fm.tolist() == [0] * 2 + [1] * 12 + [2] * 12
    assert mats.shape == (3, 8) and mats[:, 0].tolist() == [0, 1, 2] and mats[1, 1] == np.float32(1.5)
    assert np.allclose(mats[2, 4:7], [0.1, 0.2, 0.3])
    assert pg.Mesh.sphere(1.0, stacks=100, slices=100).faces.shape[0] == 2 * 100 * 99


def test_refusals(tmp_path):
    with pytest.raises(NotImplementedError, match="material='pbr'"):
        pg.Mesh.quad(1.0, material="pbr")
    torch = pytest.importorskip("torch")
    path = tmp_path / "ckpt_nht.pt"
    torch.save({"config": {"model": {"feature_type": "nht"}, "render": {"method": "3dgrt"}}}, path)
    with pytest.raises(NotImplementedError, match="model.feature_type='nht'"):
        pg.Engine(str(path))


def test_oracle_render_diffuse_wall_and_miss():
    """The oracle's loop on an empty scene: a diffuse wall gives c |cos| with alpha 1; a miss gives the background."""
    sc = po.Scene(np.zeros((0, 12)), np.zeros((0, 48)))
    wall = pg.Mesh.quad(4.0, material="diffuse", color=(0.5, 0.25, 1.0))
    v, n, f, fm, mats = pg.pack_meshes([wall])
    tris = po.packed_triangles(v, f)
    d = _unit([0.2, 0.0, -1.0])
    rgb, alpha, path = po.render_ray(sc, tris, n, f, fm, mats, [0, 0, 2.0], d, background=(1, 1, 1))
    assert alpha == 1.0 and np.allclose(rgb, np.array([0.5, 0.25, 1.0]) * abs(d[2])) and path in ([(0, 2)], [(1, 2)])
    rgb, alpha, path = po.render_ray(sc, tris, n, f, fm, mats, [0, 0, 2.0], [0, 0, 1.0], background=(0.2, 0.3, 0.4))
    assert alpha == 0.0 and np.allclose(rgb, [0.2, 0.3, 0.4]) and path == []


def test_oracle_two_facing_mirrors_stop_at_32_bounces():
    sc = po.Scene(np.zeros((0, 12)), np.zeros((0, 48)))
    m1 = pg.Mesh.quad(4.0, material="mirror")
    t = np.eye(4)
    t[2, 3] = 1.0
    m2 = pg.Mesh.quad(4.0, material="mirror", transform=t)
    v, n, f, fm, mats = pg.pack_meshes([m1, m2])
    rgb, alpha, path = po.render_ray(sc, po.packed_triangles(v, f), n, f, fm, mats, [0.1, 0.2, 0.5], _unit([0.01, 0.0, 1.0]))
    assert len(path) == po.MAX_BOUNCES and np.all(np.isfinite(rgb))

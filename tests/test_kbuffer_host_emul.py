"""Runs the DEVICE-side core of the sorted 3DGUT kernels on the host (tests/host_emul/kbuffer_host.cpp compiles
3dgrut_b200/csrc/kbuffer_walk.cuh + hit_math.cuh -- the headers the CUDA kernels are built from -- with g++) and compares it with the
oracle's k-buffer forward / backward.  Written because the kernels themselves could not be run on a GPU in round 1; it covers the buffer
walk, the compositing and the per-hit adjoint, not the thread indexing, the launch or the vector atomics."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import scenes
from helpers import image_error_report, kbuffer_premises, oracle_camera, rel_l2
from oracle import gut_oracle as go

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "host_emul")
ROOT = os.path.dirname(os.path.dirname(HERE))


def _lib():
    so, src = os.path.join(HERE, "libkbuffer_host.so"), os.path.join(HERE, "kbuffer_host.cpp")
    deps = [src] + [os.path.join(ROOT, "3dgrut_b200", "csrc", f) for f in ("kbuffer_walk.cuh", "hit_math.cuh", "gut_common.cuh")]
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in deps):
        cxx = "/opt/gcc/bin/g++" if os.path.exists("/opt/gcc/bin/g++") else "g++"
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        if not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
            pytest.skip("CUDA headers not found")
        subprocess.check_call([cxx, "-std=c++17", "-O2", "-fPIC", "-ffp-contract=off", "-w", f"-I{cuda_inc}", "-shared", "-o", so, src])
    return C.CDLL(so)


def _p(a, t=C.c_float):
    return a.ctypes.data_as(C.POINTER(t))


def _frame(name):
    """(scene, camera-to-world, clone group or None) of the named frame; the Gaussians doubled in size, so that every ray accepts more hits
    than the buffer holds and the per-ray hit order differs from the depth order of the lists."""
    if name == "ragged":  # 75x53: partial tiles on both edges
        sc = scenes.scene_c1(n=400, width=75, height=53)
    else:
        sc = scenes.scene_c1(n=400, width=64, height=48)
    sc.particles[:, 8:11] *= 2.0
    group = None
    if name == "clones":  # copies at the same position: equal hit distances, the buffer's strict insertion order decides
        from test_gut_off_default_gpu import clone_scene

        sc, group = clone_scene(sc, 60, 20, 3)
    return sc, sc.camera(2, 5), group


def _check(name, k, degree, settings=None):
    lib = _lib()
    sc, c2w, group = _frame(name)
    cfg = go.default_config()
    cfg.kernel_degree = degree
    for a, b in (settings or {}).items():
        setattr(cfg, a, b)
    cam, _ = oracle_camera(sc, c2w)
    ro, rd = sc.rays()
    pr = go.project(cfg, cam, sc.particles, sc.sph, 3)
    bn = go.bin_tiles(cfg, cam, pr)
    rgba_ref, dist_ref, hits_ref = go.render_forward_kbuffer(cfg, cam, k, ro, rd, sc.particles, pr, bn)
    label = f"host emulation {name} K={k} deg={degree}"
    pre = kbuffer_premises(label, cfg, cam, k, ro, rd, sc.particles, pr, bn, hits_ref)
    assert pre["over_k"] > 0.5 and pre["longest"] > 32  # the buffer flushes early; the lists span several 32-entry batches of the walk
    assert pre["at_flush"] > 0 or k == 1  # K = 1 drains one hit at most: rays stop at a flush
    assert pre["in_drain"] > 0 or k == 1
    if group is not None:
        sizes = np.bincount(group)[group]
        print(f"[kbuffer] {label}: {int((sizes >= 2).sum())} cloned particles, {int((pr.tiles_count[sizes >= 2] > 0).sum())} of them visible")
        assert (pr.tiles_count[sizes >= 2] > 0).sum() >= 50
    rng = np.random.default_rng(k + degree)
    d_rgba = rng.normal(size=rgba_ref.shape).astype(np.float32)
    d_dist = (0.1 * rng.normal(size=dist_ref.shape)).astype(np.float32)
    dp_ref, _ = go.render_backward_kbuffer(cfg, cam, k, ro, rd, sc.particles, sc.sph, 3, pr, bn, rgba_ref, dist_ref, d_rgba, d_dist)

    inv = np.ascontiguousarray(go.sensor_matrices(cam)[1].reshape(-1), np.float32)  # sensor -> world, 4 columns x 3
    H, W, n = sc.height, sc.width, sc.n
    ro_c, rd_c = np.ascontiguousarray(ro.reshape(-1, 3)), np.ascontiguousarray(rd.reshape(-1, 3))
    parts, rgb = np.ascontiguousarray(sc.particles), np.ascontiguousarray(pr.rgb)
    sv, rg = np.ascontiguousarray(bn.sorted_values), np.ascontiguousarray(bn.ranges.reshape(-1))
    rgba, dist, hits = np.zeros((H, W, 4), np.float32), np.zeros((H, W, 1), np.float32), np.zeros((H, W, 1), np.float32)
    args = (C.c_int(degree), C.c_float(cfg.min_kernel_density), C.c_float(cfg.min_alpha), C.c_float(cfg.max_alpha), C.c_float(cfg.min_transmittance),
            C.c_int(k), C.c_int(W), C.c_int(H), _p(inv), _p(ro_c), _p(rd_c), _p(parts), _p(rgb), _p(sv, C.c_uint32), _p(rg, C.c_uint32))
    lib.kbuffer_host_forward(*args, _p(rgba), _p(dist), _p(hits))
    mean_e, max_e, bad = image_error_report(f"{label} rgba", rgba, rgba_ref)
    assert mean_e <= 1e-5 and max_e <= 2e-2 and bad <= max(3, int(2e-4 * H * W))
    assert float(np.mean(hits == hits_ref)) >= 0.999
    acc = np.zeros((n, 16), np.float64)
    lib.kbuffer_host_backward(*args, _p(rgba_ref), _p(d_rgba), _p(dist_ref), _p(d_dist), _p(acc, C.c_double))
    # the oracle's d_particles = accumulator columns 0..10 + the SH-direction term on the position (G8); compare the columns G8 does not touch
    got = acc[:, 3:11].astype(np.float32)
    e = rel_l2(got, dp_ref[:, 3:11])
    print(f"[kbuffer] {label}: density / rotation / scale gradient rel-L2 {e:.2e} (bar 1e-3)")
    assert e <= 1e-3
    assert np.abs(acc[:, 12:15]).max() > 0


@pytest.mark.parametrize("k,degree", [(1, 2), (3, 2), (4, 2), (16, 2), (16, 4)])
def test_device_core_of_the_sorted_kernels_matches_the_oracle(k, degree):
    """K = 1 (every new hit flushes the previous one), odd K, and K = 16 = kMaxK."""
    _check("c1", k, degree)


@pytest.mark.parametrize("frame,k,settings", [("ragged", 16, {}), ("c1", 3, dict(min_transmittance=0.03)),
                                              ("c1", 16, dict(min_transmittance=0.03)), ("clones", 16, {}), ("clones", 3, {})],
                         ids=["ragged-16", "min_transmittance=0.03-3", "min_transmittance=0.03-16", "clones-16", "clones-3"])
def test_device_core_of_the_sorted_kernels_on_edge_frames(frame, k, settings):
    """A ragged frame; min_transmittance = 0.03 (rays stop at a flush and while the buffer drains, and the backward must stop at the same
    hit); cloned particles (equal hit distances: the strict > of kb_insert fixes which copy is composited first, and so how the gradient
    splits between them)."""
    _check(frame, k, 2, settings)

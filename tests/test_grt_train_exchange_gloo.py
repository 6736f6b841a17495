"""World-size-2 gloo test (CPU) of the 3DGRT training step's gradient exchange (view_parallel.FlatGradientExchange): each rank writes
its view's [N,12] / [N,48] gradients, computed by the CPU 3DGRT reference (grt_oracle_trace_bwd), into the flat buffer; one SUM
all-reduce over 60 N floats must give the serial sum of the two views' gradients, bit-identical on both ranks."""
import os
import socket

import numpy as np
import pytest

torch = pytest.importorskip("torch")
import torch.distributed as dist  # noqa: E402
import torch.multiprocessing as mp  # noqa: E402

import scenes  # noqa: E402
from oracle import gut_oracle as go  # noqa: E402

N, SIZE, VIEWS = 80, 32, 10


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _view_gradients(sc, view):
    """The CPU reference's 3DGRT backward of one view with a seeded image gradient: (d_particles [N,12], d_sph [N,48])."""
    cfg = go.grt_config()
    c2w = np.asarray(sc.camera(view, VIEWS), np.float32)
    ro, rd = sc.rays()
    rgb, alpha, dist_, _, _ = go.grt_trace(cfg, sc.particles, sc.sph, sc.sph_degree, ro[0], rd[0], c2w)
    rng = np.random.default_rng(view)
    d_rgb = rng.normal(size=rgb.shape).astype(np.float32)
    return go.grt_trace_bwd(cfg, sc.particles, sc.sph, sc.sph_degree, ro[0], rd[0], c2w, rgb, alpha, dist_, d_rgb, np.zeros_like(alpha),
                            np.zeros_like(alpha))


def _worker(rank, world, port, out_dir):
    import view_parallel as vp

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sc = scenes.scene_c1(n=N, width=SIZE, height=SIZE)
    (view,) = vp.views_for_rank(step=2, rank=rank, world=world, num_views=VIEWS)
    dp, ds = _view_gradients(sc, view)
    ex = vp.FlatGradientExchange(sc.n, torch.device("cpu"))
    d_particles, d_sph = ex.out()
    assert d_particles.data_ptr() == ex.bucket.flat.data_ptr() and d_sph.data_ptr() == ex.bucket.flat.data_ptr() + 12 * 4 * sc.n
    d_particles.copy_(torch.from_numpy(dp))
    d_sph.copy_(torch.from_numpy(ds))
    calls = []
    real = dist.all_reduce

    def counting_all_reduce(tensor, *args, **kwargs):
        calls.append(int(tensor.numel()))
        return real(tensor, *args, **kwargs)

    dist.all_reduce = counting_all_reduce
    try:
        red_p, red_s = ex.exchange()
    finally:
        dist.all_reduce = real
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), view=view, dp=red_p.numpy(), ds=red_s.numpy(), calls=np.array(calls),
             wire=ex.bytes_on_wire())
    dist.destroy_process_group()


def test_flat_exchange_is_one_all_reduce_and_matches_serial_sum(tmp_path):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [np.load(tmp_path / f"rank{r}.npz") for r in range(world)]
    views = [int(o["view"]) for o in outs]
    assert len(set(views)) == world  # disjoint cameras
    sc = scenes.scene_c1(n=N, width=SIZE, height=SIZE)
    grads = [_view_gradients(sc, v) for v in views]
    dp_sum, ds_sum = grads[0][0] + grads[1][0], grads[0][1] + grads[1][1]
    assert np.abs(dp_sum).max() > 0 and np.abs(ds_sum[:, 3:]).max() > 0  # the views reach the higher SH bands
    for o in outs:
        assert list(o["calls"]) == [60 * N]  # one collective over the whole flat buffer
        assert int(o["wire"]) == 240 * N      # ring all-reduce on 2 ranks: 2 (w-1)/w x 240 B x N
        np.testing.assert_array_equal(o["dp"], dp_sum)  # a two-term sum is exact in any order
        np.testing.assert_array_equal(o["ds"], ds_sum)


def test_flat_exchange_single_rank_is_a_no_op():
    import view_parallel as vp

    ex = vp.FlatGradientExchange(5, torch.device("cpu"))
    ex.d_particles.fill_(1.5)
    ex.d_sph.fill_(-2.0)
    dp, ds = ex.exchange()
    assert ex.bucket.flat.numel() == 60 * 5 and ex.bytes_on_wire() == 0
    assert float(dp.sum()) == 1.5 * 60 and float(ds.sum()) == -2.0 * 240

"""Host logic of the NHT training steps (train_step_nht), no GPU: the settings they refuse, the colour-refinement start step, the decoder's
world ray directions, and the flat gradient exchange with the decoder's gradient as a tail (world-size-2 gloo)."""
import os

import numpy as np
import pytest

import scenes

torch = pytest.importorskip("torch")
import torch.distributed as dist  # noqa: E402
import torch.multiprocessing as mp  # noqa: E402

from test_grt_train_exchange_gloo import _free_port  # noqa: E402


def _conf(**decoder):
    return {"n_iterations": 100, "model": {"feature_type": "nht", "nht_decoder": dict(decoder)}}


@pytest.mark.parametrize("key,value", [("unpremultiply_alpha", True), ("center_ray_encoding", True), ("enabled", False)])
def test_unbuilt_decoder_settings_are_refused_by_name(key, value):
    import train_step_nht as tsn

    with pytest.raises(NotImplementedError, match=f"model.nht_decoder.{key}"):
        tsn.nht_step_settings(_conf(**{key: value}))


def test_a_decoder_that_unpremultiplies_is_refused_and_sh_is_not_an_nht_config():
    import train_step_nht as tsn

    class Dec:
        unpremultiply_alpha = True

    with pytest.raises(NotImplementedError, match="unpremultiply_alpha"):
        tsn.nht_step_settings(_conf(), Dec())
    with pytest.raises(ValueError, match="feature_type"):
        tsn.nht_step_settings({"model": {"feature_type": "sh"}})
    assert tsn.nht_step_settings(_conf(reg_weight=1e-4)) == {"weight_decay": 1e-4, "color_refine_start": None}


def _reference_start(feature_type, n_iterations, steps):
    """Trainer._get_color_refine_start_step (threedgrut/trainer.py:153-163)."""
    if feature_type != "nht":
        return n_iterations
    color_refine_steps = int(steps or 0)
    if color_refine_steps <= 0:
        return n_iterations
    return max(0, n_iterations - color_refine_steps)


@pytest.mark.parametrize("feature_type", ["nht", "sh"])
@pytest.mark.parametrize("n_iterations", [0, 7, 30000])
@pytest.mark.parametrize("steps", [None, 0, -3, 5, 7, 12, 29999, 40000])
def test_color_refine_start_step_is_the_reference_formula(feature_type, n_iterations, steps):
    import train_step_nht as tsn

    conf = {"n_iterations": n_iterations, "model": {"feature_type": feature_type, "nht_decoder": {"color_refine_steps": steps}}}
    assert tsn.color_refine_start_step(conf) == _reference_start(feature_type, n_iterations, steps)
    if feature_type == "nht":
        start = tsn.nht_step_settings(conf)["color_refine_start"]
        assert start == (_reference_start(feature_type, n_iterations, steps) if 0 < int(steps or 0) and n_iterations > 0 else None)


def _einsum_dirs(c2w, rays_d):
    """apply_feature_decoder's directions (threedgrut/utils/render.py:70-83) for one camera-to-world pose."""
    R = torch.from_numpy(np.asarray(c2w, np.float32))[None, :3, :3]
    world = torch.einsum("bij,bhwj->bhwi", R, rays_d)
    return torch.nn.functional.normalize(world, dim=-1).reshape(-1, 3)


@pytest.mark.parametrize("view", [0, 3, 11])
def test_decoder_ray_directions_match_apply_feature_decoder(view):
    import train_step_nht as tsn

    sc = scenes.scene_c1(n=20, width=24, height=16)
    c2w = np.asarray(sc.camera(view, 17), np.float32)
    rays_d = torch.from_numpy(sc.rays()[1])
    want = _einsum_dirs(c2w, rays_d)
    gut = tsn.world_ray_directions(tsn.c2w_rotation_from_pose7(scenes.pose7_from_c2w(c2w)), rays_d)   # 3DGUT: world -> sensor pose
    grt = tsn.world_ray_directions(tsn.c2w_rotation_from_T(torch.from_numpy(c2w)[None]), rays_d)      # 3DGRT: T_to_world
    assert gut.shape == (24 * 16, 3) and grt.shape == (24 * 16, 3)
    assert (gut - want).abs().max().item() <= 1e-6
    assert (grt - want).abs().max().item() <= 1e-6


N, TAIL = 37, 1003


def _rank_grads(rank):
    g = torch.Generator().manual_seed(rank)
    return torch.randn(N, 12, generator=g), torch.randn(N, 48, generator=g), torch.randn(TAIL, generator=g)


def _worker(rank, world, port, out_dir):
    import view_parallel as vp

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ex = vp.FlatGradientExchange(N, torch.device("cpu"), tail=TAIL)
    dp, ds, dt = _rank_grads(rank)
    ex.out()[0].copy_(dp)
    ex.out()[1].copy_(ds)
    ex.d_tail.copy_(dt)
    assert ex.d_tail.data_ptr() == ex.bucket.flat.data_ptr() + 60 * 4 * N
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
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), dp=red_p.numpy(), ds=red_s.numpy(), dt=ex.d_tail.numpy(), calls=np.array(calls),
             wire=ex.bytes_on_wire())
    dist.destroy_process_group()


def test_flat_exchange_with_a_decoder_tail_sums_in_one_all_reduce(tmp_path):
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [np.load(tmp_path / f"rank{r}.npz") for r in range(world)]
    grads = [_rank_grads(r) for r in range(world)]
    for o in outs:
        assert list(o["calls"]) == [60 * N + TAIL]
        assert int(o["wire"]) == 240 * N + 4 * TAIL  # ring all-reduce on 2 ranks: 2 (w-1)/w x bytes
        for key, i in (("dp", 0), ("ds", 1), ("dt", 2)):
            np.testing.assert_array_equal(o[key], (grads[0][i] + grads[1][i]).numpy())  # a two-term sum is exact in any order
    for key in ("dp", "ds", "dt"):
        assert np.array_equal(outs[0][key].view(np.uint32), outs[1][key].view(np.uint32))


def test_flat_exchange_without_a_tail_is_unchanged():
    import view_parallel as vp

    ex = vp.FlatGradientExchange(5, torch.device("cpu"))
    assert ex.tail == 0 and ex.d_tail is None and ex.bucket.flat.numel() == 60 * 5 and len(ex.bucket.views) == 2

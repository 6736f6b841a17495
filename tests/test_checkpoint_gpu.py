"""Checkpoints of the five training steps on the GPU: a run saved at step k and resumed from the file continues bit for bit alongside the
uninterrupted run, across densification, with a compressed schedule and a random background; a state written in the reference's layout and
read back into a fresh step renders the same image bit for bit; two ranks (NCCL) save and resume as identical replicas."""
import io
import os

import numpy as np
import pytest

from helpers import rel_l2
from test_checkpoint import _same
from test_schedule_step_gpu import EXTENT, KINDS, _compressed, _mcmc, _Run

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

SAVE_AT, RESUMED = 17, 26  # MCMC relocates at 20 and 40 and adds at 25; GS densifies and prunes at 20, 30 and 40
STRATEGY = {"gut": "gs", "grt": "mcmc", "gut_nht": "mcmc", "grt_nht": "gs", "hybrid": "gs"}


def _densify_conf(kind):
    import densify

    if STRATEGY[kind] == "mcmc":
        return _mcmc()
    # thresholds low enough that every densification clones or splits Gaussians
    return densify.DensifyConfig(clone_grad_threshold=1e-7, split_grad_threshold=1e-7, densify_start=5, densify_frequency=10, densify_end=60,
                                 prune_start=5, prune_frequency=10, prune_end=60, seed=2)


def _build(run, kind, conf):
    import schedule

    return run.make(run.start(), None, schedule=schedule.TrainingSchedule.from_config(conf, scene_extent=EXTENT), densify_conf=_densify_conf(kind),
                    background="random", background_seed=3, scene_extent=EXTENT)


def _grads(st):
    """What the step's backward wrote for the exchange (and, for NHT, the decoder's gradient)."""
    tail = getattr(st.exchange, "d_tail", None)
    return list(st.exchange.out()) + ([tail] if tail is not None else [])


@pytest.mark.parametrize("kind", KINDS)
def test_a_resumed_run_continues_bit_for_bit(kind, tmp_path):
    """A trains to step SAVE_AT and is saved; B is built as A was and loaded from the file: their states are equal.  Both then train in
    lockstep for RESUMED steps, crossing densification.  The backwards add with float atomics, so two backwards of the same state agree to
    rounding only: B is handed the gradients A's backward wrote, after checking they agree, so that everything after the backward (the
    densifier's statistics, the exchange, Adam, the schedule, densification, the generators) must stay bit-identical."""
    import checkpoint

    run = _Run(kind)
    conf = _compressed(kind)
    a = _build(run, kind, conf)
    for it in range(SAVE_AT):
        run.step(a, it % 6)
    path = str(tmp_path / f"ckpt_{SAVE_AT}.pt")
    checkpoint.save(a, path, conf=conf)
    b = _build(run, kind, conf)
    checkpoint.load(path, b)
    _same(b.state_dict(), a.state_dict(), "loaded")
    assert b.frame == SAVE_AT and b.n == a.n and b.exchange.n == a.n
    if kind in ("grt", "grt_nht", "hybrid"):
        assert b._rebuild and b.num_update_bvh == a.num_update_bvh

    seen, worst = {}, [0.0]
    real_a, real_b = a._update, b._update

    def update_a(*args, **kw):
        seen["grads"] = [t.clone() for t in _grads(a)]
        return real_a(*args, **kw)

    def update_b(*args, **kw):
        for mine, theirs in zip(_grads(b), seen["grads"]):
            worst[0] = max(worst[0], rel_l2(mine.cpu(), theirs.cpu()))
            mine.copy_(theirs)
        return real_b(*args, **kw)

    a._update, b._update = update_a, update_b
    n_saved = a.n
    for it in range(SAVE_AT, SAVE_AT + RESUMED):
        run.step(a, it % 6)
        run.step(b, it % 6)
        _same(b.state_dict(), a.state_dict(), f"step {it}")
    print(f"[resume {kind}] N {n_saved} at the save -> {a.n}, worst gradient rel-L2 {worst[0]:.2e}")
    assert worst[0] <= 1e-4
    assert a.n != n_saved  # densification happened after the resume


@pytest.mark.parametrize("extras", [True, False], ids=["with_extras", "reference_only"])
@pytest.mark.parametrize("kind", KINDS)
def test_the_reference_layout_renders_what_was_trained(kind, extras):
    import checkpoint

    run = _Run(kind)
    conf = _compressed(kind)
    a = _build(run, kind, conf)
    for it in range(12):
        run.step(a, it % 6)
    buf = io.BytesIO()
    ckpt = checkpoint.reference_layout(a.state_dict(), conf=conf)
    if not extras:
        del ckpt[checkpoint.EXTRAS]
    torch.save(ckpt, buf)
    buf.seek(0)
    b = _build(run, kind, conf)
    b.load_state_dict(checkpoint.from_reference_layout(torch.load(buf, map_location=b.device, weights_only=True), feature_type=b.FEATURE_TYPE),
                      assign=True)
    assert b.frame == a.frame and b.sph_degree == a.sph_degree and b.optimizer.lrs == a.optimizer.lrs
    for v in (1, 4):  # held views
        ra, rb = run.render(a, v), run.render(b, v)
        assert torch.equal(ra, rb), v


def _rank_worker(rank, world, port, out_dir):
    import torch.distributed as dist

    import checkpoint
    import view_parallel as vp

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        run = _Run("gut", dev=torch.device("cuda", rank))
        conf = _compressed("gut")

        def train(st, start, stop):
            for it in range(start, stop):
                views = [vp.views_for_rank(it, r, world, 6)[0] for r in range(world)]
                positions = np.stack([np.asarray(run.poses[v][0, :3, 3], np.float32) for v in views])
                st.step(run.rays_o, run.rays_d, run.sensor, run.views7[views[rank]], run.targets[views[rank]], all_sensor_positions=positions)

        a = _build(run, "gut", conf)
        train(a, 0, SAVE_AT)
        path = os.path.join(out_dir, "ckpt.pt")
        checkpoint.save(a, path, conf=conf)
        b = _build(run, "gut", conf)
        checkpoint.load(path, b)
        own = torch.equal(b.background.generator.get_state(), a.background.generator.get_state())
        train(b, SAVE_AT, SAVE_AT + RESUMED)
        torch.cuda.synchronize()
        state = b.state_dict()
        out = {f"{g}.{k}": state[g][k].cpu().numpy() for g in ("params", "exp_avg", "exp_avg_sq") for k in state[g]}
        np.savez(os.path.join(out_dir, f"rank{rank}.npz"), own=own, n=b.n, frame=b.frame, degree=b.sph_degree,
                 lrs=np.array([b.optimizer.lrs[k] for k in sorted(b.optimizer.lrs)]),
                 background=b.background.generator.get_state().numpy(), **out)
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_ranks_save_and_resume_as_identical_replicas(tmp_path):
    import torch.multiprocessing as mp

    from test_grt_train_step_gpu import _free_port

    world = 2
    mp.spawn(_rank_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    outs = [np.load(tmp_path / f"rank{r}.npz") for r in range(world)]
    for r in range(world):
        assert bool(outs[r]["own"]), f"rank {r} did not resume its own background generator"
    assert not np.array_equal(outs[0]["background"], outs[1]["background"])  # seeded background_seed + rank
    for k in outs[0].files:
        if k not in ("own", "background"):
            assert np.array_equal(outs[0][k], outs[1][k]), k
    assert int(outs[0]["frame"]) == SAVE_AT + RESUMED

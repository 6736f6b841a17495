"""View-parallel training plumbing (SURVEY.md section 8e): replicate the Gaussians, give every rank disjoint
cameras, sum the per-Gaussian gradients once per step.  The reference has no multi-GPU path; this is new.

One process per GPU (torchrun); `torch.distributed` with NCCL over NVLink on a multi-GPU node, gloo in the CPU tests.
The only exchange of the path is the gradient sum, so the only collective is one all-reduce over a single flat
bucket holding [N,3]+[N,4]+[N,3]+[N,1]+[N,48] = 59 floats per Gaussian (236 B x N per rank).  The training steps use
CompactGradientExchange (3DGUT, 64 B per Gaussian) and FlatGradientExchange (3DGRT, 240 B per Gaussian)."""
from __future__ import annotations

from typing import Iterable, List, Sequence

import torch
import torch.distributed as dist


def views_for_rank(step: int, rank: int, world: int, num_views: int, views_per_rank: int = 1) -> List[int]:
    """Disjoint camera indices of global step `step`: the step's batch is world*views_per_rank consecutive views
    (mod num_views) dealt round-robin, rank r takes {i : i mod world == r}."""
    base = step * world * views_per_rank
    return [(base + j * world + rank) % num_views for j in range(views_per_rank)]


class GradientBucket:
    """Flat fp32 bucket over a fixed list of parameter shapes; one collective per step, buffers allocated once."""

    def __init__(self, shapes: Sequence[Sequence[int]], device, dtype=torch.float32):
        self.shapes = [tuple(s) for s in shapes]
        self.sizes = [int(torch.Size(s).numel()) for s in self.shapes]
        self.flat = torch.zeros(sum(self.sizes), device=device, dtype=dtype)
        self.views, off = [], 0
        for s, n in zip(self.shapes, self.sizes):
            self.views.append(self.flat[off:off + n].view(s))
            off += n

    def pack(self, grads: Iterable[torch.Tensor]):
        for v, g in zip(self.views, grads):
            v.copy_(g)

    def all_reduce(self, group=None, average: bool = False, async_op: bool = False):
        work = None
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
            work = dist.all_reduce(self.flat, op=dist.ReduceOp.SUM, group=group, async_op=async_op)
            if average and not async_op:
                self.flat.div_(dist.get_world_size(group))
        return work

    def unpack(self) -> List[torch.Tensor]:
        return self.views


def allreduce_gradients(grads: Sequence[torch.Tensor], bucket: GradientBucket | None = None, group=None, average: bool = False):
    """Sum `grads` (list of tensors, same shapes on every rank) over all ranks; returns the reduced tensors."""
    if bucket is None:
        bucket = GradientBucket([g.shape for g in grads], grads[0].device, grads[0].dtype)
    bucket.pack(grads)
    bucket.all_reduce(group=group, average=average)
    return bucket.unpack()


def broadcast_parameters(params: Sequence[torch.Tensor], src: int = 0, group=None):
    """Make replicas bit-identical at start-up (same seed already gives that; this is the belt to the braces)."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        for p in params:
            dist.broadcast(p.data, src=src, group=group)


class CompactGradientExchange:
    """The gradient exchange of the 3DGUT path with 64 instead of 240 bytes per Gaussian on the wire.

    A view's [N,48] SH gradient row is basis16(direction Gaussian <- sensor) x g, g = the masked dL/d(radiance) of the Gaussian in
    that view (gut_render.cu: project_backward_kernel).  So the ranks
      1. run `SplatRaster.trace_bwd_compact`, which writes d_particles [N,12] and g [N,4] into this object's buffers,
      2. all-reduce d_particles (48 B x N) and all-gather g (16 B x N per rank),
      3. rebuild sum_v basis(direction_v) x g_v with `SplatRaster.sph_grad_from_views` -- in view order, identical on every rank.
    `sensor_positions` must list the sensor position of every rank's view of this step in rank order (each rank can compute all of
    them from the step's poses with `SplatRaster.sensor_position`, or they are all-gathered with the batch metadata).

    With `views_per_rank` = V > 1 a step's batch is V views per rank (gradient accumulation, `views_for_rank`): the rank renders them one
    after the other into slot 0..V-1, `submit(slot)` adds the view's d_particles to the running sum and starts the all-gather of its g
    ASYNCHRONOUSLY (NCCL's stream; it overlaps the render of the next view), and `finish` does the ONE all-reduce of the step, waits for
    the gathers and rebuilds the SH gradient over all V x world views.  Per view the exposed exchange is 1/V of an all-reduce + one
    streaming kernel."""

    def __init__(self, raster, n: int, device, group=None, views_per_rank: int = 1):
        self.raster, self.n, self.group = raster, int(n), group
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        self.views_per_rank = int(views_per_rank)
        if self.views_per_rank < 1 or self.views_per_rank * self.world > 64:
            raise ValueError("views_per_rank x world must be in 1..64 (sph_grad_from_views takes at most 64 views)")
        V = self.views_per_rank
        self.d_particles = torch.empty((self.n, 12), dtype=torch.float32, device=device)   # slot 0 writes here: the running sum
        self.d_particles_view = torch.empty((self.n, 12), dtype=torch.float32, device=device) if V > 1 else None
        self.g_slots = torch.empty((V, self.n, 4), dtype=torch.float32, device=device)
        self.g = self.g_slots[0]
        self.g_all = torch.empty((V, self.world, self.n, 4), dtype=torch.float32, device=device)
        self.d_sph = torch.empty((self.n, 48), dtype=torch.float32, device=device)
        self._works = []

    def out(self, slot: int = 0):
        """The (d_particles, g) pair to pass as `out=` to trace_bwd_compact for the rank's `slot`-th view of the step."""
        return (self.d_particles if slot == 0 else self.d_particles_view), self.g_slots[slot]

    def submit(self, slot: int):
        """After trace_bwd_compact(out=self.out(slot)): accumulate, start this view's all-gather without waiting for it."""
        if slot > 0:
            self.d_particles.add_(self.d_particles_view)
        if self.world > 1:
            self._works.append(dist.all_gather_into_tensor(self.g_all[slot].view(-1), self.g_slots[slot].view(-1), group=self.group, async_op=True))
        else:
            self.g_all[slot, 0].copy_(self.g_slots[slot])

    def finish(self, n_active_features: int, particle_density: torch.Tensor, sensor_positions):
        """sensor_positions: [V * world, 3], slot-major (slot 0's ranks first).  Returns the summed (d_particles [N,12], d_sph [N,48])."""
        if self.world > 1:
            dist.all_reduce(self.d_particles, op=dist.ReduceOp.SUM, group=self.group)
            for w in self._works:
                w.wait()
        self._works = []
        self.raster.sph_grad_from_views(n_active_features, particle_density, sensor_positions, self.g_all.view(-1, self.n, 4), out=self.d_sph)
        return self.d_particles, self.d_sph

    def exchange(self, n_active_features: int, particle_density: torch.Tensor, sensor_positions):
        """Single-view step (views_per_rank == 1): submit + finish."""
        self.submit(0)
        return self.finish(n_active_features, particle_density, sensor_positions)

    def bytes_on_wire(self) -> int:
        """Bytes a rank receives + sends per step with ring collectives: all-reduce 2 (w-1)/w x 48 N, all-gathers (w-1) x 16 N per view."""
        w = self.world
        return int(2 * (w - 1) / w * 48 * self.n + self.views_per_rank * (w - 1) * 16 * self.n) if w > 1 else 0


class FlatGradientExchange:
    """The gradient exchange of the 3DGRT path: one SUM all-reduce of 60 floats per Gaussian (240 B x N).

    d_particles [N,12] and d_sph [N,48] are views of one flat fp32 buffer; `OptixTracer.trace_bwd(..., out=self.out())` writes the view's
    gradients straight into it, and `exchange` sums the buffer over the ranks in place.  The compact 64-byte exchange of the 3DGUT path does
    not apply: there a Gaussian's SH gradient in one view is basis(one direction) x g, while 3DGRT evaluates the radiance along every ray
    that hits the Gaussian, so its SH gradient is a sum over rays with different directions and has no 4-float summary."""

    def __init__(self, n: int, device, group=None, tail: int = 0):
        """tail: floats of one more gradient after the per-Gaussian rows, summed in the same all-reduce (`d_tail`, e.g. the NHT feature
        decoder's parameter gradient); 0 for none."""
        self.n, self.group, self.tail = int(n), group, int(tail)
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        self.bucket = GradientBucket([(self.n, 12), (self.n, 48)] + ([(self.tail,)] if self.tail else []), device)
        self.d_particles, self.d_sph = self.bucket.views[:2]
        self.d_tail = self.bucket.views[2] if self.tail else None

    def out(self):
        """The (d_particles, d_sph) pair to pass as `out=` to OptixTracer.trace_bwd."""
        return self.d_particles, self.d_sph

    def exchange(self):
        """Sums the buffer over the ranks (no-op on one rank), the tail included; returns (d_particles [N,12], d_sph [N,48])."""
        self.bucket.all_reduce(group=self.group)
        return self.d_particles, self.d_sph

    def bytes_on_wire(self) -> int:
        """Bytes a rank sends + receives per step with a ring all-reduce: 2 (w-1)/w x (240 N + 4 tail)."""
        w = self.world
        return int(2 * (w - 1) / w * (240 * self.n + 4 * self.tail)) if w > 1 else 0

"""Replica-consistent densification / pruning / density reset for view-parallel training (SURVEY.md section 8f row 1).

Restates the GS strategy of the reference (threedgrut/strategy/gs.py:60-328, base.py:78-107, utils/misc.py:212-216,
configs/strategy/gs.yaml) on a plain dict of raw parameter tensors plus the moment dicts of the optimizer, and makes it safe for
several replicas:

  * `update_gradient_buffer` runs on every rank with ITS OWN view's position gradient and sensor position BEFORE the gradient exchange
    (the buffer weights the gradient by the distance to that view's sensor, gs.py:127-137);
  * `densify` first sums the accumulators over the ranks, so every replica takes the same clone / split decisions, and draws the split
    offsets from a generator every rank seeds identically -- replicas stay bit-identical without ever exchanging parameters;
  * prune / reset / decay depend only on the (identical) parameters.

Device-agnostic torch code (the CPU tests run it under gloo); no kernels here."""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.distributed as dist

GROUPS = ("positions", "density", "rotation", "scale", "features_albedo", "features_specular")


@dataclass
class DensifyConfig:  # configs/strategy/gs.yaml
    clone_grad_threshold: float = 0.0002
    split_grad_threshold: float = 0.0002
    relative_size_threshold: float = 0.01
    split_n_gaussians: int = 2
    prune_density_threshold: float = 0.005
    new_max_density: float = 0.01
    density_decay_gamma: float = 0.98
    densify_start: int = 500
    densify_end: int = 15000
    densify_frequency: int = 300
    prune_start: int = 500
    prune_end: int = 15000
    prune_frequency: int = 100
    reset_start: int = 0
    reset_frequency: int = 3000
    seed: int = 0


def check_step_condition(step: int, start: int, end: int, freq: int) -> bool:  # utils/misc.py:212-216
    return bool((start >= 0 and step > start) and (step < end or end == -1) and step % freq == 0)


def load_generator(generator: torch.Generator, state, seed: int) -> None:
    """Restore a generator from get_state()'s byte tensor (on any device), or seed it `seed` when there is none."""
    if state is None:
        generator.manual_seed(int(seed))
    else:
        generator.set_state(state.detach().to("cpu", torch.uint8))


def quaternion_to_so3(q: torch.Tensor) -> torch.Tensor:
    """utils/misc.py quaternion_to_so3: rotation matrices of (unnormalised) w,x,y,z quaternions, normalised first."""
    q = torch.nn.functional.normalize(q, dim=1)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack([
        1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=1)
    return R.reshape(-1, 3, 3)


class GSDensifier:
    """params: dict of raw tensors (GROUPS, or the NHT model's optimizers.NHT_GROUPS: every group in the dict is densified); moments:
    list of dicts with the same keys (e.g. [opt.exp_avg, opt.exp_avg_sq]).
    Every mutating call replaces the tensors inside those dicts in place of the old ones (the dict objects stay the same, so an optimizer
    holding them sees the new tensors)."""

    METHOD = "gs"  # strategy.method

    def __init__(self, params: dict, moments: list, conf: DensifyConfig | None = None, group=None):
        self.params, self.moments, self.conf, self.group = params, moments, conf or DensifyConfig(), group
        dev = params["positions"].device
        n = params["positions"].shape[0]
        self.grad_norm_accum = torch.zeros((n, 1), dtype=torch.float32, device=dev)
        self.grad_norm_denom = torch.zeros((n, 1), dtype=torch.int32, device=dev)
        self.generator = torch.Generator(device=dev)
        self.generator.manual_seed(int(self.conf.seed))

    def state_dict(self) -> dict:
        """The gradient statistics (gs.py:42-57) and the split generator's state; the tensors are the densifier's own."""
        return {"grad_norm_accum": self.grad_norm_accum, "grad_norm_denom": self.grad_norm_denom, "generator": self.generator.get_state()}

    def load_state_dict(self, state: dict | None) -> None:
        """Copies of the state's buffers for the current N (load the parameters first).  A missing buffer is zeroed and a missing
        generator state re-seeded, as the constructor does (a reference checkpoint carries no generator)."""
        state = state or {}
        dev, n = self.params["positions"].device, self.n
        accum, denom = state.get("grad_norm_accum"), state.get("grad_norm_denom")
        if accum is None or denom is None:
            self._reset_buffers()
        else:
            for name, t in (("grad_norm_accum", accum), ("grad_norm_denom", denom)):
                if tuple(t.shape) != (n, 1):
                    raise ValueError(f"densifier {name}: expected shape {(n, 1)}, got {tuple(t.shape)}")
            self.grad_norm_accum = accum.detach().to(device=dev, dtype=torch.float32, copy=True).contiguous()
            self.grad_norm_denom = denom.detach().to(device=dev, dtype=torch.int32, copy=True).contiguous()
        load_generator(self.generator, state.get("generator"), self.conf.seed)

    # ---- activations of the reference model (model.py:102-118)
    def scale(self):
        return torch.exp(self.params["scale"])

    def density(self):
        return torch.sigmoid(self.params["density"])

    @property
    def n(self) -> int:
        return int(self.params["positions"].shape[0])

    # ---- gs.py:127-137
    @torch.no_grad()
    def update_gradient_buffer(self, positions_grad: torch.Tensor, sensor_position) -> None:
        sensor_position = torch.as_tensor(sensor_position, dtype=torch.float32, device=positions_grad.device)
        mask = (positions_grad != 0).max(dim=1)[0]
        distance = (self.params["positions"][mask] - sensor_position).norm(dim=1, keepdim=True)
        self.grad_norm_accum[mask] += torch.norm(positions_grad[mask] * distance, dim=-1, keepdim=True) / 2
        self.grad_norm_denom[mask] += 1

    def _sync_buffers(self):
        if dist.is_available() and dist.is_initialized() and dist.get_world_size(self.group) > 1:
            dist.all_reduce(self.grad_norm_accum, op=dist.ReduceOp.SUM, group=self.group)
            dist.all_reduce(self.grad_norm_denom, op=dist.ReduceOp.SUM, group=self.group)

    def _apply(self, param_fn, moment_fn, names=None):
        """base.py:78-107 on dicts: param_fn(name, tensor) -> new tensor, moment_fn(tensor) -> new tensor (None = keep).  names: every
        group of the parameter dict (GROUPS for the SH model, optimizers.NHT_GROUPS for NHT) unless given."""
        for name in (list(self.params) if names is None else names):
            if moment_fn is not None:
                for m in self.moments:
                    m[name] = moment_fn(m[name]).contiguous()
            if param_fn is not None:
                self.params[name] = param_fn(name, self.params[name]).contiguous()

    def _reset_buffers(self):
        dev = self.params["positions"].device
        self.grad_norm_accum = torch.zeros((self.n, 1), dtype=torch.float32, device=dev)
        self.grad_norm_denom = torch.zeros((self.n, 1), dtype=torch.int32, device=dev)

    # ---- gs.py:139-151
    @torch.no_grad()
    def densify(self, scene_extent: float) -> None:
        self._sync_buffers()
        grad_norm = self.grad_norm_accum / self.grad_norm_denom
        grad_norm[grad_norm.isnan()] = 0.0
        self.clone(grad_norm.squeeze(1), scene_extent)
        self.split(grad_norm.squeeze(1), scene_extent)

    # ---- gs.py:200-225
    @torch.no_grad()
    def clone(self, grad_norm: torch.Tensor, scene_extent: float) -> int:
        mask = grad_norm >= self.conf.clone_grad_threshold
        mask = torch.logical_and(mask, torch.max(self.scale(), dim=1).values <= self.conf.relative_size_threshold * scene_extent)
        k = int(mask.sum())
        self._apply(lambda name, p: torch.cat([p, p[mask]]), lambda v: torch.cat([v, torch.zeros((k, *v.shape[1:]), dtype=v.dtype, device=v.device)]))
        self._reset_buffers()
        return k

    # ---- gs.py:153-198
    @torch.no_grad()
    def split(self, grad_norm: torch.Tensor, scene_extent: float) -> int:
        n_init, ns = self.n, int(self.conf.split_n_gaussians)
        dev = self.params["positions"].device
        padded = torch.zeros(n_init, device=dev)
        padded[: grad_norm.shape[0]] = grad_norm  # the clones appended by clone() carry no gradient statistics
        mask = padded >= self.conf.split_grad_threshold
        mask = torch.logical_and(mask, torch.max(self.scale(), dim=1).values > self.conf.relative_size_threshold * scene_extent)
        stds = self.scale()[mask].repeat(ns, 1)
        samples = torch.randn(stds.shape, generator=self.generator, device=dev) * stds  # torch.normal(mean=0, std=stds), shared seed
        rots = quaternion_to_so3(self.params["rotation"][mask]).repeat(ns, 1, 1)
        offsets = torch.bmm(rots, samples.unsqueeze(-1)).squeeze(-1)
        k = int(mask.sum())

        def param_fn(name, p):
            repeats = [ns] + [1] * (p.dim() - 1)
            if name == "positions":
                new = p[mask].repeat(repeats) + offsets
            elif name == "scale":
                new = torch.log(torch.exp(p[mask].repeat(repeats)) / (0.8 * ns))
            else:
                new = p[mask].repeat(repeats)
            return torch.cat([p[~mask], new])

        self._apply(param_fn, lambda v: torch.cat([v[~mask], torch.zeros((ns * k, *v.shape[1:]), dtype=v.dtype, device=v.device)]))
        self._reset_buffers()
        return k

    # ---- gs.py:268-283
    @torch.no_grad()
    def prune_opacity(self) -> int:
        mask = self.density().squeeze(1) >= self.conf.prune_density_threshold
        self._apply(lambda name, p: p[mask], lambda v: v[mask])
        self.grad_norm_accum, self.grad_norm_denom = self.grad_norm_accum[mask], self.grad_norm_denom[mask]
        return int((~mask).sum())

    # ---- gs.py:303-313
    @torch.no_grad()
    def decay_density(self) -> None:
        def param_fn(name, p):
            d = self.density() * self.conf.density_decay_gamma
            return torch.log(d / (1 - d))

        self._apply(param_fn, None, names=("density",))

    # ---- gs.py:315-328
    @torch.no_grad()
    def reset_density(self) -> None:
        cap = float(torch.log(torch.tensor(self.conf.new_max_density) / (1 - torch.tensor(self.conf.new_max_density))))
        self._apply(lambda name, p: torch.clamp(p, max=cap), lambda v: torch.zeros_like(v), names=("density",))

    # ---- gs.py:74-125: what runs after the optimizer step; returns True when the number of Gaussians may have changed
    def post_optimizer_step(self, step: int, scene_extent: float, positions_lr: float = 0.0) -> bool:
        c, changed = self.conf, False
        if check_step_condition(step, c.densify_start, c.densify_end, c.densify_frequency):
            self.densify(scene_extent)
            changed = True
        if check_step_condition(step, c.prune_start, c.prune_end, c.prune_frequency):
            self.prune_opacity()
            changed = True
        if check_step_condition(step, c.reset_start, c.densify_end, c.reset_frequency):
            self.reset_density()
        return changed


# ---------------------------------------------------------------------------------------------------------------------------------------
# MCMC strategy (threedgrut/strategy/mcmc.py:50-224, strategy/src/gaussian_mcmc.cu:36-70, configs/strategy/mcmc.yaml), replica-consistent:
# every random draw (multinomial sampling of the relocation targets, the positional noise) comes from a generator all ranks seed
# identically and every decision depends only on the (identical) parameters, so replicas stay bit-identical.

@dataclass
class MCMCConfig:  # configs/strategy/mcmc.yaml
    binom_n_max: int = 51
    opacity_threshold: float = 0.005
    relocate_start: int = 500
    relocate_end: int = 25000
    relocate_frequency: int = 100
    add_start: int = 500
    add_end: int = 25000
    add_frequency: int = 100
    max_n_gaussians: int = 1_000_000
    perturb_start: int = 0
    perturb_end: int = 27500
    perturb_frequency: int = 1
    noise_lr: float = 500000.0
    seed: int = 0


def compute_relocation(opacities: torch.Tensor, scales: torch.Tensor, ratios: torch.Tensor, binoms: torch.Tensor):
    """compute_relocation_kernel (gaussian_mcmc.cu:36-70), vectorised: new opacity 1 - (1 - o)^(1/n); new scale = o / denom * scale with
    denom = sum_{i=1..n} sum_{k<i} C(i-1, k) (-1)^k / sqrt(k+1) * new_opacity^(k+1)."""
    n_max = binoms.shape[0]
    n = ratios.to(torch.int64).reshape(-1)
    o = opacities.reshape(-1)
    new_o = 1.0 - torch.pow(1.0 - o, 1.0 / n.to(o.dtype))
    k = torch.arange(n_max, device=o.device)
    coeff = torch.pow(-1.0, k.to(o.dtype)) / torch.sqrt(k.to(o.dtype) + 1.0)              # [K]
    powers = torch.pow(new_o[:, None], (k + 1).to(o.dtype)[None, :])                         # [M, K]
    cum_binoms = torch.cumsum(binoms, dim=0)                                                 # row i-1: sum_{j<i} C(j, k)
    rows = cum_binoms[(n - 1).clamp(min=0, max=n_max - 1)]                                   # [M, K]
    denom = (rows * coeff[None, :] * powers).sum(1)
    return new_o.reshape(opacities.shape), (o / denom)[:, None] * scales


class MCMCDensifier:
    """Same contract as GSDensifier: operates on the raw parameter dict and the optimizer's moment dicts."""

    METHOD = "mcmc"  # strategy.method

    def __init__(self, params: dict, moments: list, conf: MCMCConfig | None = None, group=None):
        import math

        self.params, self.moments, self.conf, self.group = params, moments, conf or MCMCConfig(), group
        dev = params["positions"].device
        n_max = int(self.conf.binom_n_max)
        self.binoms = torch.tensor([[math.comb(n, k) if k <= n else 0 for k in range(n_max)] for n in range(n_max)], dtype=torch.float32, device=dev)
        self.generator = torch.Generator(device=dev)
        self.generator.manual_seed(int(self.conf.seed))

    def state_dict(self) -> dict:
        """The generator's state: all the strategy carries between calls (the binomial table follows from the config)."""
        return {"generator": self.generator.get_state()}

    def load_state_dict(self, state: dict | None) -> None:
        """A missing generator state is re-seeded as the constructor does."""
        load_generator(self.generator, (state or {}).get("generator"), self.conf.seed)

    @property
    def n(self) -> int:
        return int(self.params["positions"].shape[0])

    def update_gradient_buffer(self, positions_grad, sensor_position) -> None:  # the MCMC strategy keeps no gradient statistics
        return None

    def _sample(self, count: int, valid_indices: torch.Tensor | None):
        """sample_new_gaussians (mcmc.py:188-222)"""
        densities = torch.sigmoid(self.params["density"])
        scales = torch.exp(self.params["scale"])
        if valid_indices is None:
            valid_indices = torch.arange(densities.shape[0], device=densities.device)
        probabilities = densities[valid_indices].flatten()
        picked = torch.multinomial(probabilities, count, replacement=True, generator=self.generator)
        sampled = valid_indices[picked]
        ratios = (torch.bincount(sampled)[sampled] + 1).clamp_(min=1, max=self.conf.binom_n_max).int()
        new_o, new_s = compute_relocation(densities[sampled, 0], scales[sampled], ratios, self.binoms)
        new_o = torch.clamp(new_o, max=1.0 - torch.finfo(torch.float32).eps, min=self.conf.opacity_threshold)
        return sampled, torch.log(new_o / (1.0 - new_o))[:, None], torch.log(new_s)

    @torch.no_grad()
    def relocate(self) -> int:
        """mcmc.py:104-131: dead Gaussians (opacity <= threshold) jump onto live ones sampled by opacity"""
        densities = torch.sigmoid(self.params["density"])[:, 0]
        dead = torch.where(densities <= self.conf.opacity_threshold)[0]
        alive = torch.where(densities > self.conf.opacity_threshold)[0]
        if len(dead) == 0 or len(alive) == 0:
            return 0
        sampled, new_d, new_s = self._sample(len(dead), alive)
        for name in list(self.params):  # every group the dict holds (SH or NHT features)
            p = self.params[name]
            if name == "density":
                p[sampled] = new_d
            elif name == "scale":
                p[sampled] = new_s
            p[dead] = p[sampled]
            for m in self.moments:
                m[name][sampled] = 0
        return int(len(dead))

    @torch.no_grad()
    def add(self) -> int:
        """mcmc.py:133-160: grow by 5 % up to max_n_gaussians, new Gaussians are copies of opacity-sampled ones"""
        cur = self.n
        target = min(int(self.conf.max_n_gaussians), int(1.05 * cur))
        count = max(0, target - cur)
        if count == 0:
            return 0
        sampled, new_d, new_s = self._sample(count, None)
        for name in list(self.params):  # every group the dict holds (SH or NHT features)
            p = self.params[name]
            if name == "density":
                p[sampled] = new_d
            elif name == "scale":
                p[sampled] = new_s
            self.params[name] = torch.cat([p, p[sampled]]).contiguous()
            for m in self.moments:
                m[name] = torch.cat([m[name], torch.zeros((count, *m[name].shape[1:]), dtype=m[name].dtype, device=m[name].device)]).contiguous()
        return count

    @torch.no_grad()
    def perturb(self, positions_lr: float) -> None:
        """mcmc.py:162-186: covariance-shaped noise on the positions, gated towards low-opacity Gaussians"""
        scales = torch.exp(self.params["scale"])
        R = quaternion_to_so3(self.params["rotation"])
        S = torch.diag_embed(scales)
        cov = R @ S @ S.transpose(1, 2) @ R.transpose(1, 2)
        densities = torch.sigmoid(self.params["density"])
        gate = 1 / (1 + torch.exp(-100 * ((1 - densities) - 0.995)))
        pos = self.params["positions"]
        noise = torch.randn(pos.shape, generator=self.generator, device=pos.device, dtype=pos.dtype) * gate * self.conf.noise_lr * positions_lr
        pos.add_(torch.bmm(cov, noise.unsqueeze(-1)).squeeze(-1))

    def post_optimizer_step(self, step: int, scene_extent: float = 1.0, positions_lr: float = 0.0) -> bool:
        c, changed = self.conf, False
        if check_step_condition(step, c.relocate_start, c.relocate_end, c.relocate_frequency):
            self.relocate()
        if check_step_condition(step, c.add_start, c.add_end, c.add_frequency):
            changed = self.add() > 0
        if check_step_condition(step, c.perturb_start, c.perturb_end, c.perturb_frequency):
            self.perturb(positions_lr)
        return changed

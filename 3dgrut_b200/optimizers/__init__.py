"""Optimizer step of the Gaussian parameters on the GPU (SURVEY.md section 8f row 2).

`SelectiveAdam` mirrors threedgrut/optimizers/__init__.py:42-124 (same constructor, `step(visibility)`), backed by
gutb200_selective_adam_update instead of the reference's lib_optimizers_cc plugin.
`FusedGaussianAdam` (ours) takes the renderer's gradients directly -- [N,12] and [N,48] w.r.t. the activated values, e.g. straight out of
the view-parallel exchange -- and performs the activation chain rule and the Adam update of all six parameter tensors in one launch.
No CPU fallback: both raise if the tensors are not CUDA tensors or the library is missing."""
from __future__ import annotations

import ctypes as C

import torch

import b200_native as native

GROUPS = ("positions", "density", "rotation", "scale", "features_albedo", "features_specular")
WIDTHS = (3, 1, 4, 3, 3, 45)


def _check(t: torch.Tensor, what: str):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
        raise RuntimeError(f"{what}: expected a contiguous float32 CUDA tensor (there is no CPU fallback)")


def selective_adam_update(param, param_grad, exp_avg, exp_avg_sq, visibility, lr, beta1, beta2, eps):
    """lib_optimizers_cc.selective_adam_update (threedgrut/optimizers/optimizers.cpp): in-place update of param / exp_avg / exp_avg_sq."""
    for t, w in ((param, "param"), (param_grad, "param_grad"), (exp_avg, "exp_avg"), (exp_avg_sq, "exp_avg_sq")):
        _check(t, w)
    n = int(param.shape[0]) if param.dim() > 0 else 0
    m = int(param.numel() // n) if n else 1
    vis = visibility.to(torch.bool).reshape(-1).contiguous()
    if vis.numel() != n:
        raise RuntimeError("visibility must have one entry per row of param")
    stream = torch.cuda.current_stream(param.device).cuda_stream
    with torch.cuda.device(param.device):
        rc = native.load().gutb200_selective_adam_update(stream, param.data_ptr(), param_grad.data_ptr(), exp_avg.data_ptr(), exp_avg_sq.data_ptr(),
                                                  vis.data_ptr(), float(lr), float(beta1), float(beta2), float(eps), n, m)
    if rc != 0:
        raise RuntimeError(f"gutb200_selective_adam_update failed ({rc})")


class SelectiveAdam(torch.optim.Adam):
    """threedgrut.optimizers.SelectiveAdam with the native kernel underneath (one tensor per parameter group, as in the reference)."""

    def __init__(self, params, lr=0.001, betas=(0.9, 0.999), eps=1e-08):
        super().__init__(params=params, lr=lr, eps=eps, betas=betas)
        native.load()  # fail now if the library is missing

    @torch.no_grad()
    def step(self, visibility):
        for group in self.param_groups:
            lr, eps = group["lr"], group["eps"]
            beta1, beta2 = group["betas"]
            assert len(group["params"]) == 1, "More than one tensor in group is not supported"
            param = group["params"][0]
            if param.grad is None:
                continue
            state = self.state[param]
            if len(state) == 0:
                state["step"] = torch.tensor(0.0, dtype=torch.float32)
                state["exp_avg"] = torch.zeros_like(param, memory_format=torch.preserve_format)
                state["exp_avg_sq"] = torch.zeros_like(param, memory_format=torch.preserve_format)
            if not param.is_contiguous() or not state["exp_avg"].is_contiguous():
                raise RuntimeError("SelectiveAdam: parameters and state must be contiguous (the update is in place)")
            selective_adam_update(param.data, param.grad.contiguous(), state["exp_avg"], state["exp_avg_sq"], visibility, lr, beta1, beta2, eps)


class FusedGaussianAdam:
    """One-launch optimizer step for the SH Gaussian model.

    params: dict name -> raw (pre-activation) leaf tensor for the six GROUPS; lrs: dict name -> learning rate (mutable: schedulers
    write `opt.lrs["positions"] = ...`).  step(d_particles, d_sph, visibility=None) consumes the renderer's gradients
    (Tracer / SplatRaster.trace_bwd outputs, or the view-parallel exchange's) -- no autograd pass over the activations is needed.
    lambda_opacity / lambda_scale add the reference's regularisers lambda_opacity mean(sigmoid(density)) + lambda_scale mean(exp(scale))
    (trainer.py:722-736) to the gradient inside the same launch."""

    def __init__(self, params: dict, lrs: dict, betas=(0.9, 0.999), eps=1e-15, selective=False):
        # the dict itself is kept (not copied) when it holds exactly the six groups: densification replaces the tensors inside it
        self.params = params if set(params.keys()) == set(GROUPS) else {k: params[k] for k in GROUPS}
        self._validate()
        self.lrs = {k: float(lrs[k]) for k in GROUPS}
        self.betas, self.eps, self.selective = (float(betas[0]), float(betas[1])), float(eps), bool(selective)
        self.exp_avg = {k: torch.zeros_like(t.data) for k, t in self.params.items()}
        self.exp_avg_sq = {k: torch.zeros_like(t.data) for k, t in self.params.items()}
        self.steps = 0
        native.load()

    @property
    def n(self) -> int:
        return int(self.params["positions"].shape[0])

    def _validate(self):
        n = self.n
        for k, w in zip(GROUPS, WIDTHS):
            t = self.params[k]
            _check(t.data, k)
            if tuple(t.shape) != (n, w):
                raise RuntimeError(f"{k}: expected shape {(n, w)}, got {tuple(t.shape)}")

    def _array(self, tensors):
        arr = (C.c_void_p * 6)()
        for i, k in enumerate(GROUPS):
            arr[i] = tensors[k].data_ptr()
        return arr

    @torch.no_grad()
    def step(self, d_particles: torch.Tensor, d_sph: torch.Tensor, visibility: torch.Tensor | None = None, lambda_opacity: float = 0.0,
             lambda_scale: float = 0.0):
        _check(d_particles, "d_particles")
        _check(d_sph, "d_sph")
        self._validate()  # the tensors may have been replaced (densification); moments must have followed
        for k in GROUPS:
            if self.exp_avg[k].shape != self.params[k].shape or self.exp_avg_sq[k].shape != self.params[k].shape:
                raise RuntimeError(f"{k}: optimizer state does not match the parameter shape {tuple(self.params[k].shape)}")
        if tuple(d_particles.shape) != (self.n, 12) or tuple(d_sph.shape) != (self.n, 48):
            raise RuntimeError("gradient shapes must be [N,12] and [N,48]")
        vis_ptr = None
        if self.selective:
            if visibility is None:
                raise RuntimeError("selective mode needs the renderer's visibility")
            vis = visibility.reshape(-1)
            if vis.dtype != torch.float32:
                vis = vis.to(torch.float32)
            vis = vis.contiguous()
            _check(vis, "visibility")
            vis_ptr = vis.data_ptr()
        self.steps += 1
        dev = d_particles.device
        lr = (C.c_float * 6)(*[self.lrs[k] for k in GROUPS])
        stream = torch.cuda.current_stream(dev).cuda_stream
        args = (stream, self.n, self._array({k: t.data for k, t in self.params.items()}), self._array(self.exp_avg), self._array(self.exp_avg_sq),
                lr, self.betas[0], self.betas[1], self.eps, self.steps, int(self.selective), d_particles.data_ptr(), d_sph.data_ptr(), vis_ptr)
        if lambda_opacity == 0.0 and lambda_scale == 0.0:
            entry, extra = "gutb200_gaussian_adam_step", ()
        else:  # d mean(sigmoid(raw)) / d density = 1 / N, d mean(exp(raw)) / d scale = 1 / (3 N)
            entry, extra = "gutb200_gaussian_adam_step_reg", (float(lambda_opacity) / max(self.n, 1), float(lambda_scale) / (3 * max(self.n, 1)))
        with torch.cuda.device(dev):
            rc = getattr(native.load(), entry)(*args, *extra)
        if rc != 0:
            raise RuntimeError(f"{entry} failed ({rc})")


NHT_GROUPS = ("positions", "density", "rotation", "scale", "features")
NHT_WIDTHS = (3, 1, 4, 3, 48)


class FusedNHTAdam:
    """One-launch optimizer step for the NHT model and its feature decoder (gutb200_nht_adam_step).

    params: dict name -> raw leaf tensor for NHT_GROUPS (features [N,48] are used raw, model.py:225); decoder_params: the decoder's flat
    fp32 parameter vector (FeatureDecoder.network.params), updated in place as the group "decoder".  lrs: dict over NHT_GROUPS + "decoder"
    (mutable, as FusedGaussianAdam's).  The Gaussian groups take betas / eps / selective as FusedGaussianAdam does; the decoder has an Adam
    of its own, as in the reference (trainer.py:573-577): decoder_betas, decoder_eps, decoder_weight_decay (L2 on the gradient) and its own
    step count, never selective.  step(..., frozen=names) skips those groups entirely: no block is launched for them, their parameters,
    moments and step counts stay as they are (torch's Adam with grad None, the reference's colour refinement)."""

    GROUPS = NHT_GROUPS + ("decoder",)

    def __init__(self, params: dict, decoder_params: torch.Tensor, lrs: dict, betas=(0.9, 0.999), eps=1e-15, selective=False,
                 decoder_betas=(0.9, 0.999), decoder_eps=1e-8, decoder_weight_decay=0.0):
        # the dict itself is kept (not copied) when it holds exactly the five groups: densification replaces the tensors inside it
        self.params = params if set(params.keys()) == set(NHT_GROUPS) else {k: params[k] for k in NHT_GROUPS}
        self.decoder_params = decoder_params
        self._validate()
        self.lrs = {k: float(lrs[k]) for k in self.GROUPS}
        self.betas, self.eps, self.selective = (float(betas[0]), float(betas[1])), float(eps), bool(selective)
        self.decoder_betas, self.decoder_eps = (float(decoder_betas[0]), float(decoder_betas[1])), float(decoder_eps)
        self.decoder_weight_decay = float(decoder_weight_decay)
        self.exp_avg = {k: torch.zeros_like(t.data) for k, t in self.params.items()}
        self.exp_avg_sq = {k: torch.zeros_like(t.data) for k, t in self.params.items()}
        # the decoder's moments live apart from the per-Gaussian dicts, which the densifiers resize row by row
        self.decoder_exp_avg = torch.zeros_like(decoder_params.data)
        self.decoder_exp_avg_sq = torch.zeros_like(decoder_params.data)
        self.steps = {k: 0 for k in self.GROUPS}
        native.load()

    @property
    def n(self) -> int:
        return int(self.params["positions"].shape[0])

    def _validate(self):
        n = self.n
        for k, w in zip(NHT_GROUPS, NHT_WIDTHS):
            t = self.params[k]
            _check(t.data, k)
            if tuple(t.shape) != (n, w):
                raise RuntimeError(f"{k}: expected shape {(n, w)}, got {tuple(t.shape)}")
        _check(self.decoder_params.data, "decoder params")
        if self.decoder_params.dim() != 1:
            raise RuntimeError("decoder params: expected the flat parameter vector")

    def _tensors(self, which: str):
        if which == "param":
            return [self.params[k].data for k in NHT_GROUPS] + [self.decoder_params.data]
        if which == "m":
            return [self.exp_avg[k] for k in NHT_GROUPS] + [self.decoder_exp_avg]
        return [self.exp_avg_sq[k] for k in NHT_GROUPS] + [self.decoder_exp_avg_sq]

    @torch.no_grad()
    def step(self, d_particles: torch.Tensor, d_features: torch.Tensor, d_decoder: torch.Tensor, visibility: torch.Tensor | None = None,
             lambda_opacity: float = 0.0, lambda_scale: float = 0.0, frozen=()):
        frozen = set(frozen)
        unknown = frozen - set(self.GROUPS)
        if unknown:
            raise ValueError(f"frozen: unknown groups {sorted(unknown)} (groups: {', '.join(self.GROUPS)})")
        for t, what in ((d_particles, "d_particles"), (d_features, "d_features"), (d_decoder, "d_decoder")):
            _check(t, what)
        self._validate()  # the tensors may have been replaced (densification); moments must have followed
        for k in NHT_GROUPS:
            if self.exp_avg[k].shape != self.params[k].shape or self.exp_avg_sq[k].shape != self.params[k].shape:
                raise RuntimeError(f"{k}: optimizer state does not match the parameter shape {tuple(self.params[k].shape)}")
        n_dec = int(self.decoder_params.numel())
        if tuple(d_particles.shape) != (self.n, 12) or tuple(d_features.shape) != (self.n, 48) or tuple(d_decoder.shape) != (n_dec,):
            raise RuntimeError(f"gradient shapes must be [N,12], [N,48] and [{n_dec}]")
        vis_ptr = None
        if self.selective:
            if visibility is None:
                raise RuntimeError("selective mode needs the renderer's visibility")
            vis = visibility.reshape(-1)
            if vis.dtype != torch.float32:
                vis = vis.to(torch.float32)
            vis = vis.contiguous()
            _check(vis, "visibility")
            vis_ptr = vis.data_ptr()
        mask = 0
        for i, k in enumerate(self.GROUPS):
            if k in frozen:
                mask |= 1 << i
            else:
                self.steps[k] += 1
        arr = lambda ts: (C.c_void_p * 6)(*[t.data_ptr() for t in ts])  # noqa: E731
        lr = (C.c_float * 6)(*[self.lrs[k] for k in self.GROUPS])
        steps = (C.c_int64 * 6)(*[self.steps[k] for k in self.GROUPS])
        reg_density, reg_scale = float(lambda_opacity) / max(self.n, 1), float(lambda_scale) / (3 * max(self.n, 1))
        dev = d_particles.device
        stream = torch.cuda.current_stream(dev).cuda_stream
        with torch.cuda.device(dev):
            rc = native.load().gutb200_nht_adam_step(stream, self.n, n_dec, arr(self._tensors("param")), arr(self._tensors("m")),
                                                     arr(self._tensors("v")), lr, steps, self.betas[0], self.betas[1], self.eps,
                                                     int(self.selective), self.decoder_betas[0], self.decoder_betas[1], self.decoder_eps,
                                                     self.decoder_weight_decay, mask, d_particles.data_ptr(), d_features.data_ptr(),
                                                     d_decoder.data_ptr(), vis_ptr, reg_density, reg_scale)
        if rc != 0:
            raise RuntimeError(f"gutb200_nht_adam_step failed ({rc})")

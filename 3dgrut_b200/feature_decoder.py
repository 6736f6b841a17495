"""Drop-in for the reference's `threedgrut.model.feature_decoder.FeatureDecoder` (Neural Harmonic Textures): per-pixel features and view
direction -> RGB through tiny-cuda-nn's NetworkWithInputEncoding, here the fused tensor-core decoder of include/nht_b200.h.

Same constructor, `forward`, EMA methods, `regularization_loss` and `extra_repr`; the parameters are one fp32 vector `network.params` of
tcnn's length and layout, so the reference trainer's state dict of `feature_decoder.module` and its `torch.optim.Adam` over `parameters()`
work unchanged, and a tcnn checkpoint loads as it is.  There is no fallback: configurations the kernels do not build raise
NotImplementedError, and the decoder runs on CUDA tensors only.
"""
from __future__ import annotations

import ctypes as C
import math

import torch
import torch.nn as nn

import b200_native as nat

WIDTH = 128


def decoder_config(ray_feature_dim: int, hidden_dim: int, num_layers: int, dir_encoding: str, dir_encoding_degree: int,
                   sh_scale: float, output_activation: str) -> nat.NhtConfig:
    """The nhtb200_config of a FeatureDecoder; NotImplementedError for configurations that are not built."""
    if dir_encoding != "SphericalHarmonics":
        if dir_encoding == "Frequency":
            raise NotImplementedError("dir_encoding='Frequency' is not built: only 'SphericalHarmonics'")
        raise ValueError(f"Unknown dir_encoding: {dir_encoding}")
    if output_activation not in nat.NHT_ACTIVATIONS:
        raise NotImplementedError(f"output_activation={output_activation!r} is not built: one of {list(nat.NHT_ACTIVATIONS)}")
    cfg = nat.NhtConfig()
    cfg.n_features, cfg.sh_degree, cfg.n_hidden_layers = int(ray_feature_dim), int(dir_encoding_degree), int(num_layers)
    cfg.width, cfg.output_activation, cfg.sh_scale = int(hidden_dim), nat.NHT_ACTIVATIONS[output_activation], float(sh_scale)
    if nat.nht_lib().nhtb200_n_params(C.byref(cfg)) < 0:
        raise NotImplementedError(f"FeatureDecoder configuration is not built: {nat.nht_lib().nhtb200_last_error().decode()}")
    return cfg


def matrix_shapes(cfg: nat.NhtConfig) -> list[tuple[int, int]]:
    """[(out, in)] of the weight matrices in params order (tcnn's FullyFusedMLP)."""
    k0 = (cfg.n_features + cfg.sh_degree ** 2 + 15) // 16 * 16
    return [(WIDTH, k0)] + [(WIDTH, WIDTH)] * (cfg.n_hidden_layers - 1) + [(16, WIDTH)]


def initial_params(cfg: nat.NhtConfig, generator: torch.Generator | None = None) -> torch.Tensor:
    """tcnn's per-matrix distribution (FullyFusedMLP::initialize_params -> initialize_xavier_uniform): U(-s, s), s = sqrt(6 / (in + out))."""
    parts = []
    for out, inp in matrix_shapes(cfg):
        s = math.sqrt(6.0 / (out + inp))
        parts.append(torch.rand(out * inp, generator=generator, dtype=torch.float32) * (2 * s) - s)
    return torch.cat(parts)


class _Decode(torch.autograd.Function):
    @staticmethod
    def forward(ctx, features, dirs, params, cfg):
        n = features.shape[0]
        out = torch.empty((n, 3), device=features.device, dtype=torch.float32)
        stream = torch.cuda.current_stream(features.device).cuda_stream
        nat.nht_check(nat.nht_lib().nhtb200_forward(C.byref(cfg), stream, n, features.data_ptr(), dirs.data_ptr(), params.data_ptr(),
                                                    out.data_ptr()), "nhtb200_forward")
        ctx.cfg = cfg
        ctx.save_for_backward(features, dirs, params)
        return out

    @staticmethod
    def backward(ctx, d_out):
        features, dirs, params = ctx.saved_tensors
        d_features = torch.empty_like(features)
        d_params = torch.empty_like(params)
        ws = backward_workspace(ctx.cfg, features.shape[0], features.device)
        decode_backward(features, dirs, params, ctx.cfg, d_out.contiguous().float(), d_features, d_params, ws)
        return d_features, None, d_params, None


def backward_workspace(cfg: nat.NhtConfig, n: int, device) -> torch.Tensor:
    """The device workspace decode_backward needs for n rows (about 1.1 GB at 800 x 800 for the shipped decoder: allocate it once per
    resolution where the backward runs every step)."""
    return torch.empty(nat.nht_lib().nhtb200_backward_workspace_bytes(C.byref(cfg), int(n)), device=device, dtype=torch.uint8)


def decode_backward(features: torch.Tensor, dirs: torch.Tensor, params: torch.Tensor, cfg: nat.NhtConfig, d_out: torch.Tensor,
                    d_features: torch.Tensor, d_params: torch.Tensor, workspace: torch.Tensor) -> None:
    """nhtb200_backward into caller tensors: d_out [n,3] -> d_features [n,F] and d_params [n_params] (overwritten, summed over the rows);
    all contiguous fp32 CUDA tensors, e.g. d_params a view of a gradient exchange buffer.  workspace: backward_workspace(cfg, >= n)."""
    n = int(features.shape[0])
    for name, t, shape in (("features", features, None), ("dirs", dirs, (n, 3)), ("d_out", d_out, (n, 3)), ("d_features", d_features, tuple(features.shape)),
                           ("d_params", d_params, tuple(params.shape))):
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and (shape is None or tuple(t.shape) == shape)):
            raise RuntimeError(f"decode_backward: {name} must be a contiguous float32 CUDA tensor{'' if shape is None else f' {list(shape)}'}")
    lib = nat.nht_lib()
    if workspace.numel() < lib.nhtb200_backward_workspace_bytes(C.byref(cfg), n):
        raise RuntimeError("decode_backward: workspace is too small for this many rows")
    stream = torch.cuda.current_stream(features.device).cuda_stream
    nat.nht_check(lib.nhtb200_backward(C.byref(cfg), stream, n, features.data_ptr(), dirs.data_ptr(), params.data_ptr(), d_out.data_ptr(),
                                       d_features.data_ptr(), d_params.data_ptr(), workspace.data_ptr()), "nhtb200_backward")


def decode(features: torch.Tensor, dirs: torch.Tensor, params: torch.Tensor, cfg: nat.NhtConfig) -> torch.Tensor:
    """rgb [n,3] fp32 of features [n,F] and raw ray directions [n,3] (the encoding applies sh_scale), differentiable in features and params."""
    for name, t in (("features", features), ("ray_directions", dirs), ("params", params)):
        if not t.is_cuda:
            raise RuntimeError(f"FeatureDecoder: {name} must be a CUDA tensor (there is no CPU path)")
    return _Decode.apply(features.contiguous().float(), dirs.detach().contiguous().float(), params.contiguous(), cfg)


class _Network(nn.Module):
    """Holds the flat parameter vector under the name tcnn's torch module uses (`params`)."""

    def __init__(self, params: torch.Tensor):
        super().__init__()
        self.params = nn.Parameter(params)


class FeatureDecoder(nn.Module):
    """Transforms N-dimensional feature maps to RGB radiance (the reference's FeatureDecoder, same arguments and methods)."""

    def __init__(
        self,
        ray_feature_dim: int,
        hidden_dim: int = 128,
        num_layers: int = 4,
        dir_encoding: str = "SphericalHarmonics",
        dir_encoding_degree: int = 3,
        sh_scale: float = 1.0,
        output_activation: str = "Sigmoid",
        ema_decay: float = 0.0,
        ema_start_step: int = 0,
        unpremultiply_alpha: bool = False,
    ):
        super().__init__()
        self.ray_feature_dim = ray_feature_dim
        self.hidden_dim = hidden_dim
        self.num_layers = num_layers
        self.sh_scale = sh_scale
        self.output_activation = output_activation
        self.unpremultiply_alpha = unpremultiply_alpha
        self._ema_decay = ema_decay
        self._ema_start_step = ema_start_step
        self._ema_shadow: dict[str, torch.Tensor] = {}
        self._ema_backup: dict[str, torch.Tensor] = {}

        self.config = decoder_config(ray_feature_dim, hidden_dim, num_layers, dir_encoding, dir_encoding_degree, sh_scale, output_activation)
        self.network = _Network(initial_params(self.config))

        if self._ema_decay > 0:
            for name, param in self.named_parameters():
                if param.requires_grad:
                    self._ema_shadow[name] = param.data.clone()

    def ema_update(self, global_step: int) -> None:
        """Update EMA shadow when global_step >= ema_start_step. No-op if ema_decay <= 0."""
        if self._ema_decay <= 0 or global_step < self._ema_start_step:
            return
        with torch.no_grad():
            for name, param in self.named_parameters():
                if param.requires_grad and name in self._ema_shadow:
                    if self._ema_shadow[name].device != param.device:
                        self._ema_shadow[name] = self._ema_shadow[name].to(param.device)
                    self._ema_shadow[name].lerp_(param.data, 1.0 - self._ema_decay)

    def apply_ema_shadow(self) -> None:
        """Use EMA weights for inference (e.g. validation). No-op if no EMA."""
        if not self._ema_shadow:
            return
        with torch.no_grad():
            for name, param in self.named_parameters():
                if param.requires_grad and name in self._ema_shadow:
                    self._ema_backup[name] = param.data.clone()
                    param.data.copy_(self._ema_shadow[name])

    def restore_ema(self) -> None:
        """Restore training weights after inference. No-op if no EMA."""
        with torch.no_grad():
            for name, param in self.named_parameters():
                if param.requires_grad and name in self._ema_backup:
                    param.data.copy_(self._ema_backup[name])
        self._ema_backup.clear()

    def ema_state_dict(self) -> dict:
        """State dict of EMA shadow for checkpoint. Empty if no EMA."""
        return {k: v.clone() for k, v in self._ema_shadow.items()}

    def load_ema_state_dict(self, state_dict: dict) -> None:
        """Load EMA shadow from checkpoint."""
        self._ema_shadow = {k: v.clone() for k, v in state_dict.items()}

    def forward(self, features: torch.Tensor, ray_directions: torch.Tensor, alpha: torch.Tensor | None = None) -> torch.Tensor:
        """RGB [H*W,3] or [B,H,W,3] of features [H*W,N] or [B,H,W,N] and ray directions of the same leading shape."""
        features_shape, ray_dirs_shape = features.shape, ray_directions.shape
        if len(features_shape) == 4:  # [B, H, W, N]
            B, H, W, N = features_shape
            assert ray_dirs_shape == (B, H, W, 3), f"Ray directions shape mismatch: expected {(B, H, W, 3)}, got {ray_dirs_shape}"
            assert N == self.ray_feature_dim, f"Expected {self.ray_feature_dim} features, got {N}"
            alpha_flat = alpha.reshape(B * H * W, 1) if alpha is not None else None
            rgb = self._process(features.reshape(B * H * W, N), ray_directions.reshape(B * H * W, 3), alpha_flat)
            return rgb.reshape(B, H, W, 3)
        if len(features_shape) == 2:  # [H*W, N]
            HW, N = features_shape
            assert ray_dirs_shape == (HW, 3), f"Ray directions shape mismatch: expected {(HW, 3)}, got {ray_dirs_shape}"
            assert N == self.ray_feature_dim, f"Expected {self.ray_feature_dim} features, got {N}"
            return self._process(features, ray_directions, alpha.reshape(HW, 1) if alpha is not None else None)
        raise ValueError(f"Expected input shape [B, H, W, N] or [H*W, N], got {features_shape}")

    def _process(self, features, ray_directions, alpha=None):
        if self.unpremultiply_alpha and alpha is not None:
            alpha_safe = alpha.clamp(min=1e-8)
            features = features / alpha_safe
        rgb = decode(features, ray_directions, self.network.params, self.config)
        if self.unpremultiply_alpha and alpha is not None:
            rgb = rgb * alpha_safe
        return rgb

    def regularization_loss(self) -> torch.Tensor:
        """Compute L2 regularization loss on decoder weights."""
        loss = torch.tensor(0.0, device=self.network.params.device)
        loss = loss + torch.sum(self.network.params**2)
        return loss

    def extra_repr(self) -> str:
        return (
            f"ray_feature_dim={self.ray_feature_dim}, "
            f"hidden_dim={self.hidden_dim}, "
            f"num_layers={self.num_layers}, "
            f"sh_scale={self.sh_scale}, "
            f"output_activation={self.output_activation}, "
            f"unpremultiply_alpha={self.unpremultiply_alpha}"
        )

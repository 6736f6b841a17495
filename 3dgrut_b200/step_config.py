"""A training step from a run configuration: `render.method` x `model.feature_type` selects one of the four steps (3DGUT / 3DGRT, SH /
NHT), and the optimizer, loss, background, post-processing, schedule, NHT decoder and densification strategy are read from the config as
the reference trainer reads them (trainer.py:116-410, model.py:782-852, strategy/gs.py, strategy/mcmc.py, configs/strategy/*.yaml).

`check_config` refuses, with NotImplementedError naming the key, every setting the steps do not build, before anything is read from disk
or allocated."""
from __future__ import annotations

import torch

import densify
from b200_native import cfg_get

METHODS = ("3dgut", "3dgrt")
STRATEGIES = {"GSStrategy": "gs", "MCMCStrategy": "mcmc"}
OPTIMIZERS = ("adam", "selective_adam")
# model.optimize_* of configs/base_gs.yaml: the steps train every group
OPTIMIZE_KEYS = ("density", "features_albedo", "features_specular", "features", "position", "rotation", "scale")


def _method(conf) -> str:
    method = str(cfg_get(conf, "render.method", "3dgut")).lower()
    if method not in METHODS:
        raise NotImplementedError(f"render.method={method!r}: the training steps built from a config are {', '.join(METHODS)}")
    return method


def _feature_type(conf) -> str:
    ft = str(cfg_get(conf, "model.feature_type", "sh")).lower()
    if ft not in ("sh", "nht"):
        raise NotImplementedError(f"model.feature_type={ft!r}: the training steps train 'sh' or 'nht'")
    return ft


def check_config(conf) -> None:
    """NotImplementedError naming the first setting of `conf` that the training loop does not build."""
    import losses
    import scene_data

    scene_data.check_dataset_config(conf)
    _method(conf)
    _feature_type(conf)
    losses.post_processing_code(cfg_get(conf, "post_processing.method", None))
    if bool(cfg_get(conf, "loss.use_l2", False)):
        raise NotImplementedError("loss.use_l2=true: the image loss is L1 + SSIM")
    opt = str(cfg_get(conf, "optimizer.type", "adam"))
    if opt not in OPTIMIZERS:
        raise NotImplementedError(f"optimizer.type={opt!r}: the steps build {', '.join(OPTIMIZERS)}")
    for name in OPTIMIZE_KEYS:
        if not bool(cfg_get(conf, f"model.optimize_{name}", True)):
            raise NotImplementedError(f"model.optimize_{name}=false: the steps train every parameter group")
    for key in ("export_usd.enabled", "with_gui", "with_viser_gui"):
        if bool(cfg_get(conf, key, False)):
            raise NotImplementedError(f"{key}=true is not built")
    strategy_config(conf)


def strategy_config(conf):
    """densify.DensifyConfig (GSStrategy, from the keys of configs/strategy/gs.yaml), densify.MCMCConfig (MCMCStrategy) or None (no
    strategy section)."""
    s = cfg_get(conf, "strategy", None)
    if s is None:
        return None
    method = cfg_get(s, "method", None)
    if method not in STRATEGIES:
        raise NotImplementedError(f"strategy.method={method!r}: the strategies built are {', '.join(STRATEGIES)}")
    g = lambda key, default: cfg_get(s, key, default)  # noqa: E731
    if method == "MCMCStrategy":
        d = densify.MCMCConfig()
        return densify.MCMCConfig(
            binom_n_max=int(g("binom_n_max", d.binom_n_max)), opacity_threshold=float(g("opacity_threshold", d.opacity_threshold)),
            relocate_start=int(g("relocate.start_iteration", d.relocate_start)), relocate_end=int(g("relocate.end_iteration", d.relocate_end)),
            relocate_frequency=int(g("relocate.frequency", d.relocate_frequency)), add_start=int(g("add.start_iteration", d.add_start)),
            add_end=int(g("add.end_iteration", d.add_end)), add_frequency=int(g("add.frequency", d.add_frequency)),
            max_n_gaussians=int(g("add.max_n_gaussians", d.max_n_gaussians)), perturb_start=int(g("perturb.start_iteration", d.perturb_start)),
            perturb_end=int(g("perturb.end_iteration", d.perturb_end)), perturb_frequency=int(g("perturb.frequency", d.perturb_frequency)),
            noise_lr=float(g("perturb.noise_lr", d.noise_lr)))
    params = g("densify.params", "positions")
    if params != "positions":
        raise NotImplementedError(f"strategy.densify.params={params!r}: the densifier accumulates the positions' gradient")
    for key in ("density_decay", "prune_weight", "prune_scale"):
        if int(g(f"{key}.start_iteration", -1)) >= 0:
            raise NotImplementedError(f"strategy.{key}.start_iteration={g(f'{key}.start_iteration', -1)}: {key} is not built")
    d = densify.DensifyConfig()
    cfg = densify.DensifyConfig(
        clone_grad_threshold=float(g("densify.clone_grad_threshold", d.clone_grad_threshold)),
        split_grad_threshold=float(g("densify.split_grad_threshold", d.split_grad_threshold)),
        relative_size_threshold=float(g("densify.relative_size_threshold", d.relative_size_threshold)),
        split_n_gaussians=int(g("densify.split.n_gaussians", d.split_n_gaussians)),
        prune_density_threshold=float(g("prune.density_threshold", d.prune_density_threshold)),
        new_max_density=float(g("reset_density.new_max_density", d.new_max_density)),
        density_decay_gamma=float(g("density_decay.gamma", d.density_decay_gamma)),
        densify_start=int(g("densify.start_iteration", d.densify_start)), densify_end=int(g("densify.end_iteration", d.densify_end)),
        densify_frequency=int(g("densify.frequency", d.densify_frequency)), prune_start=int(g("prune.start_iteration", d.prune_start)),
        prune_end=int(g("prune.end_iteration", d.prune_end)), prune_frequency=int(g("prune.frequency", d.prune_frequency)),
        reset_start=int(g("reset_density.start_iteration", d.reset_start)), reset_frequency=int(g("reset_density.frequency", d.reset_frequency)))
    reset_end = int(g("reset_density.end_iteration", cfg.densify_end))
    if reset_end != cfg.densify_end:
        raise NotImplementedError(f"strategy.reset_density.end_iteration={reset_end}: the density reset ends with densification "
                                  f"(strategy.densify.end_iteration={cfg.densify_end})")
    return cfg


def make_decoder(conf, device, arch: dict | None = None):
    """The NHT FeatureDecoder of model.nht_decoder.* (or of a checkpoint's `arch`), on `device`.  A new decoder's weights come from torch's
    generator seeded seed_initialization, so every rank starts from the same ones."""
    import feature_decoder as fd
    from b200_native import NHT_FEATURE_DIM

    g = lambda key, default: cfg_get(conf, f"model.nht_decoder.{key}", default)  # noqa: E731
    a = arch or {"ray_feature_dim": NHT_FEATURE_DIM // 2, "hidden_dim": g("hidden_dim", 128), "num_layers": g("num_layers", 3),
                 "sh_scale": g("sh_scale", 3.0), "output_activation": g("output_activation", "Sigmoid"),
                 "unpremultiply_alpha": g("unpremultiply_alpha", False)}
    if arch is None:
        torch.manual_seed(int(cfg_get(conf, "seed_initialization", 42)))
    return fd.FeatureDecoder(int(a["ray_feature_dim"]), hidden_dim=int(a["hidden_dim"]), num_layers=int(a["num_layers"]),
                             dir_encoding=str(g("dir_encoding", "SphericalHarmonics")), dir_encoding_degree=int(g("dir_encoding_degree", 3)),
                             sh_scale=float(a["sh_scale"]), output_activation=str(a["output_activation"]),
                             ema_decay=float(g("ema_decay", 0.0)) if arch is None else 0.0,
                             ema_start_step=int(g("ema_start_step", 0)) if arch is None else 0,
                             unpremultiply_alpha=bool(a.get("unpremultiply_alpha", False))).to(device)


def build_step(conf, params: dict, scene_extent: float, group=None, *, lrs: dict | None = None, sph_degree: int | None = None,
               decoder=None, background=None, train: bool = True):
    """The training step `conf` describes, holding `params` (initialization.initialize's dict).

    train=True (a run): every refusal of check_config, the schedule of TrainingSchedule.from_config(conf, scene_extent), the strategy of
    strategy.*, the optimizer of optimizer.type / eps, the loss of loss.use_* / lambda_*, model.background.color and
    post_processing.method, and a new decoder from model.nht_decoder.* for NHT.
    train=False (evaluation of a checkpoint): only the renderer and what rendering reads; `lrs`, `sph_degree` (SH), `decoder` (NHT) and
    `background` (default model.background.color) come from the caller, and nothing is refused beyond what the step itself refuses."""
    import schedule as schedule_mod

    method, ft = _method(conf), _feature_type(conf)
    kw = dict(background=background if background is not None else cfg_get(conf, "model.background.color", "black"),
              post_processing=cfg_get(conf, "post_processing.method", None), group=group, scene_extent=scene_extent)
    if train:
        check_config(conf)
        loss = lambda key, default: float(cfg_get(conf, f"loss.lambda_{key}", default)) if bool(cfg_get(conf, f"loss.use_{key}", False)) else 0.0  # noqa: E731
        kw.update(selective=str(cfg_get(conf, "optimizer.type", "adam")) == "selective_adam", eps=float(cfg_get(conf, "optimizer.eps", 1e-15)),
                  lambda_l1=loss("l1", 0.8), lambda_ssim=loss("ssim", 0.2), lambda_opacity=loss("opacity", 0.0), lambda_scale=loss("scale", 0.0),
                  densify_conf=strategy_config(conf),
                  schedule=schedule_mod.TrainingSchedule.from_config(conf, scene_extent=scene_extent, feature_type=ft))
    else:
        kw.update(sph_degree=sph_degree)
    device = params["positions"].device
    if ft == "nht":
        import train_step_nht as tsn

        kw.pop("sph_degree", None)
        cls = tsn.GaussianTrainStepGRTNHT if method == "3dgrt" else tsn.GaussianTrainStepNHT
        return cls(params, lrs, decoder if decoder is not None else make_decoder(conf, device), conf, **kw)
    if method == "3dgrt":
        from train_step_grt import GaussianTrainStepGRT as cls
    else:
        from train_step import GaussianTrainStep as cls
    return cls(params, lrs, conf=conf, **kw)

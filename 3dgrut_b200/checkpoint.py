"""Checkpoints of the training steps, in the layout of the reference trainer's `ckpt_*.pt` (Trainer.save_checkpoint,
threedgrut/trainer.py:1036-1083; resumed by Trainer.setup_training, :275-310; model/model.py:132-166 get_model_parameters, :613-691
init_from_checkpoint, :782-826 setup_optimizer; strategy/gs.py:42-57).

A file written by `save` opens in the reference's render.py, GUI, playground and PLY / USD exporters and resumes the reference Trainer; a
file the reference trainer wrote resumes a step here through `load`.  What the reference has no slot for (generator states, the schedule
state, the Adam step counts, the 3DGRT BVH cadence, the step's settings) goes under the key EXTRAS, which the reference's loaders never
read.  A checkpoint without it resumes too: generators are seeded as the constructors seed them, the schedule is rebuilt at
`global_step` from the checkpoint's `config`, and the Adam step counts come from the optimizer section.

`reference_layout` / `from_reference_layout` convert between a step's state (TrainStep.state_dict) and that layout.  They are pure
functions of dicts of tensors: no GPU, no file.  `save` / `load` add the file and the ranks."""
from __future__ import annotations

import os

import torch
import torch.distributed as dist

import schedule as schedule_mod
from b200_native import NHT_FEATURE_DIM, cfg_get

EXTRAS = "b200"
SH_GROUPS = schedule_mod.SH_GROUPS
NHT_GROUPS = schedule_mod.NHT_GROUPS
GEOMETRY = ("positions", "density", "rotation", "scale")  # frozen together by the NHT steps' colour refinement
# optimizer.params of configs/base_gs.yaml, in order: the reference's param groups follow it (model.py:783-801)
REFERENCE_ORDER = ("positions", "density", "features_albedo", "features_specular", "features", "rotation", "scale")
PARTICLE_FEATURE_DIM = 48                                     # SH: 3 + 45 coefficients; NHT: model.nht_features.dim
RAY_FEATURE_DIM = {"sh": 3, "nht": NHT_FEATURE_DIM // 2}      # model.py:200-219


def groups_of(feature_type: str) -> tuple:
    if feature_type not in ("sh", "nht"):
        raise ValueError(f"feature_type: unknown feature type {feature_type!r} (expected 'sh' or 'nht')")
    return NHT_GROUPS if feature_type == "nht" else SH_GROUPS


def check_step_counts(feature_type: str, steps: dict) -> None:
    """Refuse Adam step counts that the step cannot continue from: every SH group, and the four NHT geometry groups (which colour
    refinement freezes together), must share one count.  ValueError names the group."""
    tied = GEOMETRY if feature_type == "nht" else SH_GROUPS
    first = tied[0]
    for name in tied:
        if name not in steps:
            raise ValueError(f"optimizer: no step count for the group {name!r}")
        if int(steps[name]) != int(steps[first]):
            raise ValueError(f"optimizer: the group {name!r} has taken {int(steps[name])} Adam steps and {first!r} {int(steps[first])}; "
                             f"the step trains {', '.join(tied)} with one count")


# ---- step state -> reference layout -------------------------------------------------------------------------------------------------

def _stand_in() -> torch.nn.Parameter:
    p = torch.nn.Parameter(torch.zeros(1))
    p.grad = torch.zeros(1)
    return p


def _fill(opt: torch.optim.Optimizer, p, count: int, exp_avg, exp_avg_sq) -> None:
    """Put a group's real moments and step count into the state torch created for its stand-in (none before the first step)."""
    if count == 0:
        del opt.state[p]
        return
    st = opt.state[p]
    st["step"].fill_(float(count))
    st["exp_avg"], st["exp_avg_sq"] = exp_avg, exp_avg_sq


def _optimizer_section(state: dict, conf) -> dict:
    """The model's torch.optim.Adam state dict: one group per parameter, named and ordered as conf.optimizer.params (base_gs.yaml's order
    without a config), at the state's rates.  A real Adam over CPU stand-ins is stepped once so that torch lays out its own state, then
    handed the real moments and counts: the layout is the installed torch's."""
    groups = groups_of(state["feature_type"])
    settings = state.get("settings") or {}
    listed = cfg_get(conf, "optimizer.params", None)
    order = [str(k) for k in listed.keys()] if listed is not None else list(REFERENCE_ORDER)
    names = [k for k in order if k in groups] + [k for k in groups if k not in order]
    stand = {k: _stand_in() for k in names}
    selective = bool(settings.get("selective", False))  # optimizer.type selective_adam: the reference's SelectiveAdam is not fused
    opt = torch.optim.Adam([{"params": [stand[k]], "name": k, "lr": float(state["lrs"][k])} for k in names],
                           lr=float(cfg_get(conf, "optimizer.lr", 0.0)), eps=float(settings.get("eps", 1e-15)), fused=not selective)
    opt.step()
    for k in names:
        _fill(opt, stand[k], int(state["adam_steps"][k]), state["exp_avg"][k], state["exp_avg_sq"][k])
    return opt.state_dict()


def _decoder_section(state: dict) -> dict:
    """feature_decoder: module, optimizer (torch Adam over the decoder's one parameter, trainer.py:573-577), scheduler (a real
    CosineAnnealingLR / ExponentialLR stepped to the schedule's epoch, trainer.py:579-596), arch and, when the decoder keeps one, ema."""
    dec, settings = state["decoder"], state.get("settings") or {}
    sch = dec["scheduler"]
    p = _stand_in()
    opt = torch.optim.Adam([p], lr=float(sch["base_lr"]), weight_decay=float(settings.get("decoder_weight_decay", 0.0)))
    if sch["type"] == "cosine":
        torch_sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_max=int(sch["max_steps"]), eta_min=float(sch["eta_min"]))
    else:
        torch_sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma=float(sch["gamma"]))
    opt.step()
    epoch = int(state["schedule"]["decoder_epoch"]) if state.get("schedule") is not None else int(state["frame"])
    for _ in range(epoch):
        torch_sched.step()
    # torch's recursion and the schedule's restatement of it may differ in the last bit: the rate the step trains at is the one written
    lr = float(state["lrs"]["decoder"])
    opt.param_groups[0]["lr"] = lr
    torch_sched._last_lr = [lr]
    _fill(opt, p, int(state["adam_steps"]["decoder"]), dec["exp_avg"], dec["exp_avg_sq"])
    out = {"module": {"network.params": dec["params"]}, "optimizer": opt.state_dict(), "scheduler": torch_sched.state_dict(),
           "arch": dict(dec["arch"])}
    if dec["ema"]:
        out["ema"] = dict(dec["ema"])
    return out


def reference_layout(state: dict, conf=None, epoch: int = 0) -> dict:
    """The dict Trainer.save_checkpoint writes, of a step's state (TrainStep.state_dict()).  conf: stored as `config` as given (the
    reference's loaders need its OmegaConf object there) and read for the optimizer groups' order.  The tensors are the state's own
    (parameters wrapped in nn.Parameter without a copy)."""
    ft = state["feature_type"]
    groups = groups_of(ft)
    out = {k: torch.nn.Parameter(state["params"][k].detach()) for k in groups}
    prog = state.get("progression")
    if ft == "nht":  # the reference renders every ray feature from the first step (model.py:245-250)
        n_active = max_n = RAY_FEATURE_DIM["nht"]
    else:
        n_active, max_n = int(state["sph_degree"]), int(prog[0]) if prog is not None else int(state["sph_degree"])
    out.update(background={}, n_active_features=n_active, max_n_features=max_n, progressive_training=prog is not None,
               scene_extent=float(state["scene_extent"]), optimizer=_optimizer_section(state, conf), config=conf, feature_type=ft,
               particle_feature_dim=PARTICLE_FEATURE_DIM, ray_feature_dim=RAY_FEATURE_DIM[ft])
    if prog is not None:
        out["feature_dim_increase_interval"], out["feature_dim_increase_step"] = int(prog[1]), int(prog[2])
    out.update(global_step=int(state["frame"]), epoch=int(epoch))
    dens = state.get("densifier")
    if dens is not None and "grad_norm_accum" in dens:  # the GS strategy (gs.py:42-47); MCMC writes nothing
        out["densify_grad_norm_accum"], out["densify_grad_norm_denom"] = (dens["grad_norm_accum"],), (dens["grad_norm_denom"],)
    if ft == "nht":
        out["feature_decoder"] = _decoder_section(state)
    settings = state.get("settings") or {}
    extras = {"settings": dict(settings), "sph_degree": state["sph_degree"], "adam_steps": dict(state["adam_steps"]),
              "densifier": None if dens is None else {"method": settings.get("strategy", "gs" if "grad_norm_accum" in dens else "mcmc"),
                                                      "generator": dens.get("generator")},
              "background_generators": [state.get("background_generator")], "schedule": state.get("schedule")}
    if "num_update_bvh" in state:
        extras["num_update_bvh"] = int(state["num_update_bvh"])
    out[EXTRAS] = extras
    return out


# ---- reference layout -> step state -------------------------------------------------------------------------------------------------

def _moments(section: dict, name: str | None, param: torch.Tensor):
    """(exp_avg, exp_avg_sq, step count, rate) of the group `name` of a torch Adam state dict (None: its first group); zeros and 0 for a
    group never stepped."""
    for g in section["param_groups"]:
        if g.get("name", None) == name or name is None:
            st = section["state"].get(g["params"][0])
            if not st:
                return torch.zeros_like(param), torch.zeros_like(param), 0, float(g["lr"])
            return st["exp_avg"], st["exp_avg_sq"], int(round(float(st["step"]))), float(g["lr"])
    raise ValueError(f"optimizer: no param group named {name!r}")


def _decoder_state(fdec: dict) -> tuple[dict, float, int]:
    params = fdec["module"]["network.params"].detach()
    m, v, count, lr = _moments(fdec["optimizer"], None, params)
    s = fdec["scheduler"]
    if "T_max" in s:
        sch = {"type": "cosine", "base_lr": float(s["base_lrs"][0]), "max_steps": int(s["T_max"]), "eta_min": float(s["eta_min"])}
    else:
        sch = {"type": "exponential", "base_lr": float(s["base_lrs"][0]), "gamma": float(s["gamma"])}
    return {"params": params, "exp_avg": m, "exp_avg_sq": v, "ema": dict(fdec.get("ema") or {}), "arch": dict(fdec["arch"]),
            "scheduler": sch}, lr, count


def from_reference_layout(ckpt: dict, feature_type: str | None = None, rank: int = 0, world_size: int = 1) -> dict:
    """A step's state (what TrainStep.load_state_dict takes) of a checkpoint in the reference layout, with or without EXTRAS.
    feature_type: the step's ("sh" / "nht"); a checkpoint of the other raises ValueError naming feature_type.  rank / world_size: this
    process's; the random background's generator state is this rank's when the checkpoint was written by as many ranks, else None (the
    step re-seeds it).  The tensors are the checkpoint's own (no copy).

    Refused: an NHT `features` width other than 48 (ValueError on particle_feature_dim, as init_from_checkpoint does), Adam step counts
    that differ across groups trained together (ValueError naming the group), a post_processing section (NotImplementedError on
    post_processing.method: PPISP is not built)."""
    ft = str(ckpt.get("feature_type", "sh")).lower()
    groups = groups_of(ft)
    if feature_type is not None and ft != feature_type:
        raise ValueError(f"feature_type: the checkpoint holds {ft!r} features, the step trains {feature_type!r}")
    if "post_processing" in ckpt:
        raise NotImplementedError("post_processing.method: the checkpoint carries post-processing state (PPISP), which is not built")
    if ft == "nht" and int(ckpt["features"].shape[1]) != PARTICLE_FEATURE_DIM:
        raise ValueError(f"particle_feature_dim: the checkpoint's NHT features are {int(ckpt['features'].shape[1])} wide, the steps train "
                         f"{PARTICLE_FEATURE_DIM}")
    extras = ckpt.get(EXTRAS)
    params = {k: ckpt[k].detach() for k in groups}
    state = {"feature_type": ft, "settings": dict(extras["settings"]) if extras else {}, "frame": int(ckpt["global_step"]),
             "scene_extent": float(ckpt["scene_extent"])}
    lrs, exp_avg, exp_avg_sq, steps = {}, {}, {}, {}
    for k in groups:
        exp_avg[k], exp_avg_sq[k], steps[k], lrs[k] = _moments(ckpt["optimizer"], k, params[k])
    if ft == "nht":
        decoder, lrs["decoder"], steps["decoder"] = _decoder_state(ckpt["feature_decoder"])
    if extras:
        steps = dict(extras["adam_steps"])
    check_step_counts(ft, steps)
    if extras:
        sph = extras["sph_degree"]
    else:
        sph = int(ckpt["n_active_features"]) if ft == "sh" else None  # NHT stores its ray feature count there
    prog = None
    if ft == "sh" and ckpt.get("progressive_training"):
        prog = [int(ckpt["max_n_features"]), int(ckpt["feature_dim_increase_interval"]), int(ckpt["feature_dim_increase_step"])]
    state.update(sph_degree=sph, lrs=lrs, progression=prog, params=params, exp_avg=exp_avg, exp_avg_sq=exp_avg_sq, adam_steps=steps)
    gs = "densify_grad_norm_accum" in ckpt
    if extras:
        d = extras["densifier"]
        if d is None:
            state["densifier"] = None
        elif d["method"] == "gs":
            state["densifier"] = {"grad_norm_accum": ckpt["densify_grad_norm_accum"][0], "grad_norm_denom": ckpt["densify_grad_norm_denom"][0],
                                  "generator": d["generator"]}
        else:
            state["densifier"] = {"generator": d["generator"]}
    else:
        state["densifier"] = ({"grad_norm_accum": ckpt["densify_grad_norm_accum"][0], "grad_norm_denom": ckpt["densify_grad_norm_denom"][0],
                               "generator": None} if gs else None)
    gens = extras["background_generators"] if extras else None
    state["background_generator"] = gens[rank] if gens is not None and len(gens) == world_size else None
    if extras:
        state["schedule"] = extras["schedule"]
    elif ckpt.get("config") is not None:  # a reference run: its schedule, replayed to global_step
        state["schedule"] = schedule_mod.TrainingSchedule.from_config(ckpt["config"], scene_extent=state["scene_extent"], feature_type=ft)\
            .advance_to(state["frame"]).state_dict()
    else:
        state["schedule"] = None
    if ft == "nht":
        state["decoder"] = decoder
    if extras and "num_update_bvh" in extras:
        state["num_update_bvh"] = int(extras["num_update_bvh"])
    return state


# ---- files and ranks ----------------------------------------------------------------------------------------------------------------

def _rank_world(step) -> tuple[int, int]:
    if step.world > 1:
        return dist.get_rank(step.group), step.world
    return 0, 1


def save(step, path: str, conf=None, epoch: int = 0) -> None:
    """Write `step`'s checkpoint to `path` (torch.save of reference_layout plus EXTRAS) from rank 0; every rank must call it.  The random
    background's generator differs per rank (seeded background_seed + rank): its states are gathered into EXTRAS as a list indexed by
    rank.  The file is written next to `path` and renamed over it, so an interrupted save leaves the previous checkpoint intact.  When
    `save` returns on any rank, the file is complete."""
    state = step.state_dict()
    rank, world = _rank_world(step)
    gens = [state.get("background_generator")]
    if world > 1:
        gens = [None] * world
        own = state.get("background_generator")
        dist.all_gather_object(gens, None if own is None else own.cpu(), group=step.group)
    if rank == 0:
        ckpt = reference_layout(state, conf=conf, epoch=epoch)
        ckpt[EXTRAS]["background_generators"] = gens
        tmp = f"{path}.tmp"
        torch.save(ckpt, tmp)
        os.replace(tmp, path)
    if world > 1:
        dist.barrier(group=step.group)


def load(path: str, step, weights_only: bool = False) -> dict:
    """Resume `step` from the checkpoint at `path` (written by `save` or by the reference trainer), read straight onto the step's device
    (map_location): the loaded tensors become the step's own, so the state is on the device once.  Every rank loads the same file, so the
    replicas stay bit-identical.  A random background resumes each rank's own generator when the file was written by as many ranks;
    otherwise the generators are re-seeded (background_seed + rank), and the backgrounds drawn from then on differ from those of an
    uninterrupted run.  weights_only: torch.load's; the reference's own loader reads with False, as a `config` that is an OmegaConf object
    needs.  Returns the checkpoint dict."""
    ckpt = torch.load(path, map_location=step.device, weights_only=weights_only)
    rank, world = _rank_world(step)
    step.load_state_dict(from_reference_layout(ckpt, feature_type=step.FEATURE_TYPE, rank=rank, world_size=world), assign=True)
    return ckpt

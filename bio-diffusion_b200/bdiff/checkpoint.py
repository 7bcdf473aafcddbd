"""Saving, resuming and converting GCDM training runs.

A library run keeps its state in two places: the denoiser's parameters (`GCPNetDynamicsB200`, reference names) and the
device buffers of `GCDMTrainTail` (AdamW moments, amsgrad maxima, EMA weights, step count, clip history).
`training_state` / `load_training_state` save and restore both, plus the random generators that `GCDMTrainLoss` draws
`t` and the noise from, so that a resumed run continues bit for bit.  Build the objects in this order before loading:

    net = GCPNetDynamicsB200(...).cuda(); net.flatten_parameters(); opt = GCDMTrainTail(net.parameters(), ...)
    load_training_state(torch.load(path), net, opt)

`from_reference_checkpoint` / `to_reference_checkpoint` move a run between the library and a Lightning checkpoint of the
reference's `QM9MoleculeGenerationDDPM` / `GEOMMoleculeGenerationDDPM` (and its `-EMA.ckpt` companion written by
`EMAModelCheckpoint`).  All of these are plain functions over dicts of tensors: only the final copies touch the device.
"""
from __future__ import annotations

import warnings
from collections import OrderedDict
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import torch

from .config import DenoiserConfig, parameter_shapes
from .optim import STATE_DICT_VERSION, STATE_WORDS, GCDMTrainTail
from .schedule import gamma_table

TRAINING_STATE_VERSION = 1
DYNAMICS_PREFIX = "ddpm.dynamics_network."
GAMMA_KEY = "ddpm.gamma.gamma"


def _names_in_opt_order(net, opt: GCDMTrainTail) -> List[str]:
    by_id = {id(p): n for n, p in net.named_parameters()}
    names = [by_id.get(id(p)) for p in opt.params]
    if None in names:
        raise ValueError("the GCDMTrainTail holds parameters that are not the denoiser's")
    if len(names) != len(by_id):
        raise ValueError(f"the GCDMTrainTail holds {len(names)} of the denoiser's {len(by_id)} parameters")
    return names


def _check_weights(weights: Dict[str, torch.Tensor], cfg: DenoiserConfig, what: str) -> None:
    """ValueError naming the first difference between `weights` and the denoiser's reference names and shapes."""
    shapes = parameter_shapes(cfg)
    missing = [k for k in shapes if k not in weights]
    unexpected = [k for k in weights if k not in shapes]
    if missing or unexpected:
        raise ValueError(f"{what}: missing {missing[:3]}{'...' if len(missing) > 3 else ''}, "
                         f"unexpected {unexpected[:3]}{'...' if len(unexpected) > 3 else ''}")
    for k, s in shapes.items():
        if tuple(weights[k].shape) != tuple(s):
            raise ValueError(f"{what}: {k} has shape {tuple(weights[k].shape)}, the denoiser's is {tuple(s)}")


# ------------------------------------------------------------------------------------------------ library format
def training_state(net, opt: GCDMTrainTail, extra: Any = None, rng: bool = True) -> dict:
    """The state of a library training run, ready for `torch.save`: the denoiser's `state_dict()` (reference names),
    `opt.state_dict()`, the parameter names in `opt`'s order (a reordering is caught on load), and with `rng` the CPU and
    current-CUDA generator states.  `extra` is stored as given (epoch, data-loader position, ...).  Synchronises."""
    state = {"version": TRAINING_STATE_VERSION,
             "model": OrderedDict((k, v.detach().clone()) for k, v in net.state_dict().items()),
             "param_names": _names_in_opt_order(net, opt), "optimizer": opt.state_dict(), "extra": extra}
    if rng:
        state["rng"] = {"cpu": torch.get_rng_state(), "cuda": torch.cuda.get_rng_state(opt.device)}
    return state


def load_training_state(state: dict, net, opt: GCDMTrainTail) -> Any:
    """Restore `training_state(...)` into `net` and `opt` in place (the parameters stay views of the flat buffer that
    `flatten_parameters()` made, and `opt`'s buffers stay the ones its device table points at).  Everything is validated
    first: a mismatch raises ValueError and loads nothing.  Returns the saved `extra`."""
    if state.get("version") != TRAINING_STATE_VERSION:
        raise ValueError(f"training state version {state.get('version')!r}, expected {TRAINING_STATE_VERSION}")
    names = _names_in_opt_order(net, opt)
    if list(state["param_names"]) != names:
        raise ValueError("the saved parameter order differs from this GCDMTrainTail's (build the net, call "
                         "flatten_parameters(), then GCDMTrainTail(net.parameters()))")
    _check_weights(state["model"], net.cfg, "saved model")
    opt._check_state_dict(state["optimizer"])
    net.load_state_dict(state["model"], strict=True)
    opt.load_state_dict(state["optimizer"])
    if "rng" in state:
        torch.set_rng_state(state["rng"]["cpu"])
        torch.cuda.set_rng_state(state["rng"]["cuda"], opt.device)
    return state.get("extra")


# ------------------------------------------------------------------------------------------------ reference format
def reference_parameter_names(state_dict_keys) -> List[str]:
    """Names of the reference LightningModule's `parameters()` in order, from its checkpoint's `state_dict` key order:
    the dynamics network's parameters then `ddpm.gamma.gamma` (the `num_nodes_distribution` entries are buffers).  This
    is the order of AdamW's positional `state` keys (`configure_optimizers` passes `self.parameters()`)."""
    return [k for k in state_dict_keys if k.startswith(DYNAMICS_PREFIX) or k == GAMMA_KEY]


def _parse_reference(ckpt: dict, cfg: DenoiserConfig, need_optimizer: bool):
    """Validate a reference checkpoint against `cfg`; returns (weights by name, parameter names, AdamW state dict)."""
    sd = ckpt["state_dict"]
    if cfg.noise_schedule == "learned" or any(k.startswith("ddpm.gamma.") and k != GAMMA_KEY for k in sd):
        raise ValueError("learned noise schedules are not supported (the checkpoint's ddpm.gamma is a GammaNetwork)")
    if GAMMA_KEY not in sd:
        raise ValueError(f"checkpoint has no {GAMMA_KEY}")
    weights = {k[len(DYNAMICS_PREFIX):]: v for k, v in sd.items() if k.startswith(DYNAMICS_PREFIX)}
    _check_weights(weights, cfg, "checkpoint")
    gamma = gamma_table(cfg.num_timesteps, cfg.noise_precision, cfg.noise_schedule)
    if not torch.equal(sd[GAMMA_KEY].detach().cpu(), gamma):
        raise ValueError(f"{GAMMA_KEY} differs from this denoiser's schedule ({cfg.noise_schedule}, "
                         f"T={cfg.num_timesteps}, precision {cfg.noise_precision})")
    names = reference_parameter_names(sd.keys())
    osd = None
    if need_optimizer:
        states = ckpt.get("optimizer_states")
        if not states:
            raise ValueError("checkpoint has no optimizer_states")
        osd = states[0]
        if len(osd["param_groups"]) != 1:
            raise ValueError(f"expected one AdamW parameter group, found {len(osd['param_groups'])}")
        pg = osd["param_groups"][0]
        if len(pg["params"]) != len(names):
            raise ValueError(f"AdamW holds {len(pg['params'])} parameters, the checkpoint's state_dict {len(names)}")
        if pg.get("maximize", False):
            raise ValueError("AdamW with maximize=True is not supported")
    return weights, names, osd


def _seeded_state_words(step: int, queue_len: int) -> torch.Tensor:
    st = np.zeros(STATE_WORDS, dtype=np.int32)
    st[0] = step
    st[1] = 1                                      # a fresh Queue seeded with 3000 (qm9_mol_gen_ddpm.py:148-149)
    st[2] = 1 % queue_len
    st[8:9] = np.array([3000.0], dtype=np.float32).view(np.int32)
    return torch.from_numpy(st)


def reference_to_training_state(ckpt: dict, cfg: DenoiserConfig, param_names: List[str], hyperparameters: dict,
                                ema_ckpt: Optional[dict] = None) -> dict:
    """A reference Lightning checkpoint as a `training_state` dict (no generator states) for a GCDMTrainTail holding the
    parameters `param_names` in that order.  AdamW's lr / betas / eps / weight_decay / amsgrad and step count come from
    the checkpoint, `queue_len`, `ema_decay` and `clip` from `hyperparameters`; the clip history is seeded afresh.  Pure
    function on the host; raises ValueError on anything it cannot map."""
    weights, names, osd = _parse_reference(ckpt, cfg, True)
    pg = osd["param_groups"][0]
    by_name = {}
    for pos, name in zip(pg["params"], names):
        if name.startswith(DYNAMICS_PREFIX):
            by_name[name[len(DYNAMICS_PREFIX):]] = osd["state"].get(pos)
    have = [s is not None for s in by_name.values()]
    if any(have) and not all(have):
        raise ValueError("AdamW state exists for some dynamics parameters but not for others")
    steps = {int(s["step"]) for s in by_name.values() if s is not None}
    if len(steps) > 1:
        raise ValueError(f"AdamW step counts differ between parameters: {sorted(steps)}")
    step = steps.pop() if steps else 0

    keys = list(ckpt["state_dict"].keys())
    ema_cb = ckpt.get("callbacks", {}).get("EMA", {})
    if ema_ckpt is not None:
        ema = {k[len(DYNAMICS_PREFIX):]: v for k, v in ema_ckpt["state_dict"].items() if k.startswith(DYNAMICS_PREFIX)}
    elif ema_cb.get("ema_weights") is not None:
        lst = list(ema_cb["ema_weights"])
        if len(lst) != len(keys):
            raise ValueError(f"callbacks['EMA']['ema_weights'] has {len(lst)} entries, the state_dict {len(keys)}")
        ema = {k[len(DYNAMICS_PREFIX):]: v for k, v in zip(keys, lst) if k.startswith(DYNAMICS_PREFIX)}
    else:
        warnings.warn("we were unable to find the associated EMA weights when re-loading, "
                      "training will start with new EMA weights.", UserWarning)
        ema = weights
    _check_weights(ema, cfg, "EMA weights")

    def moment(k):
        return [by_name[n][k].detach().float().clone() if by_name[n] is not None else torch.zeros(weights[n].shape)
                for n in param_names]

    amsgrad = bool(pg["amsgrad"])
    hp = dict(hyperparameters, lr=pg["lr"], betas=tuple(pg["betas"]), eps=pg["eps"], weight_decay=pg["weight_decay"],
              amsgrad=amsgrad)
    opt_sd = {"version": STATE_DICT_VERSION, "hyperparameters": hp, "shapes": [tuple(weights[n].shape) for n in param_names],
              "exp_avg": moment("exp_avg"), "exp_avg_sq": moment("exp_avg_sq"),
              "max_exp_avg_sq": moment("max_exp_avg_sq") if amsgrad else None,
              "ema": [ema[n].detach().float().clone() for n in param_names],
              "state": _seeded_state_words(step, hp["queue_len"])}
    model = OrderedDict((n, weights[n].detach().float().clone()) for n in parameter_shapes(cfg))
    return {"version": TRAINING_STATE_VERSION, "model": model, "param_names": list(param_names), "optimizer": opt_sd,
            "extra": None}


def training_state_to_reference(state: dict, template: dict, cfg: DenoiserConfig, epoch: Optional[int] = None,
                                global_step: Optional[int] = None) -> Tuple[dict, dict]:
    """A `training_state` dict written into the reference's checkpoint format, using `template` (a reference checkpoint
    of the same model) for everything the library does not own.  Pure function on the host; see
    `to_reference_checkpoint`."""
    _, names, osd = _parse_reference(template, cfg, True)
    opt_sd = state["optimizer"]
    index = {n: i for i, n in enumerate(state["param_names"])}
    hp = opt_sd["hyperparameters"]
    step = int(opt_sd["state"][0])
    pg0 = osd["param_groups"][0]
    step_like = next((s["step"] for s in osd["state"].values() if "step" in s), torch.tensor(0.0))

    def as_step(v):
        if isinstance(step_like, torch.Tensor):
            return torch.full_like(step_like, float(v))
        return type(step_like)(v)

    def like(t, ref):
        return t.detach().to(device=ref.device, dtype=ref.dtype).clone()

    tsd = template["state_dict"]
    keys = list(tsd.keys())
    weights, ema_w = OrderedDict(), {}
    for k, v in tsd.items():
        n = k[len(DYNAMICS_PREFIX):]
        if k.startswith(DYNAMICS_PREFIX):
            weights[k] = like(state["model"][n], v)
            ema_w[k] = like(opt_sd["ema"][index[n]], v)
        else:
            weights[k] = v

    adam = {}
    for pos, name in zip(pg0["params"], names):
        if not name.startswith(DYNAMICS_PREFIX):
            if pos in osd["state"]:
                adam[pos] = osd["state"][pos]
            continue
        i, ref = index[name[len(DYNAMICS_PREFIX):]], tsd[name]
        s = {"step": as_step(step), "exp_avg": like(opt_sd["exp_avg"][i], ref),
             "exp_avg_sq": like(opt_sd["exp_avg_sq"][i], ref)}
        if hp["amsgrad"]:
            s["max_exp_avg_sq"] = like(opt_sd["max_exp_avg_sq"][i], ref)
        adam[pos] = s
    group = dict(pg0, lr=hp["lr"], betas=type(pg0["betas"])(hp["betas"]), eps=hp["eps"],
                 weight_decay=hp["weight_decay"], amsgrad=hp["amsgrad"])

    callbacks = dict(template.get("callbacks", {}))
    ema_state = dict(callbacks.get("EMA", {"cur_step": None}))
    old = ema_state.get("ema_weights")
    old = list(old) if old is not None else list(tsd.values())   # the EMA callback starts from the state_dict's values
    ema_state["ema_weights"] = [ema_w.get(k, old[j]) for j, k in enumerate(keys)]
    callbacks["EMA"] = ema_state

    ckpt = dict(template)
    ckpt["state_dict"] = weights
    ckpt["optimizer_states"] = [dict(osd, state=adam, param_groups=[group])] + list(template["optimizer_states"][1:])
    ckpt["callbacks"] = callbacks
    if epoch is not None:
        ckpt["epoch"] = epoch
    if global_step is not None:
        ckpt["global_step"] = global_step
    ema_ckpt = dict(ckpt)
    ema_ckpt["state_dict"] = OrderedDict(zip(keys, ema_state["ema_weights"]))
    return ckpt, ema_ckpt


def from_reference_checkpoint(ckpt: dict, net, opt: Optional[GCDMTrainTail] = None,
                              ema_ckpt: Optional[dict] = None) -> None:
    """Load a reference Lightning checkpoint (a dict, e.g. `torch.load(path, map_location="cpu")`) into `net` and, when
    given, `opt`.

    Weights: the `ddpm.dynamics_network.` entries, strictly; `ddpm.gamma.gamma` must equal this denoiser's schedule
    (a different schedule, precision or T raises).  AdamW: `optimizer_states[0]`, mapped from positions to names through
    the checkpoint's own parameter order (never through `net`'s), with its hyperparameters and step count.  EMA weights:
    the `-EMA.ckpt` companion's `state_dict` when `ema_ckpt` is given, else `callbacks["EMA"]["ema_weights"]`, else the
    weights with a UserWarning (the reference's precedence).  The clip history restarts from one entry of 3000, as a
    resumed reference run's `Queue` does.  Everything is checked before anything is copied: a mismatch raises ValueError
    and loads nothing."""
    if opt is None:
        weights, _, _ = _parse_reference(ckpt, net.cfg, False)
        net.load_state_dict(weights, strict=True)
        return
    state = reference_to_training_state(ckpt, net.cfg, _names_in_opt_order(net, opt), opt.hyperparameters, ema_ckpt)
    load_training_state(state, net, opt)


def to_reference_checkpoint(template: dict, net, opt: GCDMTrainTail, epoch: Optional[int] = None,
                            global_step: Optional[int] = None) -> Tuple[dict, dict]:
    """Write the library run into the reference's checkpoint format: returns `(ckpt, ema_ckpt)`, to be saved as
    `<name>.ckpt` and `<name>-EMA.ckpt`.  `template` is a reference checkpoint of the same model; what the library does
    not own (the `num_nodes_distribution` buffers, `ddpm.gamma.gamma`, `hyper_parameters`, `loops`, other callbacks,
    `lr_schedulers`) is carried over from it untouched.  Filled in: the dynamics weights, AdamW's per-position `state`
    (with `step` stored as the template stores it) and `param_groups` hyperparameters, `callbacks["EMA"]["ema_weights"]`
    (entries outside the dynamics network keep the template's values) and, when given, `epoch` / `global_step`.
    `ema_ckpt` is the same checkpoint with the EMA weights as `state_dict`, as `EMAModelCheckpoint._save_checkpoint`
    writes it.  Synchronises."""
    return training_state_to_reference(training_state(net, opt, rng=False), template, net.cfg, epoch, global_step)

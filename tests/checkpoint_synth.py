"""Reference-format Lightning checkpoints synthesised on the CPU, for the checkpoint converter tests.

The layout (key order, shapes, dtypes, which entries are parameters) comes from tests/golden/checkpoint_layout.pt, made
from the reference's own modules.  The contents are made here: seeded weights, a few `torch.optim.AdamW(amsgrad=True,
lr=1e-4, weight_decay=1e-12)` steps with seeded gradients (the reference's optimiser config), the EMA callback's update
(`apply_ema`, src/utils/__init__.py:133-140) over every `state_dict()` value, and the keys Lightning writes."""
from collections import OrderedDict

import torch

from conftest import load_golden

EMA_DECAY = 0.9999


def layout(cname):
    return load_golden("checkpoint_layout")[cname]


def synth_checkpoint(cname, steps=3, seed=0, scale=0.1):
    """Returns (ckpt, params): `params` are the reference-ordered CPU parameters AdamW stepped (its `state` is the
    checkpoint's)."""
    import bdiff
    lay = layout(cname)
    cfg = bdiff.DenoiserConfig.named(cname)
    g = torch.Generator().manual_seed(seed)
    values = OrderedDict()
    for key, shape, dtype in lay["state_dict"]:
        if key == "ddpm.gamma.gamma":
            values[key] = bdiff.schedule.gamma_table(cfg.num_timesteps, cfg.noise_precision, cfg.noise_schedule)
        elif key == "ddpm.num_nodes_distribution.num_nodes":
            values[key] = torch.tensor(sorted(lay["histogram"]), dtype=getattr(torch, dtype))
        elif key == "ddpm.num_nodes_distribution.prob":
            p = torch.tensor([float(lay["histogram"][k]) for k in sorted(lay["histogram"])])
            values[key] = (p / p.sum()).to(getattr(torch, dtype))
        else:
            values[key] = (torch.randn(shape, generator=g) * scale).to(getattr(torch, dtype))
    params = [torch.nn.Parameter(values[k].clone(), requires_grad=k != "ddpm.gamma.gamma") for k in lay["parameters"]]
    by_key = dict(zip(lay["parameters"], params))
    opt = torch.optim.AdamW(params, lr=1e-4, weight_decay=1e-12, amsgrad=True)
    sd = lambda: OrderedDict((k, by_key[k].detach() if k in by_key else v) for k, v in values.items())
    ema = [v.detach().clone() for v in sd().values()]
    for _ in range(steps):
        for p in params:
            if p.requires_grad:
                p.grad = torch.randn(p.shape, generator=g) * 0.01
        opt.step()
        for w, e in zip(sd().values(), ema):
            if e.dtype != torch.long and w.dtype != torch.long:
                diff = e.data - w.data
                diff.mul_(1.0 - EMA_DECAY)
                e.sub_(diff)
    ckpt = {
        "epoch": 1, "global_step": steps, "pytorch-lightning_version": "1.7.7",
        "state_dict": OrderedDict((k, v.clone()) for k, v in sd().items()),
        "loops": {"fit_loop": {"epoch_progress": {"current": {"completed": 1}}}},
        "callbacks": {"EMA": {"cur_step": steps - 1, "ema_weights": ema},
                      "EMAModelCheckpoint{'monitor': 'val/loss', 'mode': 'min'}": {"best_model_score": torch.tensor(1.5)}},
        "optimizer_states": [opt.state_dict()],
        "lr_schedulers": [{"best": 1.0, "num_bad_epochs": 0}],
        "hyper_parameters": {"diffusion_cfg": {"num_timesteps": cfg.num_timesteps}},
    }
    return ckpt, params


def assert_same(a, b, path="ckpt"):
    """Recursive bit-for-bit equality of checkpoint dicts (tensors: dtype, shape and bits)."""
    assert type(a) is type(b) or (isinstance(a, dict) and isinstance(b, dict)), f"{path}: {type(a)} vs {type(b)}"
    if isinstance(a, torch.Tensor):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), path
    elif isinstance(a, dict):
        assert list(a.keys()) == list(b.keys()), f"{path}: keys differ"
        for k in a:
            assert_same(a[k], b[k], f"{path}[{k!r}]")
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), f"{path}: length"
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, f"{path}[{i}]")
    else:
        assert a == b, f"{path}: {a!r} vs {b!r}"

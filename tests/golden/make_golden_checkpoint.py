#!/usr/bin/env python
"""Golden fixture for the checkpoint converters (bdiff/checkpoint.py): the layout of the reference's Lightning
checkpoints, generated from the REFERENCE's own modules in the build container (through oracle/ref_shim.py).
Run:  python tests/golden/make_golden_checkpoint.py

checkpoint_layout.pt holds, for each shipped config (qm9, qm9_cond, geom), names and shapes only (no weights):
  state_dict   [(key, shape, dtype name)] in the `state_dict()` order of the LightningModule (`ddpm.` prefix);
  parameters   the `parameters()` names in order: the positions of AdamW's `state` (configure_optimizers passes
               `self.parameters()`, qm9_mol_gen_ddpm.py:1246-1264);
  buffers      the keys that are buffers;
  histogram    the `n_nodes` histogram used to size the `num_nodes_distribution` buffers.

The script builds the LightningModule itself (`QM9MoleculeGenerationDDPM` / `GEOMMoleculeGenerationDDPM`, with
Lightning's base class replaced by `nn.Module`) and checks that its `state_dict()` is exactly `ddpm.` + the
`EquivariantVariationalDiffusion`'s: the molecular metrics, node-type distribution and gradient-norm `Queue` are plain
Python objects, and the `torchmetrics.MeanMetric` modules it registers keep their states out of the state_dict.  That
last point holds because torchmetrics (0.10.2 in the reference's environment) registers metric states with
`Metric.add_state(..., persistent=False)` by default and `MeanMetric` does not override it; torchmetrics is not installed
here, so the stand-in below registers its states the same way, and the check confirms that the module adds nothing
else."""
import inspect
import os
import socket
import sys
from types import SimpleNamespace
from unittest.mock import MagicMock

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "bio-diffusion_b200"))
import ref_shim  # noqa: E402

from bdiff.datasets import GEOM_N_NODES, QM9_N_NODES  # noqa: E402

EXTRA_STUBS = ["openbabel", "rdkit.Chem.rdForceFieldHelpers", "torch_geometric.loader.dataloader", "torch_geometric.typing"]


def _no_network(*a, **kw):
    raise RuntimeError("make_golden_checkpoint.py runs offline")


# BasicMolecularMetrics fetches the QM9 SMILES list when it is not given one; the script never needs it
socket.getaddrinfo = socket.create_connection = _no_network
socket.socket.connect = _no_network
OUT = os.path.join(ROOT, "tests", "golden", "checkpoint_layout.pt")


class _LightningModule(nn.Module):
    """Lightning's base class as far as the module's __init__ uses it."""

    def save_hyperparameters(self, logger=False):
        frame = inspect.currentframe().f_back
        args = {k: v for k, v in frame.f_locals.items() if k not in ("self", "__class__", "kwargs")}
        self.hparams = SimpleNamespace(**args)


class _MeanMetric(nn.Module):
    """torchmetrics.MeanMetric's state registration: `add_state` defaults to persistent=False."""

    def __init__(self, *a, **kw):
        super().__init__()
        self.register_buffer("value", torch.tensor(0.0), persistent=False)
        self.register_buffer("weight", torch.tensor(0.0), persistent=False)


def lightning_module(cname):
    """The reference LightningModule for a shipped config, with the dataset histogram of that config."""
    ref_shim.install()
    for name in EXTRA_STUBS:         # imported by the module's file for sampling metrics and plots, not used here
        sys.modules.setdefault(name, MagicMock())
    sys.modules["pytorch_lightning"].LightningModule = _LightningModule
    sys.modules["torchmetrics"].MeanMetric = _MeanMetric
    geom = cname == "geom"
    if geom:
        import src.models.geom_mol_gen_ddpm as M
        cls = M.GEOMMoleculeGenerationDDPM
    else:
        import src.models.qm9_mol_gen_ddpm as M
        cls = M.QM9MoleculeGenerationDDPM
    M.LightningModule = _LightningModule
    M.torchmetrics.MeanMetric = _MeanMetric
    M.BasicMolecularMetrics = MagicMock()   # sampling metrics: a plain object with no tensors (and it would download)
    cond = ("alpha",) if cname == "qm9_cond" else ()
    model_cfg, module_cfg, layer_cfg, diffusion_cfg, dataloader_cfg = ref_shim.qm9_cfgs(
        conditioning=cond, include_charges=cname == "qm9", num_atom_types=16 if geom else 5, geom=geom)
    diffusion_cfg["num_eval_samples"] = 8
    diffusion_cfg["verbose"] = False
    dataloader_cfg["dataset"] = "GEOM" if geom else "QM9"
    dataloader_cfg["data_dir"] = "/nonexistent"
    dataloader_cfg["smiles_filepath"] = None
    torch.manual_seed(0)
    return cls(optimizer=None, scheduler=None, model_cfg=model_cfg, module_cfg=module_cfg, layer_cfg=layer_cfg,
               diffusion_cfg=diffusion_cfg, dataloader_cfg=dataloader_cfg)


def layout(cname):
    hist = GEOM_N_NODES if cname == "geom" else QM9_N_NODES
    ddpm, _ = ref_shim.build_reference_ddpm(cname, seed=0, n_nodes_hist=dict(hist))
    sd = ddpm.state_dict()
    module = lightning_module(cname)
    mkeys = list(module.state_dict().keys())
    assert mkeys == ["ddpm." + k for k in sd], f"{cname}: the LightningModule's state_dict is not ddpm.'s"
    assert [n for n, _ in module.named_parameters()] == ["ddpm." + n for n, _ in ddpm.named_parameters()]
    for k in mkeys:
        assert tuple(module.state_dict()[k].shape) == tuple(sd[k[5:]].shape), k
    return {"state_dict": [("ddpm." + k, tuple(v.shape), str(v.dtype).replace("torch.", "")) for k, v in sd.items()],
            "parameters": ["ddpm." + n for n, _ in ddpm.named_parameters()],
            "buffers": ["ddpm." + n for n, _ in ddpm.named_buffers()],
            "histogram": {int(k): int(v) for k, v in hist.items()}}


def main():
    out = {c: layout(c) for c in ("qm9", "qm9_cond", "geom")}
    torch.save(out, OUT)
    for c, v in out.items():
        print(f"{c}: {len(v['state_dict'])} state_dict entries, {len(v['parameters'])} parameters, "
              f"buffers {v['buffers']}")


if __name__ == "__main__":
    main()

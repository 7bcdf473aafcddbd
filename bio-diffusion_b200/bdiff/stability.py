"""Batched molecular-stability check on the GPU — mirrors `check_molecular_stability(positions, atom_types,
dataset_info)` of the reference (src/datamodules/components/edm/__init__.py:91-124), for a whole sampled batch in one
kernel (`bdiff_check_stability`) instead of a Python loop over molecules with an n x n cdist each."""
import ctypes as C
from typing import Dict, Sequence, Tuple, Union

import numpy as np
import torch

from . import _lib


def _allowed_mask(atom_decoder: Sequence[str], allowed_bonds: Dict[str, Union[int, Sequence[int]]]) -> np.ndarray:
    out = np.zeros(len(atom_decoder), dtype=np.uint32)
    for i, sym in enumerate(atom_decoder):
        v = allowed_bonds[sym]
        for c in ([v] if isinstance(v, int) else list(v)):
            if not 0 <= int(c) < 32:
                raise ValueError(f"allowed bond count {c} for {sym} outside [0, 32)")
            out[i] |= np.uint32(1) << np.uint32(c)
    return out


def _check_batch(positions: torch.Tensor, atom_types: torch.Tensor, num_nodes: torch.Tensor, a: int) -> torch.Tensor:
    """positions [N,3], atom_types [N] in [0, a), num_nodes [B] >= 0 summing to N; returns num_nodes int64 on the host."""
    nn = num_nodes.detach().to(torch.int64).cpu()
    n = int(positions.shape[0])
    if positions.shape != (n, 3) or atom_types.shape != (n,) or int(nn.sum()) != n or (nn < 0).any():
        raise ValueError("positions [N,3], atom_types [N] and num_nodes (summing to N) expected")
    if n and (int(atom_types.min()) < 0 or int(atom_types.max()) >= a):
        raise ValueError("atom type outside the decoder")
    return nn


def stability_inputs(positions: torch.Tensor, atom_types: torch.Tensor, num_nodes: torch.Tensor, dataset_info: dict,
                     allowed_bonds: Dict[str, Union[int, Sequence[int]]]) -> torch.Tensor:
    """The argument checks of check_molecular_stability_batch that do not depend on the device; returns num_nodes int64
    on the host."""
    dec = list(dataset_info["atom_decoder"])
    _allowed_mask(dec, allowed_bonds)
    return _check_batch(positions, atom_types, num_nodes, len(dec))


def check_molecular_stability_batch(positions: torch.Tensor, atom_types: torch.Tensor, num_nodes: torch.Tensor,
                                    dataset_info: dict, allowed_bonds: Dict[str, Union[int, Sequence[int]]],
                                    margins: Tuple[float, float, float] = (10.0, 5.0, 3.0),
                                    limit_bonds_to_one: bool = False):
    """positions [N,3] and atom_types [N] (CUDA, molecules concatenated), num_nodes [B]; `dataset_info` as in the
    reference (`atom_decoder`, `bonds1`, `bonds2`, `bonds3` = get_bond_length_arrays(atom_encoder)), `allowed_bonds`
    and `margins` = the constants of edm/constants.py.  Returns (molecule_stable bool[B], nr_stable_bonds int32[B],
    n int32[B]) — per molecule what the reference function returns — and the per-atom bond counts int32[N]."""
    if positions.device.type != "cuda":
        raise _lib.BdiffError("check_molecular_stability_batch runs on CUDA tensors only (no CPU fallback)")
    lib = _lib.load()
    dev = positions.device
    dec = list(dataset_info["atom_decoder"])
    a = len(dec)
    tabs = [torch.as_tensor(np.asarray(dataset_info[k], dtype=np.float32)).reshape(a, a).contiguous().to(dev)
            for k in ("bonds1", "bonds2", "bonds3")]
    mask = torch.from_numpy(_allowed_mask(dec, allowed_bonds).view(np.int32)).to(dev)
    x = positions.detach().to(torch.float32).contiguous()
    t = atom_types.detach().to(torch.int32).contiguous()
    nn = _check_batch(x, t, num_nodes, a)
    n = int(x.shape[0])
    b = int(nn.numel())
    off = torch.zeros(b + 1, dtype=torch.int32)
    off[1:] = torch.cumsum(nn, 0).to(torch.int32)
    off = off.to(dev)
    nr_bonds = torch.zeros(n, dtype=torch.int32, device=dev)
    nr_stable = torch.zeros(b, dtype=torch.int32, device=dev)
    stable = torch.zeros(b, dtype=torch.int32, device=dev)
    rc = lib.bdiff_check_stability(
        C.c_void_p(torch.cuda.current_stream(dev).cuda_stream), C.c_void_p(x.data_ptr()), C.c_void_p(t.data_ptr()),
        C.c_void_p(off.data_ptr()), C.c_int32(b), C.c_int32(a), C.c_void_p(tabs[0].data_ptr()),
        C.c_void_p(tabs[1].data_ptr()), C.c_void_p(tabs[2].data_ptr()), C.c_float(margins[0]), C.c_float(margins[1]),
        C.c_float(margins[2]), C.c_void_p(mask.data_ptr()), C.c_int32(int(bool(limit_bonds_to_one))),
        C.c_void_p(nr_bonds.data_ptr()), C.c_void_p(nr_stable.data_ptr()), C.c_void_p(stable.data_ptr()))
    if rc != 0:
        raise _lib.BdiffError(f"bdiff_check_stability failed with code {rc}")
    return stable.bool(), nr_stable, nn.to(torch.int32).to(dev), nr_bonds


def bond_orders_batch(positions: torch.Tensor, atom_types: torch.Tensor, num_nodes: torch.Tensor, dataset_info: dict,
                      margins: Tuple[float, float, float] = (10.0, 5.0, 3.0)):
    """The (X, A, E) graph `make_mol_edm` builds before handing it to RDKit (rdkit_functions.py:276-321), for a whole batch:
    returns `bonds` int64 [M, 4] with rows (molecule, i, j, bond type) for every pair i > j with a bond, in the order the
    reference's `torch.nonzero(A)` loop adds them to the RWMol, and the dense per-molecule int8 matrices E (packed, with
    their offsets).  limit_bonds_to_one = ("GEOM" in dataset_info["name"]) as in the reference."""
    if positions.device.type != "cuda":
        raise _lib.BdiffError("bond_orders_batch runs on CUDA tensors only (no CPU fallback)")
    lib = _lib.load()
    dev = positions.device
    dec = list(dataset_info["atom_decoder"])
    a = len(dec)
    tabs = [torch.as_tensor(np.asarray(dataset_info[k], dtype=np.float32)).reshape(a, a).contiguous().to(dev)
            for k in ("bonds1", "bonds2", "bonds3")]
    x = positions.detach().to(torch.float32).contiguous()
    t = atom_types.detach().to(torch.int32).contiguous()
    nn = _check_batch(x, t, num_nodes, a)                     # a type outside the decoder would index past the tables
    n = int(x.shape[0])
    b = int(nn.numel())
    off = torch.zeros(b + 1, dtype=torch.int32)
    off[1:] = torch.cumsum(nn, 0).to(torch.int32)
    poff = torch.zeros(b + 1, dtype=torch.int64)
    poff[1:] = torch.cumsum(nn * nn, 0)
    e = torch.zeros(max(int(poff[-1]), 1), dtype=torch.int8, device=dev)
    off_d, poff_d = off.to(dev), poff.to(dev)
    limit = "GEOM" in str(dataset_info.get("name", ""))
    rc = lib.bdiff_bond_orders(
        C.c_void_p(torch.cuda.current_stream(dev).cuda_stream), C.c_void_p(x.data_ptr()), C.c_void_p(t.data_ptr()),
        C.c_void_p(off_d.data_ptr()), C.c_void_p(poff_d.data_ptr()), C.c_int32(b), C.c_int32(a),
        C.c_void_p(tabs[0].data_ptr()), C.c_void_p(tabs[1].data_ptr()), C.c_void_p(tabs[2].data_ptr()),
        C.c_float(margins[0]), C.c_float(margins[1]), C.c_float(margins[2]), C.c_int32(int(limit)), C.c_void_p(e.data_ptr()))
    if rc != 0:
        raise _lib.BdiffError(f"bdiff_bond_orders failed with code {rc}")
    flat = torch.nonzero(e[: int(poff[-1])]).reshape(-1)                     # ascending = (molecule, i, j) row-major
    mol = torch.searchsorted(poff_d[1:], flat, right=True)
    loc = flat - poff_d[mol]
    nk = nn.to(dev)[mol]
    bonds = torch.stack((mol, loc // nk, loc % nk, e[flat].to(torch.int64)), dim=1)
    return bonds, e, poff_d

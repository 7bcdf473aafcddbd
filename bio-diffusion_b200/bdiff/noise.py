"""Counter-based Gaussian noise (Philox4x32-10 + Box-Muller) and the sampling constants of the native chain.

Every value is a pure function of (seed, draw index, element index); include/bdiff.h ("sampling through the C ABI alone")
states the layout.  `philox_noise(seed)` hands those draws to the `noise=` hook of GCDMSampler in draw order, so the Python
chain can replay what `bdiff_sample` (GCDMSampler.sample(seed=...)) computes inside its kernels.
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Tuple

import torch

from . import _lib
from .config import DenoiserConfig


def _stream() -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def noise_fill(seed: int, draw_index: int, shape: Tuple[int, ...], device=None) -> torch.Tensor:
    """Draw `draw_index` of `seed` as an fp32 tensor of `shape` (row-major element order) on a CUDA device."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    out = torch.empty(shape, dtype=torch.float32, device=dev)
    rows = int(shape[0]) if len(shape) else 1
    cols = math.prod(shape[1:]) if len(shape) > 1 else 1
    with torch.cuda.device(dev):
        rc = _lib.load().bdiff_noise_fill(_stream(), int(seed), int(draw_index), rows, cols, C.c_void_p(out.data_ptr()))
    if rc != 0:
        raise _lib.BdiffError(f"bdiff_noise_fill failed (code {rc})")
    return out


def philox_words(seed: int, draw_index: int, blocks: int, device=None) -> torch.Tensor:
    """The raw Philox4x32-10 words of blocks 0 .. blocks-1 of a draw: int64 [blocks, 4] holding the uint32 values."""
    dev = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
    out = torch.empty((blocks, 4), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        rc = _lib.load().bdiff_philox_fill(_stream(), int(seed), int(draw_index), int(blocks), C.c_void_p(out.data_ptr()))
    if rc != 0:
        raise _lib.BdiffError(f"bdiff_philox_fill failed (code {rc})")
    return out.long() & 0xFFFFFFFF


class philox_noise:
    """NoiseFn for GCDMSampler's `noise=` hook: call k returns draw k of `seed` (draw 0 first).  Stateful over the draw
    order, like the device generator it stands in for; make a new one per chain."""

    def __init__(self, seed: int, device=None):
        self.seed = int(seed)
        self.device = device
        self.draws = 0

    def __call__(self, shape: Tuple[int, ...]) -> torch.Tensor:
        out = noise_fill(self.seed, self.draws, tuple(shape), self.device)
        self.draws += 1
        return out


def sample_config(cfg: DenoiserConfig) -> _lib.SampleConfig:
    """The bdiff_sample_config of a denoiser configuration."""
    if not cfg.noise_schedule.startswith("polynomial"):
        raise NotImplementedError(f"noise schedule '{cfg.noise_schedule}' (shipped configs use polynomial_2)")
    nb = [0.0 if v is None else float(v) for v in cfg.norm_biases]
    return _lib.SampleConfig(num_atom_types=cfg.num_atom_types, include_charges=int(cfg.include_charges),
                             model_timesteps=cfg.num_timesteps, reserved=0,
                             schedule_power=float(cfg.noise_schedule.split("_")[1]),
                             noise_precision=float(cfg.noise_precision),
                             norm_values=(C.c_float * 3)(*[float(v) for v in cfg.norm_values]),
                             norm_biases=(C.c_float * 3)(*nb))


def schedule_tables(cfg: DenoiserConfig, num_timesteps: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The library's host-side tables (bdiff_schedule_tables; no GPU needed): coef [num_timesteps, 4], decode [4]."""
    coef = torch.empty((num_timesteps, 4), dtype=torch.float32)
    dec = torch.empty(4, dtype=torch.float32)
    sc = sample_config(cfg)
    rc = _lib.load().bdiff_schedule_tables(C.byref(sc), int(num_timesteps), C.c_void_p(coef.data_ptr()),
                                           C.c_void_p(dec.data_ptr()))
    if rc != 0:
        raise _lib.BdiffError(f"bdiff_schedule_tables failed (code {rc})")
    return coef, dec


def repaint_tables(cfg: DenoiserConfig, num_timesteps: int, num_resamplings: int, jump_length: int,
                   return_frames: int = 1) -> dict:
    """The library's RePaint program (bdiff_repaint_tables; no GPU needed), with the keys of schedule.repaint_program:
    rev [ops, 4], known [ops, 2], jump [jumps, 4], decode [4], s_of_op / slot / jump_after [ops], num_jumps, and the first
    draw of each op (op_draw [ops]), jump (jump_draw [jumps]) and of the decode (decode_draw)."""
    sc = sample_config(cfg)
    lib = _lib.load()
    args = (C.byref(sc), int(num_timesteps), int(num_resamplings), int(jump_length), int(return_frames))
    ops, jumps = C.c_int32(0), C.c_int32(0)
    if lib.bdiff_repaint_tables(*args, C.byref(ops), C.byref(jumps), *([None] * 10)) != 0:
        raise _lib.BdiffError("bdiff_repaint_tables refused its arguments")
    o, j = ops.value, jumps.value
    t = dict(rev=torch.empty((o, 4)), known=torch.empty((o, 2)), jump=torch.empty((j, 4)), decode=torch.empty(4),
             s_of_op=torch.empty(o, dtype=torch.int32), slot=torch.empty(o, dtype=torch.int32),
             jump_after=torch.empty(o, dtype=torch.uint8), op_draw=torch.empty(o, dtype=torch.int64),
             jump_draw=torch.empty(j, dtype=torch.int64))
    dd = C.c_uint64(0)
    ptrs = [C.c_void_p(t[k].data_ptr()) for k in ("rev", "known", "jump", "decode", "s_of_op", "slot", "jump_after",
                                                  "op_draw", "jump_draw")]
    if lib.bdiff_repaint_tables(*args, C.byref(ops), C.byref(jumps), *ptrs, C.byref(dd)) != 0:
        raise _lib.BdiffError("bdiff_repaint_tables failed")
    t.update(num_jumps=j, decode_draw=dd.value, jump_after=t["jump_after"].bool())
    return t

"""Optimiser side of a GCDM training step on the CUDA library: adaptive gradient-norm clipping, AdamW(amsgrad) and the
EMA of the weights as three multi-tensor kernels (`bdiff_optimizer_step`, csrc/bdiff_optim.cu) — mirrors what the
reference does with `configure_gradient_clipping` (qm9_mol_gen_ddpm.py:1267-1304), `torch.optim.AdamW`
(configs/model/*_mol_gen_ddpm.yaml:3-8) and the `EMA` callback (src/utils/__init__.py:71-160) every step.
No host synchronisation in `step()`; the gradient-norm history lives on the device."""
import ctypes as C
from typing import Iterable

import numpy as np
import torch

from . import _lib

STATE_WORDS = 8 + 120


class OptHyper(C.Structure):
    _fields_ = [("lr", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float),
                ("weight_decay", C.c_float), ("ema_decay", C.c_float), ("amsgrad", C.c_int32), ("clip", C.c_int32),
                ("queue_len", C.c_int32)]


class GCDMTrainTail:
    """opt = GCDMTrainTail(model.parameters()); loss.backward(); opt.step(); opt.zero_grad()

    Gradients are accumulated by autograd into persistent buffers owned by this object (`p.grad` is pointed at them
    once), so the device-side pointer table never changes.  `ema_parameters()` are the averaged weights the reference
    evaluates with (`evaluate_ema_weights_instead`)."""

    def __init__(self, params: Iterable[torch.nn.Parameter], lr=1e-4, betas=(0.9, 0.999), eps=1e-8,
                 weight_decay=1e-12, amsgrad=True, ema_decay=0.9999, clip_gradients=True, queue_len=50):
        self.params = [p for p in params if p.requires_grad]
        if not self.params:
            raise ValueError("no trainable parameters")
        dev = self.params[0].device
        if dev.type != "cuda":
            raise _lib.BdiffError("GCDMTrainTail needs CUDA parameters (no CPU fallback)")
        for p in self.params:
            if p.dtype != torch.float32 or not p.is_contiguous() or p.device != dev:
                raise ValueError("parameters must be contiguous fp32 tensors on one device")
        if not 1 <= queue_len <= 120:
            raise ValueError("queue_len must be in [1, 120]")
        self.lib = _lib.load()
        self.device = dev
        self.hyper = OptHyper(lr, betas[0], betas[1], eps, weight_decay, ema_decay, int(bool(amsgrad)),
                              int(bool(clip_gradients)), int(queue_len))
        z = lambda p: torch.zeros_like(p)
        # all gradients in ONE flat buffer (each tensor at a multiple of 64 floats): zero_grad is one memset and the DDP
        # exchange one all-reduce of the buffer itself, no packing
        offs, tot = [], 0
        for p in self.params:
            offs.append(tot)
            tot += (p.numel() + 63) // 64 * 64
        self.grad_flat = torch.zeros(tot, dtype=torch.float32, device=dev)
        self.grads = [self.grad_flat[o:o + p.numel()].view_as(p) for o, p in zip(offs, self.params)]
        self.exp_avg = [z(p) for p in self.params]
        self.exp_avg_sq = [z(p) for p in self.params]
        self.max_exp_avg_sq = [z(p) for p in self.params] if amsgrad else None
        self.ema = [p.detach().clone() for p in self.params]
        for p, g in zip(self.params, self.grads):
            p.grad = g
        self._build_table()
        st = np.zeros(STATE_WORDS, dtype=np.int32)
        st[1] = 1                                   # history seeded with one entry of 3000 (qm9_mol_gen_ddpm.py:148-149)
        st[2] = 1 % queue_len
        st[8:9] = np.array([3000.0], dtype=np.float32).view(np.int32)
        self.state = torch.from_numpy(st).to(dev)
        self.kernel_launches = 0

    def _build_table(self):
        """Device-side pointer table; rebuilt if a parameter's storage moved (GCPNetDynamicsB200.flatten_parameters)."""
        dev, amsgrad = self.device, self.max_exp_avg_sq is not None
        chunk = int(self.lib.bdiff_optimizer_chunk())
        self._ptrs = [p.data_ptr() for p in self.params]
        rec = np.zeros((len(self.params), 7), dtype=np.int64)
        ct, cs = [], []
        for i, p in enumerate(self.params):
            rec[i] = (p.data_ptr(), self.grads[i].data_ptr(), self.exp_avg[i].data_ptr(), self.exp_avg_sq[i].data_ptr(),
                      self.max_exp_avg_sq[i].data_ptr() if amsgrad else 0, self.ema[i].data_ptr(), p.numel())
            for s in range(0, p.numel(), chunk):
                ct.append(i)
                cs.append(s)
        self.table = torch.from_numpy(rec).to(dev)
        self.chunk_tensor = torch.tensor(ct, dtype=torch.int32, device=dev)
        self.chunk_start = torch.tensor(cs, dtype=torch.int64, device=dev)
        self.partial = torch.zeros(len(ct), dtype=torch.float64, device=dev)

    def zero_grad(self):
        self.grad_flat.zero_()

    def allreduce_grads(self, group=None) -> int:
        """DDP gradient exchange (configs/trainer/ddp.yaml): in-place mean over the ranks of the flat gradient buffer, ONE
        NCCL all-reduce.  Returns the number of collectives issued (0 on a single rank)."""
        from .distributed import allreduce_mean_flat_
        return allreduce_mean_flat_(self.grad_flat, group)

    def step(self):
        for p, g in zip(self.params, self.grads):
            if p.grad is None or p.grad.data_ptr() != g.data_ptr():
                raise _lib.BdiffError("p.grad was replaced; keep the buffers GCDMTrainTail installed (use opt.zero_grad())")
        if any(p.data_ptr() != q for p, q in zip(self.params, self._ptrs)):
            self._build_table()
        rc = self.lib.bdiff_optimizer_step(
            C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream), C.c_void_p(self.table.data_ptr()),
            C.c_void_p(self.chunk_tensor.data_ptr()), C.c_void_p(self.chunk_start.data_ptr()),
            C.c_int32(self.chunk_tensor.numel()), C.c_void_p(self.partial.data_ptr()), C.c_void_p(self.state.data_ptr()),
            C.byref(self.hyper))
        if rc != 0:
            raise _lib.BdiffError(f"bdiff_optimizer_step failed with code {rc}")
        # the kernels wrote the parameters through raw pointers: bump their version counters so that everything keyed on
        # (data_ptr, _version) — GCPNetDynamicsB200.sync_weights, autograd's saved-tensor checks — sees the update
        torch.autograd.graph.increment_version(self.params)
        self.kernel_launches += 3

    def ema_parameters(self):
        return self.ema

    def report(self):
        """Host copy of the control state (synchronises): step count, last gradient norm / limit / coefficient."""
        s = self.state.cpu().numpy()
        f = s.view(np.float32)
        n = int(s[1])
        return {"step": int(s[0]), "norm": float(f[3]), "limit": float(f[4]), "coef": float(f[5]),
                "clipped": bool(s[6]), "history": sorted(f[8:8 + n].tolist())}

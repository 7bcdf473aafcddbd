"""Optimiser side of a GCDM training step on the CUDA library: adaptive gradient-norm clipping, AdamW(amsgrad) and the
EMA of the weights as three multi-tensor kernels (`bdiff_optimizer_step`, csrc/bdiff_optim.cu) — mirrors what the
reference does with `configure_gradient_clipping` (qm9_mol_gen_ddpm.py:1267-1304), `torch.optim.AdamW`
(configs/model/*_mol_gen_ddpm.yaml:3-8) and the `EMA` callback (src/utils/__init__.py:71-160) every step.
No host synchronisation in `step()`; the gradient-norm history lives on the device."""
import contextlib
import ctypes as C
from typing import Iterable

import numpy as np
import torch

from . import _lib

STATE_WORDS = 8 + 120
STATE_DICT_VERSION = 1


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
        self._set_hyper(dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=bool(amsgrad),
                             ema_decay=ema_decay, clip=bool(clip_gradients), queue_len=int(queue_len)))
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
        self._ema_swapped = False

    def _set_hyper(self, hp):
        # the Python floats are kept as given so that a checkpoint written from them reproduces its source bit for bit;
        # the kernels read the float32 copy in OptHyper
        self.hyperparameters = dict(hp)
        self.hyper = OptHyper(hp["lr"], hp["betas"][0], hp["betas"][1], hp["eps"], hp["weight_decay"], hp["ema_decay"],
                              int(hp["amsgrad"]), int(hp["clip"]), hp["queue_len"])

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
        if self._ema_swapped:
            raise _lib.BdiffError("the EMA weights are swapped in; swap them back (swap_ema()) before step()")
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

    def swap_ema(self):
        """Exchange the parameters and the EMA weights in place (the reference's `replace_model_weights` /
        `restore_original_weights`, src/utils/__init__.py:206-235); calling it twice restores both bit for bit.  The
        parameters' version counters move, so GCPNetDynamicsB200.sync_weights repacks.  step() refuses to run while the
        EMA weights are swapped in."""
        with torch.no_grad():
            for p, e in zip(self.params, self.ema):
                tmp = p.detach().clone()
                p.detach().copy_(e)
                e.copy_(tmp)
        torch.autograd.graph.increment_version(self.params)
        self._ema_swapped = not self._ema_swapped

    @contextlib.contextmanager
    def ema_applied(self):
        """`with opt.ema_applied(): evaluate(net)` — the parameters hold the EMA weights inside the block only."""
        self.swap_ema()
        try:
            yield self
        finally:
            self.swap_ema()

    def state_dict(self) -> dict:
        """Everything `step()` reads besides the parameters and gradients, as detached clones on the parameters' device:
        hyperparameters, per-tensor shapes, the AdamW moments (and amsgrad maxima), the EMA weights and a copy of the
        control words (`state`: step count, history length, ring position, last norm / limit / coefficient / clipped
        flag and the gradient-norm history, laid out as `bdiff_optimizer_step` documents in include/bdiff.h)."""
        if self._ema_swapped:
            raise _lib.BdiffError("the EMA weights are swapped in; swap them back (swap_ema()) before state_dict()")
        clone = lambda ts: [t.detach().clone() for t in ts]
        return {"version": STATE_DICT_VERSION, "hyperparameters": dict(self.hyperparameters),
                "shapes": [tuple(p.shape) for p in self.params], "exp_avg": clone(self.exp_avg),
                "exp_avg_sq": clone(self.exp_avg_sq),
                "max_exp_avg_sq": clone(self.max_exp_avg_sq) if self.max_exp_avg_sq is not None else None,
                "ema": clone(self.ema), "state": self.state.detach().clone()}

    def _check_state_dict(self, sd: dict) -> None:
        """Raise ValueError naming the first difference between `sd` and this tail's structure; changes nothing."""
        if sd.get("version") != STATE_DICT_VERSION:
            raise ValueError(f"state_dict version {sd.get('version')!r}, expected {STATE_DICT_VERSION}")
        hp = sd["hyperparameters"]
        for k in ("amsgrad", "queue_len"):
            if hp[k] != self.hyperparameters[k]:
                raise ValueError(f"{k}: state_dict has {hp[k]!r}, this GCDMTrainTail has {self.hyperparameters[k]!r}")
        if len(sd["shapes"]) != len(self.params):
            raise ValueError(f"state_dict holds {len(sd['shapes'])} tensors, this GCDMTrainTail {len(self.params)}")
        for i, (s, p) in enumerate(zip(sd["shapes"], self.params)):
            if tuple(s) != tuple(p.shape):
                raise ValueError(f"tensor {i}: state_dict shape {tuple(s)}, parameter shape {tuple(p.shape)}")
        keys = ["exp_avg", "exp_avg_sq", "ema"] + (["max_exp_avg_sq"] if hp["amsgrad"] else [])
        for k in keys:
            ts = sd[k]
            if ts is None or len(ts) != len(self.params):
                raise ValueError(f"{k}: expected {len(self.params)} tensors")
            for i, (t, p) in enumerate(zip(ts, self.params)):
                if tuple(t.shape) != tuple(p.shape) or t.dtype != torch.float32:
                    raise ValueError(f"{k}[{i}]: {tuple(t.shape)} {t.dtype}, expected {tuple(p.shape)} torch.float32")
        st = sd["state"]
        if tuple(st.shape) != (STATE_WORDS,) or st.dtype != torch.int32:
            raise ValueError(f"state: {tuple(st.shape)} {st.dtype}, expected ({STATE_WORDS},) torch.int32")
        w = st.cpu()
        step, n, pos, q = int(w[0]), int(w[1]), int(w[2]), hp["queue_len"]
        if step < 0 or not 0 <= n <= q or not 0 <= pos < q:
            raise ValueError(f"state: step {step}, history length {n}, ring position {pos} do not fit queue_len {q}")

    def load_state_dict(self, sd: dict) -> None:
        """Validate `sd` against this tail (tensor count, shapes, amsgrad, queue_len: ValueError on a mismatch, nothing
        loaded), then copy it in place: the buffers, the device pointer table and the `p.grad` buffers stay the same
        objects.  The saved hyperparameters replace the constructor's, as torch.optim does."""
        if self._ema_swapped:
            raise _lib.BdiffError("the EMA weights are swapped in; swap them back (swap_ema()) before load_state_dict()")
        self._check_state_dict(sd)
        with torch.no_grad():
            for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq", "ema"):
                dst = getattr(self, k)
                if dst is not None:
                    for d, s in zip(dst, sd[k]):
                        d.copy_(s)
            self.state.copy_(sd["state"])
        hp = dict(sd["hyperparameters"])
        hp["betas"] = tuple(hp["betas"])
        self._set_hyper(hp)

    def report(self):
        """Host copy of the control state (synchronises): step count, last gradient norm / limit / coefficient."""
        s = self.state.cpu().numpy()
        f = s.view(np.float32)
        n = int(s[1])
        return {"step": int(s[0]), "norm": float(f[3]), "limit": float(f[4]), "coef": float(f[5]),
                "clipped": bool(s[6]), "history": sorted(f[8:8 + n].tolist())}

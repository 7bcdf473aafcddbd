"""GCPNetDynamicsB200 — drop-in for the reference's `GCPNetDynamics` (src/models/components/gcpnet.py:933-1232).

Same constructor signature, same parameter names/shapes (so `load_state_dict` of reference checkpoints works
with strict=True, state-dict prefix `ddpm.dynamics_network.`), same call contract

    forward(batch, xh[N,3+F], t[N,1], **kwargs) -> (batch, net_out[N,3+F])

but every arithmetic step runs in libbdiff_sm90.so (hand-written sm_90a kernels).  To plug it into the
reference, add it to the `dynamics_networks` dict of src/models/qm9_mol_gen_ddpm.py:101-105 (INTEGRATION.md).
There is no CPU / PyTorch fallback: tensors must live on a CUDA device and the library must be built.

Under autograd (`torch.is_grad_enabled()` and trainable parameters — what the reference's training_step does,
qm9_mol_gen_ddpm.py:340-362) `forward` runs the library's training pass instead of the sampler kernels:
`bdiff_train_forward` keeps the tape, `loss.backward()` reaches `bdiff_train_backward` through a
`torch.autograd.Function` and every parameter receives its gradient (no gradient flows to xh / t: in the GCDM objective
they are data).
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Any, Dict, Optional, Tuple

import torch
from torch import nn

from . import _lib
from .config import DenoiserConfig, parameter_shapes


def _version(t: torch.Tensor) -> int:
    """Version counter of a tensor; inference tensors (the reference samples under torch.inference_mode) have none."""
    try:
        return t._version
    except RuntimeError:
        return -1


class _Node(nn.Module):
    """Anonymous container used to reproduce the reference's dotted parameter names."""


def _register(root: nn.Module, dotted: str, param: nn.Parameter) -> None:
    parts = dotted.split(".")
    mod = root
    for p in parts[:-1]:
        if p not in mod._modules:
            mod.add_module(p, _Node())
        mod = mod._modules[p]
    mod.register_parameter(parts[-1], param)


class _DenoiseTrainFn(torch.autograd.Function):
    """net_out = denoiser(params; xh, t, context) with the library's tape; backward = bdiff_train_backward."""

    @staticmethod
    def forward(ctx, net, batch_index, mask, xh, t, context, num_mols, *params):
        out = net._train_forward(batch_index, mask, xh, t, context, num_mols)
        ctx.net = net
        ctx.tape_id = net._tape_id
        ctx.needs = tuple(p.requires_grad for p in params)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_out):
        net = ctx.net
        if ctx.tape_id != net._tape_id:
            raise RuntimeError("GCPNetDynamicsB200 keeps ONE training tape: a later forward under autograd replaced the "
                               "one this backward needs (call backward() before the next training forward)")
        grads = net._train_backward(d_out)
        return (None,) * 7 + tuple(g if need else None for g, need in zip(grads, ctx.needs))


class GCPNetDynamicsB200(nn.Module):
    def __init__(self, model_cfg=None, module_cfg=None, layer_cfg=None, diffusion_cfg=None, dataloader_cfg=None,
                 *, config: Optional[DenoiserConfig] = None, mode: str = "parity"):
        super().__init__()
        self.cfg = config if config is not None else DenoiserConfig.from_reference_cfgs(
            model_cfg, module_cfg, layer_cfg, diffusion_cfg, dataloader_cfg)
        self.num_x_dims = 3
        self.num_context_node_features = self.cfg.num_context
        self.mode = mode
        self._shapes = parameter_shapes(self.cfg)
        for name, shape in self._shapes.items():
            _register(self, name, nn.Parameter(torch.empty(shape)))
        self.reset_parameters()
        self._handle = None          # bdiff_handle* (created lazily on the first CUDA call)
        self._weights_key = None
        self._plan_key = None
        self._plan_info = None       # (B, N, E)
        self._plan_epoch = 0         # bumped by every bdiff_plan_topology call (device buffers may have moved)
        self._keepalive = None
        self._flat = None            # training: the parameters are views of this flat buffer (library layout)
        self._grad_flat = None
        self._layout = None          # name -> (offset, count)
        self._tape_id = 0

    # ------------------------------------------------------------------------------------------ parameters
    def reset_parameters(self) -> None:
        """nn.Linear's default init (kaiming-uniform, bound 1/sqrt(fan_in)) for every weight/bias pair."""
        with torch.no_grad():
            for name, p in self.named_parameters():
                if name.endswith("weight"):
                    fan_in = p.shape[1]
                else:
                    fan_in = self._shapes[name[:-4] + "weight"][1]
                bound = 1.0 / math.sqrt(fan_in)
                p.uniform_(-bound, bound)

    # ------------------------------------------------------------------------------------------ C-ABI handle
    def _ensure_handle(self):
        if self._handle is not None:
            return self._handle
        lib = _lib.load()
        c = self.cfg
        cfg = _lib.Config(num_h=c.num_h, num_context=c.num_context, num_layers=c.num_layers, h_hidden=c.h_hidden,
                          chi_hidden=c.chi_hidden, e_hidden=c.e_hidden, xi_hidden=c.xi_hidden,
                          mode=_lib.MODE_TENSOR if self.mode == "tensor" else _lib.MODE_PARITY_FP32)
        h = C.c_void_p()
        rc = lib.bdiff_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise _lib.BdiffError(f"bdiff_create failed (code {rc}): {lib.bdiff_last_error(None).decode()}")
        self._handle = h
        return h

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None:
                _lib.load().bdiff_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

    @staticmethod
    def _stream() -> C.c_void_p:
        return C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def sync_weights(self, force: bool = False) -> None:
        """Repack the module's parameters into the kernel layout (bdiff_set_weight per tensor)."""
        key = tuple((p.data_ptr(), _version(p)) for p in self.parameters())
        if not force and key == self._weights_key:
            return
        lib = _lib.load()
        h = self._ensure_handle()
        st = self._stream()
        for name, p in self.named_parameters():
            if not p.is_cuda:
                raise _lib.BdiffError("GCPNetDynamicsB200 parameters must be on a CUDA device (no CPU fallback)")
            t = p.detach()
            if t.dtype != torch.float32 or not t.is_contiguous():
                t = t.float().contiguous()
            shape = (C.c_int64 * t.dim())(*t.shape)
            _lib.check(h, lib.bdiff_set_weight(h, st, name.encode(), C.c_void_p(t.data_ptr()), shape, t.dim()),
                       f"bdiff_set_weight({name})")
        missing = lib.bdiff_weights_missing(h)
        if missing != 0:
            raise _lib.BdiffError(f"{missing} parameter tensors were not set")
        _lib.check(h, lib.bdiff_prepare(h, st), "bdiff_prepare")
        self._weights_key = key

    def plan(self, batch_index: torch.Tensor, mask: torch.Tensor, num_mols: Optional[int] = None) -> Tuple[int, int, int]:
        """Build (or reuse) the implicit edge plan for (batch_index, mask): replaces get_fully_connected_edge_index."""
        key = (batch_index.data_ptr(), _version(batch_index), mask.data_ptr(), _version(mask), batch_index.shape[0])
        if key == self._plan_key:
            return self._plan_info
        if not batch_index.is_cuda:
            raise _lib.BdiffError("batch_index must be a CUDA tensor (no CPU fallback)")
        lib = _lib.load()
        h = self._ensure_handle()
        bi = batch_index.to(torch.int64).contiguous()
        mk = mask.to(torch.uint8).contiguous()
        n = bi.shape[0]
        b = int(num_mols) if num_mols is not None else int(bi[-1].item()) + 1
        e = C.c_int64(0)
        self._plan_key = None        # a failed call may leave no plan (or not this one): never reuse the old key
        _lib.check(h, lib.bdiff_plan_topology(h, self._stream(), b, n, C.c_void_p(bi.data_ptr()),
                                              C.c_void_p(mk.data_ptr()), C.byref(e)), "bdiff_plan_topology")
        self._plan_key = key
        self._plan_epoch += 1
        self._plan_info = (b, n, int(e.value))
        self._keepalive = (batch_index, mask)
        return self._plan_info

    def edge_index(self) -> torch.Tensor:
        """The reference's edge_index int64 [2, E] for the current plan (bit-exact; built on demand)."""
        lib = _lib.load()
        _, _, e = self._plan_info
        dev = self._keepalive[0].device
        out = torch.empty((2, e), dtype=torch.int64, device=dev)
        _lib.check(self._handle, lib.bdiff_edge_index(self._handle, self._stream(), C.c_void_p(out.data_ptr())),
                   "bdiff_edge_index")
        return out

    def debug_tap(self, which: str) -> torch.Tensor:
        """Copy of an intermediate tensor of the last forward (parity tests)."""
        lib = _lib.load()
        rows, cols = C.c_int64(), C.c_int64()
        _lib.check(self._handle, lib.bdiff_debug_tap(self._handle, self._stream(), which.encode(), None,
                                                     C.byref(rows), C.byref(cols)), f"bdiff_debug_tap({which})")
        out = torch.empty((rows.value, cols.value), dtype=torch.float32, device=self._keepalive[0].device)
        _lib.check(self._handle, lib.bdiff_debug_tap(self._handle, self._stream(), which.encode(),
                                                     C.c_void_p(out.data_ptr()), C.byref(rows), C.byref(cols)),
                   f"bdiff_debug_tap({which})")
        return out

    # ------------------------------------------------------------------------------------------ forward
    def denoise(self, batch_index: torch.Tensor, mask: torch.Tensor, xh: torch.Tensor, t: torch.Tensor,
                context: Optional[torch.Tensor] = None, num_mols: Optional[int] = None) -> torch.Tensor:
        if not xh.is_cuda:
            raise _lib.BdiffError("GCPNetDynamicsB200 runs on CUDA tensors only (no CPU fallback)")
        lib = _lib.load()
        self.sync_weights()
        _, n, _ = self.plan(batch_index, mask, num_mols)
        xh_c, t_c, ctx_c = self._inputs(n, xh, t, context)
        out = torch.empty_like(xh_c)
        _lib.check(self._handle, lib.bdiff_denoise_forward(
            self._handle, self._stream(), C.c_void_p(xh_c.data_ptr()), C.c_void_p(t_c.data_ptr()),
            C.c_void_p(ctx_c.data_ptr()) if ctx_c is not None else None, C.c_void_p(out.data_ptr())),
            "bdiff_denoise_forward")
        return out

    def wants_grad(self) -> bool:
        return torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())

    def forward(self, batch: Any, xh: torch.Tensor, t: torch.Tensor, **kwargs: Any):
        """Reference contract: gcpnet.py:1042-1052.  Reads batch.batch / batch.mask / batch.props_context.
        Under autograd with trainable parameters the result carries a grad_fn (training pass), else sampler kernels."""
        if kwargs.get("xh_self_cond") is not None or kwargs.get("x_self_cond") is not None:
            raise NotImplementedError("self-conditioning is not supported (shipped configs have self_condition=false)")
        ctx = getattr(batch, "props_context", None)
        num_mols = getattr(batch, "num_graphs", None)
        num_mols = num_mols if isinstance(num_mols, int) else None
        fn = self.denoise_train if self.wants_grad() else self.denoise
        return batch, fn(batch.batch, batch.mask, xh, t, ctx, num_mols)

    # ------------------------------------------------------------------------------------------ training pass
    def flatten_parameters(self) -> torch.Tensor:
        """Make every parameter a view of ONE flat fp32 CUDA buffer in the library's canonical layout
        (bdiff_param_layout), so the training pass reads the live weights with no per-step upload.  Idempotent; values
        are preserved.  Call it (or run one training forward) BEFORE handing the parameters to an optimiser that records
        their storage (GCDMTrainTail re-reads the pointers on its own)."""
        lib = _lib.load()
        h = self._ensure_handle()
        params = list(self.named_parameters())
        dev = params[0][1].device
        if dev.type != "cuda":
            raise _lib.BdiffError("GCPNetDynamicsB200 parameters must be on a CUDA device (no CPU fallback)")
        if self._layout is None:
            lay = {}
            for name, _ in params:
                off, cnt = C.c_int64(), C.c_int64()
                _lib.check(h, lib.bdiff_param_layout(h, name.encode(), C.byref(off), C.byref(cnt)), f"bdiff_param_layout({name})")
                lay[name] = (int(off.value), int(cnt.value))
            self._layout = lay
        total = int(lib.bdiff_param_floats(h))
        if self._flat is None or self._flat.device != dev:
            self._flat = torch.zeros(total, dtype=torch.float32, device=dev)
            self._grad_flat = torch.zeros(total, dtype=torch.float32, device=dev)
        base = self._flat.data_ptr()
        with torch.no_grad():
            for name, p in params:
                off, cnt = self._layout[name]
                if cnt != p.numel():
                    raise _lib.BdiffError(f"parameter {name}: {p.numel()} elements, the library expects {cnt}")
                if p.data_ptr() != base + 4 * off or p.dtype != torch.float32:
                    view = self._flat[off:off + cnt].view(p.shape)
                    view.copy_(p.detach())
                    p.data = view
        return self._flat

    def _inputs(self, n: int, xh, t, context):
        xh_c = xh.detach().to(torch.float32).contiguous()
        t_c = t.detach().to(torch.float32).reshape(-1).contiguous()
        if t_c.numel() == 1:
            t_c = t_c.expand(n).contiguous()
        if xh_c.shape != (n, 3 + self.cfg.num_h) or t_c.shape[0] != n:
            raise ValueError(f"xh must be [{n},{3 + self.cfg.num_h}] and t [{n},1]")
        ctx_c = None
        if self.cfg.num_context:
            if context is None:
                raise ValueError("this configuration is property-conditional: batch.props_context is required")
            ctx_c = context.detach().to(torch.float32).reshape(n, self.cfg.num_context).contiguous()
        return xh_c, t_c, ctx_c

    def _train_forward(self, batch_index, mask, xh, t, context, num_mols):
        if not xh.is_cuda:
            raise _lib.BdiffError("GCPNetDynamicsB200 runs on CUDA tensors only (no CPU fallback)")
        lib = _lib.load()
        flat = self.flatten_parameters()
        _, n, _ = self.plan(batch_index, mask, num_mols)
        xh_c, t_c, ctx_c = self._inputs(n, xh, t, context)
        out = torch.empty_like(xh_c)
        _lib.check(self._handle, lib.bdiff_train_forward(
            self._handle, self._stream(), C.c_void_p(flat.data_ptr()), C.c_void_p(xh_c.data_ptr()),
            C.c_void_p(t_c.data_ptr()), C.c_void_p(ctx_c.data_ptr()) if ctx_c is not None else None,
            C.c_void_p(out.data_ptr())), "bdiff_train_forward")
        self._tape_id += 1
        return out

    def _train_backward(self, d_out: torch.Tensor):
        lib = _lib.load()
        d = d_out.detach().to(torch.float32).contiguous()
        _lib.check(self._handle, lib.bdiff_train_backward(self._handle, self._stream(), C.c_void_p(d.data_ptr()),
                                                          C.c_void_p(self._grad_flat.data_ptr())), "bdiff_train_backward")
        g = self._grad_flat.clone()        # autograd may keep / accumulate into what we return; the flat buffer is reused
        out = []
        for name, p in self.named_parameters():
            off, cnt = self._layout[name]
            out.append(g[off:off + cnt].view(p.shape))
        return out

    def denoise_train(self, batch_index: torch.Tensor, mask: torch.Tensor, xh: torch.Tensor, t: torch.Tensor,
                      context: Optional[torch.Tensor] = None, num_mols: Optional[int] = None) -> torch.Tensor:
        """`denoise` with a grad_fn: fp32 training pass of the library (one tape at a time)."""
        return _DenoiseTrainFn.apply(self, batch_index, mask, xh, t, context, num_mols, *self.parameters())

    def set_train_precision(self, tf32: bool) -> None:
        """GEMMs of the training pass: fp32 (default) or TF32 tensor cores."""
        lib = _lib.load()
        _lib.check(self._ensure_handle(), lib.bdiff_train_precision(self._ensure_handle(), int(bool(tf32))), "bdiff_train_precision")

    def profile_forward(self, batch_index, mask, xh, t, context=None, num_mols=None):
        """One eager forward with CUDA events around every kernel class (inside the library, on the launch
        stream).  Returns ({class: milliseconds}, net_out).  Synchronises; for bench.py's roofline block."""
        lib = _lib.load()
        self.sync_weights()
        _, n, _ = self.plan(batch_index, mask, num_mols)
        xh_c, t_c, ctx_c = self._inputs(n, xh, t, context)
        out = torch.empty_like(xh_c)
        ms = (C.c_float * 8)()
        _lib.check(self._handle, lib.bdiff_profile_forward(
            self._handle, self._stream(), C.c_void_p(xh_c.data_ptr()), C.c_void_p(t_c.data_ptr()),
            C.c_void_p(ctx_c.data_ptr()) if ctx_c is not None else None, C.c_void_p(out.data_ptr()), ms),
            "bdiff_profile_forward")
        names = ("prep", "edge_embed", "node_embed", "edge_message", "node_update", "finalize", "total")
        prof = {k: float(ms[i]) for i, k in enumerate(names)}
        if ms[7] < 0:       # tensor mode default: all layers ran as ONE persistent kernel (k_layers_tc)
            prof["layers_fused"] = prof.pop("edge_message")
            prof.pop("node_update")
        return prof, out

    @property
    def kernels_per_forward(self) -> int:
        """libbdiff kernels in one denoiser forward: prep, node_frames, edge_embed, node_embed, finalize plus either
        one persistent k_layers_tc (tensor mode) or 2 per layer (parity mode)."""
        return 5 + (1 if self.mode == "tensor" else 2 * self.cfg.num_layers)

    def launch_count(self) -> int:
        return int(_lib.load().bdiff_launch_count(self._handle)) if self._handle is not None else 0

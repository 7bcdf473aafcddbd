"""PropertyClassifier — drop-in for EDM's EGNN property classifier (reference: src/__init__.py:233-419, EGNN / E_GCL_mask),
the network `get_classifier` (:97-114) loads to score the QM9 property-conditional evaluation and the property-optimisation
workload (mol_gen_eval_conditional_qm9.py:299-315, mol_gen_eval_optimization_qm9.py).

Same parameter names and shapes as the reference, so EDM's `best_checkpoint.npy` loads with strict=True, and the same
dense call `forward(h0, x, edges, edge_attr, node_mask, edge_mask, n_nodes)`, so `test_with_property_classifier` runs
unchanged.  Every arithmetic step runs in libbdiff_sm90.so (`bdiff_classifier_forward`) on packed molecules; `predict`
takes the sampler's packed output directly.  There is no CPU / PyTorch fallback.

Under autograd (`torch.is_grad_enabled()` and some parameter requires grad — the train branch of
`train_with_property_classifier`, :144-204) `forward` and `predict` run the library's training pass instead:
`bdiff_classifier_train_forward` keeps a tape, `loss.backward()` reaches `bdiff_classifier_train_backward` through a
`torch.autograd.Function` and every parameter receives its gradient (x and h0 are data: they get none).  A torch optimiser
steps the parameters in place; the next call repacks them (`sync_weights`).
"""
from __future__ import annotations

import ctypes as C
import math
import os
import pickle
from typing import Optional

import torch
from torch import nn

from . import _lib
from .dynamics import _register, _version

IN_NODE_NF = 5
HIDDEN_NF = 128
MAX_ATOMS = 128


def classifier_parameter_shapes(n_layers: int, attention: bool, node_attr: bool, hidden_nf: int = HIDDEN_NF) -> dict:
    """Reference state-dict names and shapes of EGNN(in_node_nf=5, in_edge_nf=0, hidden_nf, n_layers, attention,
    node_attr) (src/__init__.py:385-403; E_GCL_mask deletes coord_mlp)."""
    h = hidden_nf
    out = {"embedding.weight": (h, IN_NODE_NF), "embedding.bias": (h,)}
    for i in range(n_layers):
        p = f"gcl_{i}."
        out[p + "edge_mlp.0.weight"] = (h, 2 * h + 1)
        out[p + "edge_mlp.0.bias"] = (h,)
        out[p + "edge_mlp.2.weight"] = (h, h)
        out[p + "edge_mlp.2.bias"] = (h,)
        out[p + "node_mlp.0.weight"] = (h, 2 * h + (IN_NODE_NF if node_attr else 0))
        out[p + "node_mlp.0.bias"] = (h,)
        out[p + "node_mlp.2.weight"] = (h, h)
        out[p + "node_mlp.2.bias"] = (h,)
        if attention:
            out[p + "att_mlp.0.weight"] = (1, h)
            out[p + "att_mlp.0.bias"] = (1,)
    out.update({"node_dec.0.weight": (h, h), "node_dec.0.bias": (h,), "node_dec.2.weight": (h, h), "node_dec.2.bias": (h,),
                "graph_dec.0.weight": (h, h), "graph_dec.0.bias": (h,), "graph_dec.2.weight": (1, h),
                "graph_dec.2.bias": (1,)})
    return out


def predict_inputs(x: torch.Tensor, one_hot: torch.Tensor, num_nodes) -> torch.Tensor:
    """Validates the packed batch of `PropertyClassifier.predict` on the host; returns num_nodes as int64 [B] on the CPU."""
    nn_ = torch.as_tensor(num_nodes).reshape(-1).to("cpu", torch.int64)
    n = int(x.shape[0])
    if x.dim() != 2 or x.shape[1] != 3:
        raise ValueError(f"x must be [N, 3], got {tuple(x.shape)}")
    if one_hot.dim() != 2 or one_hot.shape != (n, IN_NODE_NF):
        raise ValueError(f"one_hot must be [N, {IN_NODE_NF}] = [{n}, {IN_NODE_NF}], got {tuple(one_hot.shape)}")
    if nn_.numel() < 1 or int(nn_.sum()) != n or bool((nn_ < 1).any()):
        raise ValueError("num_nodes must be positive and sum to the number of atoms")
    if int(nn_.max()) > MAX_ATOMS:
        raise ValueError(f"a molecule has {int(nn_.max())} atoms: the classifier takes at most {MAX_ATOMS}")
    return nn_


class _ClassifierTrainFn(torch.autograd.Function):
    """pred = classifier(params; x, one_hot) with the library's tape; backward = bdiff_classifier_train_backward."""

    @staticmethod
    def forward(ctx, clf, x, one_hot, off, *params):
        pred = clf._run(x, one_hot, off, train=True)
        ctx.clf = clf
        ctx.tape_id = clf._tape_id
        ctx.needs = tuple(p.requires_grad for p in params)
        return pred

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_pred):
        clf = ctx.clf
        if ctx.tape_id != clf._tape_id:
            raise _lib.BdiffError("PropertyClassifier keeps ONE training tape: a later forward under autograd replaced the "
                                  "one this backward needs (call backward() before the next training forward)")
        grads = clf._train_backward(d_pred)
        return (None,) * 4 + tuple(g if need else None for g, need in zip(grads, ctx.needs))


class PropertyClassifier(nn.Module):
    """EGNN(in_node_nf, in_edge_nf, hidden_nf, device, act_fn, n_layers, coords_weight, attention, node_attr) with the
    reference's constructor arguments; only in_node_nf = 5, in_edge_nf = 0, hidden_nf = 128 and SiLU are supported."""

    def __init__(self, in_node_nf: int = IN_NODE_NF, in_edge_nf: int = 0, hidden_nf: int = HIDDEN_NF, device="cpu",
                 act_fn: Optional[nn.Module] = None, n_layers: int = 7, coords_weight: float = 1.0,
                 attention: bool = True, node_attr: int = 0):
        super().__init__()
        if in_node_nf != IN_NODE_NF:
            raise NotImplementedError(f"in_node_nf must be {IN_NODE_NF} (the QM9 one-hot), got {in_node_nf}")
        if in_edge_nf != 0:
            raise NotImplementedError("edge attributes are not supported (in_edge_nf must be 0)")
        if hidden_nf != HIDDEN_NF:
            raise NotImplementedError(f"hidden_nf must be {HIDDEN_NF}, got {hidden_nf}")
        if act_fn is not None and not isinstance(act_fn, nn.SiLU):
            raise NotImplementedError("only the SiLU activation (the reference default) is supported")
        if not 1 <= int(n_layers) <= 64:
            raise NotImplementedError("n_layers must be in [1, 64]")
        self.hidden_nf = hidden_nf
        self.n_layers = int(n_layers)
        self.attention = bool(attention)
        self.node_attr = int(bool(node_attr))
        self._shapes = classifier_parameter_shapes(self.n_layers, self.attention, bool(self.node_attr))
        for name, shape in self._shapes.items():
            _register(self, name, nn.Parameter(torch.empty(shape)))
        self.reset_parameters()
        self._handle = None
        self._weights_key = None
        self._layout = None          # training: name -> (offset, count) in the flat gradient buffer
        self._grad_flat = None
        self._tape_id = 0
        self.to(device)

    @classmethod
    def from_dir(cls, model_dir: str, device="cpu") -> "PropertyClassifier":
        """Mirror of get_classifier (src/__init__.py:97-114): `args.pickle` (nf, n_layers, attention, node_attr) and the
        state dict in `best_checkpoint.npy`."""
        with open(os.path.join(model_dir, "args.pickle"), "rb") as f:
            args = pickle.load(f)
        clf = cls(in_node_nf=IN_NODE_NF, in_edge_nf=0, hidden_nf=args.nf, n_layers=args.n_layers,
                  attention=args.attention, node_attr=args.node_attr)
        sd = torch.load(os.path.join(model_dir, "best_checkpoint.npy"), map_location="cpu")
        clf.load_state_dict(sd, strict=True)
        return clf.to(device)

    def reset_parameters(self) -> None:
        """nn.Linear's default init range (uniform, bound 1/sqrt(fan_in)) for every weight / bias pair."""
        with torch.no_grad():
            for name, p in self.named_parameters():
                fan_in = p.shape[1] if name.endswith("weight") else self._shapes[name[:-4] + "weight"][1]
                bound = 1.0 / math.sqrt(fan_in)
                p.uniform_(-bound, bound)

    # ------------------------------------------------------------------------------------------ C-ABI handle
    def _ensure_handle(self):
        if self._handle is not None:
            return self._handle
        lib = _lib.load()
        cfg = _lib.ClassifierConfig(in_node_nf=IN_NODE_NF, in_edge_nf=0, hidden_nf=self.hidden_nf, n_layers=self.n_layers,
                                    attention=int(self.attention), node_attr=self.node_attr)
        h = C.c_void_p()
        rc = lib.bdiff_classifier_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise _lib.BdiffError(f"bdiff_classifier_create failed (code {rc}): "
                                  f"{lib.bdiff_classifier_last_error(None).decode()}")
        self._handle = h
        return h

    def __del__(self):
        try:
            if getattr(self, "_handle", None) is not None:
                _lib.load().bdiff_classifier_destroy(self._handle)
                self._handle = None
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            msg = _lib.load().bdiff_classifier_last_error(self._handle)
            raise _lib.BdiffError(f"{what} failed (code {rc}): {msg.decode() if msg else '?'}")

    def sync_weights(self, force: bool = False) -> None:
        """Repack the parameters into the kernel layout when one of them changed (storage or version counter)."""
        key = tuple((p.data_ptr(), _version(p)) for p in self.parameters())
        if not force and key == self._weights_key:
            return
        lib = _lib.load()
        h = self._ensure_handle()
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        for name, p in self.named_parameters():
            if not p.is_cuda:
                raise _lib.BdiffError("PropertyClassifier parameters must be on a CUDA device (no CPU fallback)")
            t = p.detach().to(torch.float32).contiguous()
            shape = (C.c_int64 * t.dim())(*t.shape)
            self._check(lib.bdiff_classifier_set_weight(h, st, name.encode(), C.c_void_p(t.data_ptr()), shape, t.dim()),
                        f"bdiff_classifier_set_weight({name})")
        self._weights_key = key

    # ------------------------------------------------------------------------------------------ forward
    def wants_grad(self) -> bool:
        return torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters())

    def predict(self, x: torch.Tensor, one_hot: torch.Tensor, num_nodes: torch.Tensor) -> torch.Tensor:
        """pred [B] (normalised property) of packed molecules: x [N, 3], one_hot [N, 5] (the sampler's out[:, :3] and
        out[:, 3:8]), num_nodes [B] with 1 <= n <= 128 summing to N.  Under autograd with trainable parameters the
        result carries a grad_fn (the training pass; its values are bit-identical to the inference kernels')."""
        nn_ = predict_inputs(x, one_hot, num_nodes)
        if not x.is_cuda:
            raise _lib.BdiffError("PropertyClassifier runs on CUDA tensors only (no CPU fallback)")
        off = torch.zeros(int(nn_.numel()) + 1, dtype=torch.int32)
        off[1:] = torch.cumsum(nn_, 0).to(torch.int32)
        if self.wants_grad():
            return _ClassifierTrainFn.apply(self, x, one_hot, off, *self.parameters())
        return self._run(x, one_hot, off, train=False)

    def _run(self, x, one_hot, off, train: bool) -> torch.Tensor:
        """bdiff_classifier_forward (train = False) or bdiff_classifier_train_forward (keeps the tape)."""
        self.sync_weights()
        lib = _lib.load()
        b = int(off.numel()) - 1
        xc = x.detach().to(torch.float32).contiguous()
        oh = one_hot.detach().to(device=xc.device, dtype=torch.float32).contiguous()
        pred = torch.empty(b, dtype=torch.float32, device=xc.device)
        fn, what = ((lib.bdiff_classifier_train_forward, "bdiff_classifier_train_forward") if train
                    else (lib.bdiff_classifier_forward, "bdiff_classifier_forward"))
        self._check(fn(self._handle, C.c_void_p(torch.cuda.current_stream(xc.device).cuda_stream), b,
                       off.numpy().ctypes.data_as(C.POINTER(C.c_int32)), C.c_void_p(xc.data_ptr()),
                       C.c_void_p(oh.data_ptr()), C.c_void_p(pred.data_ptr())), what)
        if train:
            self._tape_id += 1
        return pred

    def param_layout(self) -> dict:
        """name -> (offset, count) of every parameter in the library's flat gradient buffer (bdiff_classifier_param_layout)."""
        if self._layout is None:
            lib = _lib.load()
            h = self._ensure_handle()
            lay = {}
            for name, _ in self.named_parameters():
                off, cnt = C.c_int64(), C.c_int64()
                self._check(lib.bdiff_classifier_param_layout(h, name.encode(), C.byref(off), C.byref(cnt)),
                            f"bdiff_classifier_param_layout({name})")
                lay[name] = (int(off.value), int(cnt.value))
            self._layout = lay
        return self._layout

    def _train_backward(self, d_pred: torch.Tensor):
        lib = _lib.load()
        lay = self.param_layout()
        d = d_pred.detach().to(torch.float32).contiguous()
        if self._grad_flat is None or self._grad_flat.device != d.device:
            self._grad_flat = torch.empty(int(lib.bdiff_classifier_param_floats(self._handle)), dtype=torch.float32,
                                          device=d.device)
        self._check(lib.bdiff_classifier_train_backward(
            self._handle, C.c_void_p(torch.cuda.current_stream(d.device).cuda_stream), C.c_void_p(d.data_ptr()),
            C.c_void_p(self._grad_flat.data_ptr())), "bdiff_classifier_train_backward")
        g = self._grad_flat.clone()        # autograd may keep / accumulate into what we return; the flat buffer is reused
        out = []
        for name, p in self.named_parameters():
            off, cnt = lay[name]
            out.append(g[off:off + cnt].view(p.shape).to(p.dtype))
        return out

    def forward(self, h0: torch.Tensor, x: torch.Tensor, edges=None, edge_attr=None, node_mask: torch.Tensor = None,
                edge_mask: torch.Tensor = None, n_nodes: int = None) -> torch.Tensor:
        """The reference's dense call (EGNN.forward, src/__init__.py:405-419): h0 [B*n, 5], x [B*n, 3], node_mask
        [B*n, 1], edge_mask [B*n*n, 1] = node-mask outer product without the diagonal (the construction of both evaluation
        scripts); `edges` is not read.  Packs the real atoms on the device and runs the same kernels as `predict`."""
        if edge_attr is not None:
            raise NotImplementedError("edge attributes are not supported")
        n_nodes = int(n_nodes)
        nt = int(h0.shape[0])
        if n_nodes < 1 or nt % n_nodes:
            raise ValueError("h0 must hold B * n_nodes rows")
        b = nt // n_nodes
        mask = node_mask.reshape(b, n_nodes) != 0
        if mask.shape[0] * n_nodes * n_nodes != edge_mask.numel():
            raise ValueError("edge_mask must hold B * n_nodes^2 entries")
        expect = mask.unsqueeze(1) & mask.unsqueeze(2)
        expect &= ~torch.eye(n_nodes, dtype=torch.bool, device=mask.device).unsqueeze(0)
        if not torch.equal(edge_mask.reshape(b, n_nodes, n_nodes) != 0, expect):
            raise ValueError("edge_mask must be the node-mask outer product with the diagonal removed (the construction "
                             "of the reference's evaluation scripts); other masks are not supported")
        m = mask.reshape(-1)
        num_nodes = mask.sum(1)
        if bool((num_nodes < 1).any()):
            raise ValueError("every molecule of the batch needs at least one atom")
        return self.predict(x.reshape(nt, 3)[m], h0.reshape(nt, -1)[m], num_nodes)

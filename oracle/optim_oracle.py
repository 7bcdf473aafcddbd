"""CPU restatement of the optimiser side of a GCDM training step (SURVEY.md §8 a21).  TEST INFRASTRUCTURE ONLY.

Follows, in order:
  * `get_grad_norm`                      /root/reference/src/models/__init__.py:90-113
  * `Queue` (history of norms)           /root/reference/src/models/__init__.py:442-466, seeded with 3000
                                         (qm9_mol_gen_ddpm.py:148-149)
  * `configure_gradient_clipping`        /root/reference/src/models/qm9_mol_gen_ddpm.py:1267-1304 (limit = 1.5 mean + 2 std,
                                         Lightning's clip_gradients(..., "norm") = torch.nn.utils.clip_grad_norm_)
  * AdamW(lr 1e-4, weight_decay 1e-12, amsgrad)   configs/model/qm9_mol_gen_ddpm.yaml:3-8; arithmetic of torch 1.12
                                         torch/optim/adamw.py::_single_tensor_adamw (third-party, pinned by
                                         tests/test_optim_oracle.py against torch.optim.AdamW of this image)
  * EMA (decay 0.9999, every step)       /root/reference/src/utils/__init__.py:133-142 (the non-apex arithmetic)
Pinned against torch.optim.AdamW + torch.nn.utils.clip_grad_norm_ + the reference's own Queue / EMA classes in
tests/test_optim_oracle.py (the latter two through oracle/ref_shim.py in the build container; the committed golden
fixture tests/golden/optim_steps.pt carries their outputs to the GPU box).
"""
import math

import numpy as np
import torch


class NormQueue:
    """src/models/__init__.py:442-466 (insert at the front, drop the oldest beyond max_len)."""

    def __init__(self, max_len=50, seed_value=3000.0):
        self.items = [float(seed_value)]
        self.max_len = max_len

    def add(self, item):
        self.items.insert(0, float(item))
        if len(self.items) > self.max_len:
            self.items.pop()

    def limit(self):
        return 1.5 * float(np.mean(self.items)) + 2.0 * float(np.std(self.items))


class TrainTailOracle:
    def __init__(self, params, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-12, amsgrad=True,
                 ema_decay=0.9999, clip=True, queue_len=50):
        self.p = [p.detach().clone().float() for p in params]
        self.m = [torch.zeros_like(p) for p in self.p]
        self.v = [torch.zeros_like(p) for p in self.p]
        self.vmax = [torch.zeros_like(p) for p in self.p]
        self.ema = [p.clone() for p in self.p]
        self.lr, self.b1, self.b2, self.eps, self.wd = lr, betas[0], betas[1], eps, weight_decay
        self.amsgrad, self.ema_decay, self.clip = amsgrad, ema_decay, clip
        self.queue = NormQueue(queue_len)
        self.step_count = 0
        self.last = {}

    def step(self, grads):
        grads = [g.detach().float() for g in grads]
        norm = float(torch.norm(torch.stack([torch.norm(g, 2.0) for g in grads]), 2.0))      # get_grad_norm
        coef, limit = 1.0, 0.0
        if self.clip:
            limit = self.queue.limit()
            coef = min(limit / (norm + 1e-6), 1.0)                                          # clip_grad_norm_
            self.queue.add(limit if norm > limit else norm)
        self.step_count += 1
        t = self.step_count
        bc1 = 1.0 - self.b1 ** t
        bc2 = 1.0 - self.b2 ** t
        for i, g in enumerate(grads):
            g = g * np.float32(coef)
            self.p[i].mul_(1.0 - self.lr * self.wd)
            self.m[i].mul_(self.b1).add_(g, alpha=1.0 - self.b1)
            self.v[i].mul_(self.b2).addcmul_(g, g, value=1.0 - self.b2)
            if self.amsgrad:
                torch.maximum(self.vmax[i], self.v[i], out=self.vmax[i])
                denom = (self.vmax[i].sqrt() / math.sqrt(bc2)).add_(self.eps)
            else:
                denom = (self.v[i].sqrt() / math.sqrt(bc2)).add_(self.eps)
            self.p[i].addcdiv_(self.m[i], denom, value=-self.lr / bc1)
            diff = self.ema[i] - self.p[i]                                                  # apply_ema
            diff.mul_(1.0 - self.ema_decay)
            self.ema[i].sub_(diff)
        self.last = {"norm": norm, "limit": limit, "coef": coef}
        return self.last


# ------------------------------------------------------------------ gradients of tests/golden/optim_long.pt
# (drawn from numpy's PCG64 generator, the same numbers on every machine, so the fixture need not store them)
LONG_SIZES = [1, 3, 16384, 16385, 32773]
LONG_RUNS = [  # queue_len, amsgrad, steps, {step: gradient scale} of the spikes (every other step: scale 0.5 .. 2)
    (1, True, 14, {5: 4.0, 9: 60.0}),
    (3, False, 16, {7: 3.0, 11: 80.0}),
    (50, True, 64, {53: 3.0, 58: 200.0}),
    (120, True, 134, {123: 3.0, 127: 50.0, 130: 1.0}),
]


def long_run_grads(queue_len, steps, spikes):
    """Initial parameters, then for every step the gradient of every tensor (float32, seeded by queue_len)."""
    rng = np.random.default_rng(4000 + queue_len)
    init = [torch.from_numpy(rng.standard_normal(n, dtype=np.float32) * np.float32(0.1)) for n in LONG_SIZES]
    grads = []
    for k in range(steps):
        sc = np.float32(spikes.get(k, 0.5 + 1.5 * rng.random()))
        grads.append([torch.from_numpy(rng.standard_normal(n, dtype=np.float32) * sc) for n in LONG_SIZES])
    return init, grads


def fingerprint_index(n, chunk=16384):
    """Entries of an n-element tensor that optim_long.pt stores: both ends, +-4 around every chunk border, every 97th."""
    idx = set(range(min(n, 8))) | set(range(max(0, n - 8), n)) | set(range(0, n, 97))
    for b in range(chunk, n, chunk):
        idx |= set(range(b - 4, min(n, b + 4)))
    return torch.tensor(sorted(idx), dtype=torch.int64)

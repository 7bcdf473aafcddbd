#!/usr/bin/env python
"""Golden fixture for the optimiser tail (SURVEY.md §8 a21), generated with the REFERENCE's own pieces in the build
container: `Queue` and `get_grad_norm` imported unmodified from /root/reference/src/models/__init__.py (through
oracle/ref_shim.py), torch.optim.AdamW(lr 1e-4, weight_decay 1e-12, amsgrad=True) and
torch.nn.utils.clip_grad_norm_ (what Lightning's clip_gradients(..., "norm") calls), and the EMA arithmetic of
src/utils/__init__.py:133-142.  Run:  python tests/golden/make_golden_optim.py

optim_steps.pt: 8 steps, queue_len 50, two gradient spikes.
optim_long.pt: queue_len 1, 3, 50 and 120, each run for more than queue_len + 10 steps, with gradient spikes after the
history window has filled (the seeded 3000 has been evicted), tensors of 1, 3, 16384, 16385 and 32773 elements (one chunk
of the kernels is 16384 elements), one run with amsgrad=False.  Its gradients are not stored: `long_run_grads`
(oracle/optim_oracle.py) draws them from numpy's PCG64 generator, which gives the same numbers on every machine, and the
test draws them again.  The final state is stored as fingerprints (norm, sum and the entries at `fingerprint_index`:
chunk borders, tensor ends and a stride) so that the fixture stays small."""
import os
import sys

import torch
import torch._dynamo  # noqa: F401  (torch.optim imports it lazily; must happen before the stub modules are installed)

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_shim  # noqa: E402

ref_shim.install()      # stub modules + /root/reference on sys.path
from src.models import Queue, get_grad_norm  # noqa: E402
from optim_oracle import LONG_RUNS, LONG_SIZES, fingerprint_index, long_run_grads  # noqa: E402


def fingerprint(t):
    t = t.detach().reshape(-1)
    return {"norm": float(t.double().norm()), "sum": float(t.double().sum()), "vals": t[fingerprint_index(t.numel())].clone()}


def long_run(queue_len, amsgrad, steps, spikes):
    init, grads = long_run_grads(queue_len, steps, spikes)
    params = [torch.nn.Parameter(p.clone()) for p in init]
    opt = torch.optim.AdamW(params, lr=1e-4, weight_decay=1e-12, amsgrad=amsgrad)
    queue = Queue(max_len=queue_len)
    queue.add(3000)
    ema = [p.detach().clone() for p in params]
    log = []
    for gs in grads:
        for p, g in zip(params, gs):
            p.grad = g.clone()
        limit = 1.5 * queue.mean() + 2 * queue.std()
        norm = get_grad_norm(params)
        torch.nn.utils.clip_grad_norm_(params, max_norm=float(limit), norm_type=2.0)
        queue.add(float(limit) if float(norm) > limit else float(norm))
        opt.step()
        for w, e in zip(params, ema):
            diff = e.data - w.data
            diff.mul_(1.0 - 0.9999)
            e.sub_(diff)
        log.append({"norm": float(norm), "limit": float(limit), "clipped": bool(float(norm) > limit)})
    return {"queue_len": queue_len, "amsgrad": amsgrad, "steps": steps, "spikes": spikes, "log": log,
            "params": [fingerprint(p) for p in params], "ema": [fingerprint(e) for e in ema],
            "max_exp_avg_sq": [fingerprint(opt.state[p]["max_exp_avg_sq"]) for p in params] if amsgrad else None,
            "history": sorted(float(x) for x in queue.items)}


torch.manual_seed(11)
shapes = [(64, 77), (64,), (32, 8), (1, 64), (17,), (20000,)]
params = [torch.nn.Parameter(torch.randn(s) * 0.1) for s in shapes]
init = [p.detach().clone() for p in params]
opt = torch.optim.AdamW(params, lr=1e-4, weight_decay=1e-12, amsgrad=True)
queue = Queue()
queue.add(3000)
ema = [p.detach().clone() for p in params]
decay = 0.9999
steps, log = [], []
scales = [1.0, 0.5, 2.0, 4000.0, 1.0, 300.0, 1.0, 1.0]          # two spikes exercise the clipping branch
for k, sc in enumerate(scales):
    grads = [torch.randn(s) * sc for s in shapes]
    for p, g in zip(params, grads):
        p.grad = g.clone()
    limit = 1.5 * queue.mean() + 2 * queue.std()
    norm = get_grad_norm(params)
    torch.nn.utils.clip_grad_norm_(params, max_norm=float(limit), norm_type=2.0)
    queue.add(float(limit) if float(norm) > limit else float(norm))
    opt.step()
    for w, e in zip(params, ema):
        diff = e.data - w.data
        diff.mul_(1.0 - decay)
        e.sub_(diff)
    steps.append(grads)
    log.append({"norm": float(norm), "limit": float(limit), "clipped": bool(float(norm) > limit)})
out = {"shapes": shapes, "init": init, "grads": steps, "log": log,
       "params": [p.detach().clone() for p in params], "ema": ema,
       "exp_avg": [opt.state[p]["exp_avg"].clone() for p in params],
       "max_exp_avg_sq": [opt.state[p]["max_exp_avg_sq"].clone() for p in params],
       "history": sorted(float(x) for x in queue.items)}
torch.save(out, os.path.join(os.path.dirname(os.path.abspath(__file__)), "optim_steps.pt"))
print("wrote optim_steps.pt;", [(round(l["norm"], 2), round(l["limit"], 2), l["clipped"]) for l in log])

runs = [long_run(*r) for r in LONG_RUNS]
torch.save({"sizes": LONG_SIZES, "runs": runs}, os.path.join(os.path.dirname(os.path.abspath(__file__)), "optim_long.pt"))
for r in runs:
    clipped = [k for k, l in enumerate(r["log"]) if l["clipped"]]
    print(f"wrote optim_long.pt run queue_len={r['queue_len']} amsgrad={r['amsgrad']}: clipped at steps {clipped}")

#!/usr/bin/env python
"""Times one training step of the EGNN property classifier (bdiff.PropertyClassifier, 7 layers, attention) at QM9 batch
size 128, molecule sizes drawn from the QM9 histogram: the train branch of train_with_property_classifier
(src/__init__.py:160-190) — zero_grad, the dense call, L1 loss, backward, torch.optim.Adam.step — against the same step
through the oracle's dense torch autograd path (the reference's un-fused arithmetic over all B * n_max^2 pairs) on the
same GPU.  The first step's gradients of both paths are compared.  CUDA-event timings, warm-up, median of >= 20 steps.
Prints the card's name and power limit and one JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "bio-diffusion_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402
import bdiff  # noqa: E402
import classifier_oracle as CO  # noqa: E402


def median_ms(fn, runs, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--runs", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_classifier_train needs a CUDA device")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)
    print(f"device: {card}")

    sd = CO.random_state_dict(1)
    clf = bdiff.PropertyClassifier(n_layers=7, attention=1, node_attr=0)
    clf.load_state_dict(sd, strict=True)
    clf.to(dev)
    sizes = bdiff.sample_num_nodes(bdiff.QM9_N_NODES, args.batch, seed=0)
    g = torch.Generator().manual_seed(1)
    n = int(sizes.sum())
    x = (torch.randn((n, 3), generator=g) * 1.5).to(dev)
    oh = torch.nn.functional.one_hot(torch.randint(0, 5, (n,), generator=g), 5).float().to(dev)
    label = torch.randn(args.batch, generator=g).to(dev)
    d = CO.dense_batch(x, oh, sizes)
    bs, nmax, _ = d["positions"].shape
    h0, xd = d["one_hot"].view(bs * nmax, -1), d["positions"].view(bs * nmax, -1)
    nm, em = d["atom_mask"].view(bs * nmax, 1).float(), d["edge_mask"].float()
    base = {k: v.to(dev).requires_grad_(True) for k, v in sd.items()}
    l1 = torch.nn.L1Loss()

    def lib_loss():
        return l1(clf(h0=h0, x=xd, edges=None, edge_attr=None, node_mask=nm, edge_mask=em, n_nodes=nmax), label)

    def base_loss():
        return l1(CO.dense_forward(base, 7, True, False, h0, xd, nm, em, nmax), label)

    lib_loss().backward()
    base_loss().backward()
    worst = max((p.grad - base[k].grad).abs().max().item() / max(base[k].grad.norm().item(), 1e-12)
                for k, p in clf.named_parameters())
    opt_lib = torch.optim.Adam(clf.parameters(), lr=1e-4)
    opt_base = torch.optim.Adam(list(base.values()), lr=1e-4)

    def step(opt, fn):
        def run():
            opt.zero_grad()
            fn().backward()
            opt.step()
        return run

    ms_lib = median_ms(step(opt_lib, lib_loss), args.runs)
    ms_base = median_ms(step(opt_base, base_loss), args.runs)
    res = {"workload": "classifier_train_step", "device": card, "batch": args.batch, "atoms": n, "n_max": nmax,
           "pairs_packed": int((sizes ** 2).sum()), "pairs_dense": bs * nmax * nmax,
           "ms_step_library": round(ms_lib, 3), "ms_step_torch_dense": round(ms_base, 3),
           "speedup": round(ms_base / ms_lib, 2), "worst_grad_diff_vs_torch_fp32": worst}
    print(json.dumps(res))


if __name__ == "__main__":
    main()

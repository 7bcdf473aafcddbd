#!/usr/bin/env python
"""Times the EGNN property classifier (bdiff.PropertyClassifier) at QM9 batch size 128, molecule sizes drawn from the QM9
histogram: the dense drop-in call (what test_with_property_classifier makes), packed `predict`, and the oracle's dense
torch path on the same GPU (the reference's un-fused arithmetic: all B * n_max^2 pairs, ~20 ops per layer).  Outputs are
compared.  Then one property-optimisation iteration (mol_gen_eval_optimization_qm9.py:133-241: `optimize` with 10 steps,
then a classifier pass over every molecule) with the classifier's share of it.  CUDA-event timings, warm-up, median of
>= 20 runs.  Prints the card's name and power limit and one JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "bio-diffusion_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402
import bdiff  # noqa: E402
import classifier_oracle as CO  # noqa: E402
import gcpnet_oracle as O  # noqa: E402


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
    ap.add_argument("--opt-runs", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_classifier needs a CUDA device")
    dev = torch.device("cuda:0")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)
    print(f"device: {card}")

    sd = CO.random_state_dict(1)
    clf = bdiff.PropertyClassifier(n_layers=7, attention=1, node_attr=0)
    clf.load_state_dict(sd, strict=True)
    clf.to(dev).requires_grad_(False)
    sizes = bdiff.sample_num_nodes(bdiff.QM9_N_NODES, args.batch, seed=0)
    g = torch.Generator().manual_seed(1)
    n = int(sizes.sum())
    x = (torch.randn((n, 3), generator=g) * 1.5).to(dev)
    oh = torch.nn.functional.one_hot(torch.randint(0, 5, (n,), generator=g), 5).float().to(dev)
    d = CO.dense_batch(x, oh, sizes)
    bs, nmax, _ = d["positions"].shape
    h0, xd = d["one_hot"].view(bs * nmax, -1), d["positions"].view(bs * nmax, -1)
    nm, em = d["atom_mask"].view(bs * nmax, 1).float(), d["edge_mask"].float()
    sd_dev = {k: v.to(dev) for k, v in sd.items()}

    with torch.no_grad():
        packed = clf.predict(x, oh, sizes)
        dense = clf(h0=h0, x=xd, edges=None, edge_attr=None, node_mask=nm, edge_mask=em, n_nodes=nmax)
        base = CO.dense_forward(sd_dev, 7, True, False, h0, xd, nm, em, nmax)
        ref64 = CO.packed_forward({k: v.double() for k, v in sd.items()}, 7, True, False, x.double().cpu(),
                                  oh.double().cpu(), sizes)
        ms_packed = median_ms(lambda: clf.predict(x, oh, sizes), args.runs)
        ms_dense = median_ms(lambda: clf(h0=h0, x=xd, edges=None, edge_attr=None, node_mask=nm, edge_mask=em,
                                         n_nodes=nmax), args.runs)
        ms_base = median_ms(lambda: CO.dense_forward(sd_dev, 7, True, False, h0, xd, nm, em, nmax), args.runs)

    # one optimisation iteration: optimize(10 steps) + scoring, on a qm9_cond denoiser
    ocfg = O.config_named("qm9_cond")
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named("qm9_cond"), mode="tensor")
    net.load_state_dict(O.random_state_dict(ocfg, 7, scale=0.5), strict=True)
    net.cuda()
    sampler = bdiff.GCDMSampler(net)
    ctx = torch.randn((args.batch, 1), generator=g).to(dev)
    torch.manual_seed(0)
    out, _, _ = sampler.sample(sizes, ctx, num_timesteps=10)
    samples, o = [], 0
    for k in sizes.tolist():
        samples.append((out[o:o + k, :3], out[o:o + k, 3:8]))
        o += k
    state = {}

    def optimize():
        state["out"], _, _ = sampler.optimize(samples, sizes, ctx, num_timesteps=10)

    def score():
        with torch.no_grad():
            state["pred"] = clf.predict(state["out"][:, :3], state["out"][:, 3:8], sizes)

    ms_opt = median_ms(optimize, args.opt_runs)
    ms_score = median_ms(score, args.opt_runs)
    res = {
        "device": card, "batch": args.batch, "atoms": n, "pairs": int((sizes * sizes).sum()), "n_max": nmax,
        "dense_pairs": bs * nmax * nmax,
        "ms_packed_predict": ms_packed, "ms_dense_dropin": ms_dense, "ms_oracle_dense_torch": ms_base,
        "speedup_vs_oracle_dense": ms_base / ms_packed,
        "max_abs_diff_packed_vs_fp64": (packed.double().cpu() - ref64).abs().max().item(),
        "max_abs_diff_oracle_fp32_vs_fp64": (base.double().cpu() - ref64).abs().max().item(),
        "dense_equals_packed": bool(torch.equal(dense, packed)),
        "ms_optimize_10_steps": ms_opt, "ms_classifier_scoring": ms_score,
        "classifier_share_of_iteration": ms_score / (ms_opt + ms_score),
    }
    print(json.dumps(res))


if __name__ == "__main__":
    main()

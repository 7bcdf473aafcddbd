#!/usr/bin/env python
"""Times GCDMSampler.inpaint (torch's generator draws the noise: four randn launches per denoise op, two per jump) against
GCDMSampler.inpaint(seed=...) (bdiff_inpaint: the noise is computed inside the kernels) on the bench workload: QM9,
128 molecules x 19 atoms, the first 5 atoms of every molecule fixed, T = 1000, tensor mode, at r = j = 1 and r = j = 10.
The arms alternate within every round; the best and the median round are reported.  Prints one JSON line with the GPU's
name, power limit and SM clock.

  python tools/bench_native_inpaint.py [--rounds 3] [--rj 1,10] [--timesteps 1000] [--batch 128] [--atoms 19]
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bio-diffusion_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import torch  # noqa: E402
import bdiff  # noqa: E402
import gcpnet_oracle as O  # noqa: E402
from bench import gpu_info  # noqa: E402
from bench_native_sample import sm_clock_mhz  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--rj", default="1,10", help="comma-separated values of r = j")
    ap.add_argument("--timesteps", type=int, default=1000)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--atoms", type=int, default=19)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_native_inpaint needs a CUDA device")
    T, b, nat = args.timesteps, args.batch, args.atoms
    cfg = bdiff.DenoiserConfig.named("qm9")
    net = bdiff.GCPNetDynamicsB200(config=cfg, mode="tensor")
    net.load_state_dict(O.random_state_dict(O.config_named("qm9"), seed=7), strict=True)
    net.cuda()
    sampler = bdiff.GCDMSampler(net)
    n = b * nat
    g = torch.Generator().manual_seed(9)
    types = torch.randint(0, cfg.num_atom_types, (n,), generator=g)
    mol = dict(x=(torch.randn((n, 3), generator=g) * 1.5).cuda(), one_hot=torch.eye(cfg.num_atom_types)[types].cuda(),
               charges=torch.randint(1, 10, (n, 1), generator=g).float().cuda(), num_nodes=torch.full((b,), nat),
               batch_index=torch.repeat_interleave(torch.arange(b), torch.full((b,), nat)).cuda())
    fixed = ((torch.arange(n) % nat) < 5).cuda()

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    res, clocks = {}, []
    for rj in (int(v) for v in args.rj.split(",")):
        arms = {"inpaint": lambda: sampler.inpaint(mol, fixed, rj, rj, num_timesteps=T),
                "inpaint_seed": lambda: sampler.inpaint(mol, fixed, rj, rj, num_timesteps=T, seed=123)}
        for fn in arms.values():                  # warm-up: plan, weights, graph capture of both arms
            timed(fn)
        secs = {name: [] for name in arms}
        for _ in range(args.rounds):
            for name, fn in arms.items():
                secs[name].append(timed(fn))
                clocks.append(sm_clock_mhz())
        r = {name: {"best_s": round(min(v), 4), "median_s": round(statistics.median(v), 4)} for name, v in secs.items()}
        r["seed_vs_inpaint_best"] = round(min(secs["inpaint_seed"]) / min(secs["inpaint"]) - 1.0, 4)
        r["seed_vs_inpaint_median"] = round(statistics.median(secs["inpaint_seed"]) / statistics.median(secs["inpaint"]) - 1.0, 4)
        res[f"r=j={rj}"] = r
    known = [c for c in clocks if c is not None]
    print(json.dumps({"workload": f"qm9 B={b}x{nat} T={T} tensor mode, 5 fixed atoms per molecule", "rounds": args.rounds,
                      "gpu": gpu_info(0), "sm_clock_mhz_min_max": [min(known), max(known)] if known else None,
                      "arms": res}), flush=True)


if __name__ == "__main__":
    main()

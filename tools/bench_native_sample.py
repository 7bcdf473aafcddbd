#!/usr/bin/env python
"""Times GCDMSampler.sample (torch's generator draws the noise, two randn launches per step) against
GCDMSampler.sample(seed=...) (bdiff_sample: the noise is computed inside the step kernels) on the bench workload: QM9,
128 molecules x 19 atoms, T = 1000, tensor mode.  The arms alternate within every round; the best and the median round
are reported.  Prints one JSON line with the GPU's name, power limit and SM clock.

  python tools/bench_native_sample.py [--rounds 5] [--timesteps 1000] [--batch 128] [--atoms 19]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bio-diffusion_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import torch  # noqa: E402
import bdiff  # noqa: E402
import gcpnet_oracle as O  # noqa: E402
from bench import gpu_info  # noqa: E402


def sm_clock_mhz():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return float(q.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.TimeoutExpired):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--timesteps", type=int, default=1000)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--atoms", type=int, default=19)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_native_sample needs a CUDA device")
    T, b, nat = args.timesteps, args.batch, args.atoms
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named("qm9"), mode="tensor")
    net.load_state_dict(O.random_state_dict(O.config_named("qm9"), seed=7), strict=True)
    net.cuda()
    sampler = bdiff.GCDMSampler(net)
    sizes = torch.full((b,), nat)
    arms = {"sample": lambda: sampler.sample(sizes, num_timesteps=T),
            "sample_seed": lambda: sampler.sample(sizes, num_timesteps=T, seed=123)}

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    for fn in arms.values():                      # warm-up: plan, weights, graph capture of both arms
        timed(fn)
    secs = {name: [] for name in arms}
    clocks = []
    for _ in range(args.rounds):
        for name, fn in arms.items():
            secs[name].append(timed(fn))
            clocks.append(sm_clock_mhz())
    res = {name: {"best_s": round(min(v), 4), "median_s": round(statistics.median(v), 4),
                  "molecules_per_s_best": round(b / min(v), 3), "ms_per_step_best": round(1e3 * min(v) / (T + 1), 4)}
           for name, v in secs.items()}
    res["seed_vs_sample_best"] = round(min(secs["sample_seed"]) / min(secs["sample"]) - 1.0, 4)
    res["seed_vs_sample_median"] = round(statistics.median(secs["sample_seed"]) / statistics.median(secs["sample"]) - 1.0, 4)
    known = [c for c in clocks if c is not None]
    print(json.dumps({"workload": f"qm9 B={b}x{nat} T={T} tensor mode", "rounds": args.rounds, "gpu": gpu_info(0),
                      "sm_clock_mhz_min_max": [min(known), max(known)] if known else None, "arms": res}), flush=True)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Times GCDMSampler.inpaint (RePaint) against GCDMSampler.sample on the bench workload: QM9, 128 molecules x 19 atoms,
T = 1000, tensor mode, the first 5 atoms of every molecule fixed.  (r, j) = (1, 1) and (10, 10); the arms alternate within
every round and the best round is reported.  Prints one JSON line: ms per denoiser forward, molecules/s, library kernels
per op, NaN-guard hits per arm, and the GPU's name and power limit.

  python tools/bench_inpaint.py [--rounds 2] [--timesteps 1000] [--batch 128] [--atoms 19]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bio-diffusion_b200"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import torch  # noqa: E402
import bdiff  # noqa: E402
import gcpnet_oracle as O  # noqa: E402
from bdiff.schedule import repaint_schedule  # noqa: E402
from bench import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--timesteps", type=int, default=1000)
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--atoms", type=int, default=19)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_inpaint needs a CUDA device")
    T, b, nat = args.timesteps, args.batch, args.atoms
    ocfg = O.config_named("qm9")
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named("qm9"), mode="tensor")
    net.load_state_dict(O.random_state_dict(ocfg, seed=7), strict=True)
    net.cuda()
    sampler = bdiff.GCDMSampler(net)
    n = b * nat
    g = torch.Generator().manual_seed(9)
    mol = dict(x=(torch.randn((n, 3), generator=g) * 1.5).cuda(),
               one_hot=torch.eye(ocfg.num_atom_types)[torch.randint(0, ocfg.num_atom_types, (n,), generator=g)].cuda(),
               charges=torch.randint(1, 10, (n, 1), generator=g).float().cuda(), num_nodes=torch.full((b,), nat),
               batch_index=torch.repeat_interleave(torch.arange(b), nat).cuda())
    fixed = ((torch.arange(n) % nat) < 5).cuda()
    sizes = torch.full((b,), nat)

    arms = {"sample": (lambda: sampler.sample(sizes, num_timesteps=T), T)}
    for r, j in ((1, 1), (10, 10)):
        ops = sum(repaint_schedule(r, j, T))
        arms[f"inpaint_r{r}_j{j}"] = ((lambda r=r, j=j: sampler.inpaint(mol, fixed, r, j, num_timesteps=T)), ops)

    def timed(fn):
        k0 = sampler.kernel_launches
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, sampler.kernel_launches - k0

    timed(arms["sample"][0])                                   # warm-up: modules, plan, graph capture
    timed(arms["inpaint_r1_j1"][0])
    best, nan_hits = {}, {}
    for _ in range(args.rounds):
        for name, (fn, ops) in arms.items():
            sampler.nan_guard_count(reset=True)
            sec, launches = timed(fn)
            nan_hits[name] = nan_hits.get(name, 0) + sampler.nan_guard_count()
            if name not in best or sec < best[name][0]:
                best[name] = (sec, launches, ops)
    res = {}
    for name, (sec, launches, ops) in best.items():
        res[name] = {"seconds": round(sec, 3), "denoiser_forwards": ops + 1,
                     "ms_per_forward": round(1e3 * sec / (ops + 1), 3), "molecules_per_s": round(b / sec, 3),
                     "library_kernels_per_op": round((launches - net.kernels_per_forward - 2) / ops, 2),
                     "randn_per_op": 4 if name != "sample" else 2, "nan_guard_hits_all_rounds": nan_hits[name]}
    base = res["sample"]["ms_per_forward"]
    for name in res:
        res[name]["per_forward_vs_sample"] = round(res[name]["ms_per_forward"] / base - 1.0, 4)
    print(json.dumps({"workload": f"qm9 B={b}x{nat} T={T} tensor mode, 5 fixed atoms per molecule", "rounds": args.rounds,
                      "gpu": gpu_info(0), "arms": res}), flush=True)


if __name__ == "__main__":
    main()

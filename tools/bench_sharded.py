#!/usr/bin/env python
"""Molecules/s of the sharded generation and scoring workloads on N GPUs (torchrun, NCCL; one rank per GPU), strong
scaling (the batch is split over the ranks):

  inpaint_qm9_cond     inpaint_sharded, r = j = 1, T steps, QM9-conditional, batch 128 from the QM9 histogram
  optimize_predict     optimize_sharded (--opt-steps) + predict_sharded, QM9-conditional, batch 128: one iteration of
                       the property-optimisation loop, molecules kept on their rank (gather=False) and only the scores
                       gathered
  inpaint_geom_hist    inpaint_sharded, r = j = 1, T steps, GEOM-Drugs, 512 molecules from the GEOM histogram

The first 5 atoms of every molecule are fixed.  Untrained seeded weights, tensor mode.  Every workload runs once untimed
(module load, plan, graph capture), then --rounds timed runs between barriers with a device synchronise; the best round
is reported.  Rank 0 prints one JSON line with the card's name, power limit and SM clocks read right after the runs.

  torchrun --nproc_per_node N tools/bench_sharded.py [--timesteps 1000] [--opt-steps 10] [--rounds 1]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "bio-diffusion_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import bdiff  # noqa: E402
import classifier_oracle as CO  # noqa: E402  (seeded classifier weights only)
import gcpnet_oracle as O  # noqa: E402  (seeded denoiser weights only)
from bdiff import distributed as D  # noqa: E402


def card(index):
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                        "-i", str(index)], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else torch.cuda.get_device_name(index)


def workload(cname, seed, scale, histogram, batch, dev):
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named(cname), mode="tensor")
    net.load_state_dict(O.random_state_dict(O.config_named(cname), seed, scale=scale), strict=True)
    s = bdiff.GCDMSampler(net.to(dev))
    sizes = bdiff.sample_num_nodes(histogram, batch, seed=0)
    g = torch.Generator().manual_seed(1)
    b, n = len(sizes), int(sizes.sum())
    bi = torch.repeat_interleave(torch.arange(b), sizes)
    x = torch.randn((n, 3), generator=g) * 1.5
    x = x - (torch.zeros((b, 3)).index_add_(0, bi, x) / sizes[:, None].float())[bi]
    types = torch.randint(0, s.cfg.num_atom_types, (n,), generator=g)
    mol = dict(x=x.to(dev), one_hot=torch.eye(s.cfg.num_atom_types)[types].to(dev), num_nodes=sizes, batch_index=bi.to(dev))
    first = torch.cumsum(sizes, 0) - sizes
    fixed = ((torch.arange(n) - first[bi]) < 5).to(dev)
    ctx = torch.randn((b, s.cfg.num_context), generator=g).to(dev) if s.cfg.num_context else None
    return s, sizes, mol, fixed, ctx


def timed(fn, rounds):
    fn()
    best = None
    for _ in range(rounds):
        dist.barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        dist.barrier()
        sec = time.perf_counter() - t0
        best = sec if best is None else min(best, sec)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--timesteps", type=int, default=1000)
    ap.add_argument("--opt-steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--only", default=None, help="comma-separated subset of the workloads")
    args = ap.parse_args()
    rank, world, local_rank = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    dist.init_process_group("nccl", device_id=dev)
    torch.manual_seed(0)
    only = set(args.only.split(",")) if args.only else None
    T, res = args.timesteps, {}

    if only is None or {"inpaint_qm9_cond", "optimize_predict"} & only:
        s, sizes, mol, fixed, ctx = workload("qm9_cond", 7, 0.5, bdiff.QM9_N_NODES, 128, dev)
        if only is None or "inpaint_qm9_cond" in only:
            sec = timed(lambda: D.inpaint_sharded(s, mol, fixed, 1, 1, 1, T, ctx), args.rounds)
            res["inpaint_qm9_cond"] = {"molecules": len(sizes), "atoms": int(sizes.sum()), "timesteps": T,
                                       "seconds": round(sec, 3), "molecules_per_s": round(len(sizes) / sec, 3)}
        if only is None or "optimize_predict" in only:
            clf = bdiff.PropertyClassifier(n_layers=7, attention=True, node_attr=0)
            clf.load_state_dict(CO.random_state_dict(9), strict=True)
            clf.to(dev).requires_grad_(False)
            samples, o = [], 0
            for k in sizes.tolist():
                samples.append((mol["x"][o:o + k], mol["one_hot"][o:o + k]))
                o += k

            def iteration():
                out, mine = D.optimize_sharded(s, samples, sizes, ctx, args.opt_steps, gather=False)
                my_sizes = sizes[torch.tensor(mine, dtype=torch.long)]
                scores = clf.predict(out[:, :3], out[:, 3:8], my_sizes) if mine else torch.zeros(0, device=dev)
                return D.gather_shards(scores, sizes, per_atom=False)
            sec = timed(iteration, args.rounds)
            res["optimize_predict"] = {"molecules": len(sizes), "atoms": int(sizes.sum()), "optimize_steps": args.opt_steps,
                                       "seconds": round(sec, 4), "molecules_per_s": round(len(sizes) / sec, 1)}
    if only is None or "inpaint_geom_hist" in only:
        s, sizes, mol, fixed, _ = workload("geom", 7, 1.0, bdiff.GEOM_N_NODES, 512, dev)
        sec = timed(lambda: D.inpaint_sharded(s, mol, fixed, 1, 1, 1, T), args.rounds)
        res["inpaint_geom_hist"] = {"molecules": len(sizes), "atoms": int(sizes.sum()), "timesteps": T,
                                    "shard_imbalance": round(D.shard_imbalance(sizes.tolist(), world), 4),
                                    "seconds": round(sec, 3), "molecules_per_s": round(len(sizes) / sec, 3)}
    if rank == 0:
        print(json.dumps({"bench_sharded": {"gpus": world, "rounds": args.rounds, "device": card(local_rank),
                                            "workloads": res}}), flush=True)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()

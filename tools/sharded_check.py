"""N GPUs (torchrun, NCCL): the sharded entry points of bdiff.distributed against single-GPU calls.  For every workload —
sample with and without frames, inpaint (r = j = 1 with and without frames, r = j = 2), optimize, the property
classifier and the stability check — it checks that
  (1) each rank's local output (gather=False) equals the plain single-GPU call on that rank's sub-batch, from the same
      decorrelated generator state (bit-exact);
  (2) the gathered output is bit-identical on every rank, and its rows of this rank's molecules are the local output;
and, for the optimisation loop, that (3) the scores of the gather=False shards, gathered, equal `predict` on the gathered
molecules (the classifier's tiles of pairs start at other offsets in a different batch, so fp32 sums may be associated
differently: <= 1e-5 relative).  Tensor mode, T = 4.  Rank 0 prints one JSON line; the exit code is non-zero on a failure.

  torchrun --nproc_per_node 2 tools/sharded_check.py
"""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, "bio-diffusion_b200"), os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import bdiff  # noqa: E402
import classifier_oracle as CO  # noqa: E402  (seeded classifier weights only)
import gcpnet_oracle as O  # noqa: E402  (seeded denoiser weights only)
from bdiff import distributed as D  # noqa: E402

T = 4


def sampler_for(cname, seed, scale, dev):
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named(cname), mode="tensor")
    net.load_state_dict(O.random_state_dict(O.config_named(cname), seed, scale=scale), strict=True)
    return bdiff.GCDMSampler(net.to(dev))


def molecules(cfg, sizes, dev, seed=4):
    g = torch.Generator().manual_seed(seed)
    b, n = len(sizes), int(sizes.sum())
    bi = torch.repeat_interleave(torch.arange(b), sizes)
    x = torch.randn((n, 3), generator=g) * 1.5
    x = x - (torch.zeros((b, 3)).index_add_(0, bi, x) / sizes[:, None].float())[bi]
    types = torch.randint(0, cfg.num_atom_types, (n,), generator=g)
    mol = dict(x=x.to(dev), one_hot=torch.eye(cfg.num_atom_types)[types].to(dev), num_nodes=sizes, batch_index=bi.to(dev))
    if cfg.include_charges:
        mol["charges"] = torch.randint(1, 10, (n, 1), generator=g).float().to(dev)
    return mol, (torch.rand(n, generator=g) < 0.4).to(dev)


def split(mol, fixed, ctx, sizes, mine):
    """The sub-batch of molecules `mine` as a single-GPU caller would build it."""
    rows = D._atom_rows(sizes.tolist(), mine).to(fixed.device)
    idx = torch.tensor(mine, dtype=torch.long)
    loc = {k: mol[k].index_select(0, rows) for k in ("x", "one_hot", "charges") if k in mol}
    loc["num_nodes"] = sizes[idx]
    loc["batch_index"] = torch.repeat_interleave(torch.arange(len(mine)), loc["num_nodes"]).to(fixed.device)
    return loc, fixed.index_select(0, rows), (ctx[idx.to(ctx.device)] if ctx is not None else None), rows


def same_on_every_rank(t):
    ref = t.clone()
    dist.broadcast(ref, 0)
    ok = torch.tensor([int(torch.equal(ref, t))], device=t.device)
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    return bool(ok.item())


def check(name, sharded, single, rows_of, results):
    """sharded(gather) -> (out, mine); single(mine) -> the plain call on the sub-batch; rows_of(full, mine) -> local rows."""
    sharded(False)                                       # graphs of this rank's shard shape, and the RNG fold
    state = torch.cuda.get_rng_state()
    local, mine = sharded(False)
    torch.cuda.set_rng_state(state)
    ref = single(mine) if mine else None
    torch.cuda.set_rng_state(state)
    full, _ = sharded(True)
    local_t = local if isinstance(local, tuple) else (local,)
    full_t = full if isinstance(full, tuple) else (full,)
    ref_t = ref if isinstance(ref, tuple) else (ref,)
    ok_local = ref is None or all(torch.equal(a, b) for a, b in zip(local_t, ref_t))
    ok_rows = all(torch.equal(rows_of(f, mine, i), a) for i, (f, a) in enumerate(zip(full_t, local_t)))
    ok_same = all(same_on_every_rank(f.to(torch.int32) if f.dtype == torch.bool else f) for f in full_t)
    flags = torch.tensor([int(ok_local), int(ok_rows)], device=full_t[0].device)
    dist.all_reduce(flags, op=dist.ReduceOp.MIN)
    results[name] = {"local_equals_single_gpu_call": bool(flags[0]), "gathered_rows_equal_local": bool(flags[1]),
                     "gathered_identical_on_ranks": ok_same}


def main():
    rank, world, local_rank = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    dist.init_process_group("nccl", device_id=dev)
    torch.manual_seed(17)
    results = {}

    def atoms(sizes, frames_dim=0):
        return lambda full, mine, i: full.index_select(frames_dim, D._atom_rows(sizes.tolist(), mine).to(full.device))

    # sample (GEOM) with and without frames
    s = sampler_for("geom", 2, 1.0, dev)
    sizes = torch.tensor([12, 30, 7, 44, 19, 61, 3, 25])
    for frames in (1, 4):
        check(f"sample_geom_f{frames}", lambda g: D.sample_sharded(s, sizes, None, T, gather=g, return_frames=frames),
              lambda mine: s.sample(sizes[torch.tensor(mine)], None, T, return_frames=frames)[0],
              atoms(sizes, int(frames > 1)), results)
    # inpaint (QM9-conditional)
    s = sampler_for("qm9_cond", 7, 0.5, dev)
    sizes = torch.tensor([9, 1, 17, 29, 12, 19, 14, 22, 5])
    ctx = torch.randn((len(sizes), 1), generator=torch.Generator().manual_seed(3)).to(dev)
    mol, fixed = molecules(s.cfg, sizes, dev)
    for r, j, frames in ((1, 1, 1), (1, 1, 4), (2, 2, 1)):
        def single(mine, r=r, j=j, frames=frames):
            loc, fx, c, _ = split(mol, fixed, ctx, sizes, mine)
            return s.inpaint(loc, fx, r, j, frames, T, c)
        check(f"inpaint_qm9_cond_r{r}_j{j}_f{frames}",
              lambda g, r=r, j=j, frames=frames: D.inpaint_sharded(s, mol, fixed, r, j, frames, T, ctx, gather=g),
              single, atoms(sizes, int(frames > 1)), results)
    # optimize (QM9-conditional), then the scores of the optimised molecules
    samples, o = [], 0
    for k in sizes.tolist():
        samples.append((mol["x"][o:o + k], mol["one_hot"][o:o + k]))
        o += k

    def single_opt(mine):
        loc, _, c, _ = split(mol, fixed, ctx, sizes, mine)
        z = s._optimize_latent(s.cfg, samples, sizes, dev)          # the whole batch's check, as optimize_sharded does
        rows = D._atom_rows(sizes.tolist(), mine).to(dev)
        return s.sample(loc["num_nodes"], c, T, z_init=z.index_select(0, rows))[0]
    check("optimize_qm9_cond", lambda g: D.optimize_sharded(s, samples, sizes, ctx, T, gather=g), single_opt,
          atoms(sizes), results)
    clf = bdiff.PropertyClassifier(n_layers=7, attention=True, node_attr=0)
    clf.load_state_dict(CO.random_state_dict(9), strict=True)
    clf.to(dev).requires_grad_(False)
    local, mine = D.optimize_sharded(s, samples, sizes, ctx, T, gather=False)
    my_sizes = sizes[torch.tensor(mine, dtype=torch.long)]
    scores = clf.predict(local[:, :3], local[:, 3:8], my_sizes) if mine else torch.zeros(0, device=dev)
    gathered_scores = D.gather_shards(scores, sizes, per_atom=False)
    full = D.gather_shards(local, sizes)
    direct = clf.predict(full[:, :3], full[:, 3:8], sizes)
    rel = ((gathered_scores - direct).abs().max() / direct.abs().max().clamp(min=1.0)).item()
    results["scores_of_shards_vs_predict_on_gathered"] = {"max_rel_diff": rel, "bit_equal": bool(torch.equal(gathered_scores, direct)),
                                                          "within_1e-5": rel <= 1e-5}
    # predict and the stability check on the gathered molecules
    check("predict", lambda g: D.predict_sharded(clf, full[:, :3], full[:, 3:8], sizes, gather=g),
          lambda mine: clf.predict(*(full.index_select(0, D._atom_rows(sizes.tolist(), mine).to(dev))[:, a:b]
                                     for a, b in ((0, 3), (3, 8))), sizes[torch.tensor(mine)]),
          lambda f, mine, i: f.index_select(0, torch.tensor(mine, dtype=torch.long, device=f.device)), results)
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "stability.pt"), weights_only=False)["geom"]
    info = {"atom_decoder": fx["atom_decoder"], "bonds1": fx["bonds"][0], "bonds2": fx["bonds"][1], "bonds3": fx["bonds"][2]}
    st_sizes = torch.tensor(fx["sizes"])
    pos, types = fx["x"].to(dev), fx["atom_types"].to(dev)

    def single_stab(mine):
        rows = D._atom_rows(st_sizes.tolist(), mine).to(dev)
        return bdiff.check_molecular_stability_batch(pos.index_select(0, rows), types.index_select(0, rows),
                                                     st_sizes[torch.tensor(mine)], info, fx["allowed_bonds"], fx["margins"])

    def stab_rows(f, mine, i):
        idx = D._atom_rows(st_sizes.tolist(), mine) if i == 3 else torch.tensor(mine, dtype=torch.long)
        return f.index_select(0, idx.to(f.device))
    check("stability_geom", lambda g: D.stability_sharded(pos, types, st_sizes, info, fx["allowed_bonds"], gather=g,
                                                          margins=fx["margins"]), single_stab, stab_rows, results)

    ok = all(all(v for k, v in r.items() if isinstance(v, bool) and k != "bit_equal") for r in results.values())
    if rank == 0:
        print(json.dumps({"sharded_check": {"world": world, "device": torch.cuda.get_device_name(dev), "ok": ok,
                                            "checks": results}}), flush=True)
    dist.destroy_process_group()
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()

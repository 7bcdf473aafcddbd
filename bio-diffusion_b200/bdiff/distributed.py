"""Multi-GPU generation and scoring: shard independent molecules across ranks, one final gather (SURVEY.md §8e).

The reference samples on one device only (src/mol_gen_sample.py:108-112).  Molecules are independent except
for the `_orientations` boundary quirk (SURVEY.md fact 2), so each rank runs the whole chain on its own
sub-batch with no communication and the final blocks are exchanged once (NCCL all_gather of padded blocks over
NVLink; gloo on CPU for tests).  The same holds for every per-molecule workload: `sample_sharded`,
`inpaint_sharded`, `optimize_sharded` (chains, optionally with frames), `predict_sharded` (property classifier)
and `stability_sharded` (the batched stability check).  Each validates the whole batch on every rank before its
shard runs, so a bad argument raises everywhere instead of leaving the other ranks in the gather.  With
gather=False each returns this rank's output and molecules; `gather_shards` gathers such outputs later.

Parity policy: PER-SHARD — the oracle for rank r is the reference run on rank r's sub-batch (what a user sharding
the reference by hand would get).  Batch-level decisions of the chain are therefore made per shard: the orientation
quirk at shard boundaries, and the CoG drift fix of `_finish`, applied when the largest per-molecule drift of the
(sub-)batch exceeds 5e-2 (DESIGN.md §5).

Training (config 5) is plain replica data parallelism in the reference (Lightning DDP, one all-reduce of all gradients
per step, configs/trainer/ddp.yaml); `allreduce_mean_` below is that exchange for a list of gradient tensors: packed
into buckets, ONE collective per bucket, averaged, unpacked in place.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist

from . import stability as _stability
from .classifier import predict_inputs
from .sampler import GCDMSampler
from .schedule import check_frames, check_repaint


def lpt_shards(num_nodes: Sequence[int], world_size: int) -> List[List[int]]:
    """Longest-processing-time bin packing of molecules by cost n^2 (edge count). Deterministic.

    Returns, per rank, the molecule ids it owns (ascending, so each shard keeps the caller's order).
    """
    order = sorted(range(len(num_nodes)), key=lambda i: (-int(num_nodes[i]) ** 2, i))
    loads = [0] * world_size
    shards: List[List[int]] = [[] for _ in range(world_size)]
    for i in order:
        r = min(range(world_size), key=lambda k: (loads[k], k))
        shards[r].append(i)
        loads[r] += int(num_nodes[i]) ** 2
    return [sorted(s) for s in shards]


def _source_rows(shards: Sequence[Sequence[int]], rows_per_mol: Sequence[int], pad: int) -> torch.Tensor:
    """Row g of the caller's order (molecule after molecule, molecule i owning rows_per_mol[i] rows) -> the row holding it
    in the concatenation of the ranks' blocks, each block padded to `pad` rows.  int64 [sum rows] on the host."""
    rows = torch.tensor([int(v) for v in rows_per_mol], dtype=torch.int64)
    start = torch.zeros(rows.numel(), dtype=torch.int64)           # first row of each molecule in the concatenation
    for r, s in enumerate(shards):
        if s:
            idx = torch.tensor(list(s), dtype=torch.int64)
            cnt = rows[idx]
            start[idx] = r * pad + torch.cumsum(cnt, 0) - cnt
    first = torch.cumsum(rows, 0) - rows                           # first row of each molecule in the caller's order
    return torch.arange(int(rows.sum())) + torch.repeat_interleave(start - first, rows)


def _gather_rows(local: torch.Tensor, shards: Sequence[Sequence[int]], rows_per_mol: Sequence[int], world: int,
                 group=None, row_dim: int = 0) -> torch.Tensor:
    """all_gather every rank's block (axis `row_dim` holds the rank's rows, molecule after molecule in shard order) padded
    to the longest one, then put the rows in the caller's molecule order with one index_select on the device.  Every rank
    calls it, one with an empty shard too.  The result is data: it carries no autograd history."""
    if local.dtype == torch.bool:                                    # not every backend moves bool
        return _gather_rows(local.to(torch.uint8), shards, rows_per_mol, world, group, row_dim).bool()
    counts = [sum(int(rows_per_mol[i]) for i in s) for s in shards]
    blk = local.detach().movedim(row_dim, 0)
    tail = tuple(blk.shape[1:])
    width = math.prod(tail)
    pad = max(max(counts), 1)
    buf = torch.zeros((pad, width), dtype=local.dtype, device=local.device)
    buf[: blk.shape[0]] = blk.reshape(blk.shape[0], width)
    if world > 1:
        parts = [torch.empty_like(buf) for _ in range(world)]
        dist.all_gather(parts, buf, group=group)
        buf = torch.cat(parts)
    src = _source_rows(shards, rows_per_mol, pad).to(local.device)
    out = buf.index_select(0, src).reshape((src.numel(),) + tail)
    return out.movedim(0, row_dim).contiguous() if row_dim else out


def gather_results(local_out: torch.Tensor, local_mols: Sequence[int], num_nodes: Sequence[int],
                   world_size: int, group=None) -> torch.Tensor:
    """all_gather the per-rank [N_r, D] blocks and restore the global molecule order -> [N, D] on every rank."""
    return _gather_rows(local_out, lpt_shards(num_nodes, world_size), num_nodes, world_size, group)


def gather_shards(local_out: torch.Tensor, num_nodes, per_atom: bool = True, row_dim: int = 0, group=None) -> torch.Tensor:
    """Gathers what a sharded entry point returned with gather=False, on every rank, in the caller's molecule order:
    per-atom blocks [N_r, ...] (per_atom=True; [F, N_r, ...] frames with row_dim=1) or per-molecule rows [B_r, ...]
    (per_atom=False).  `num_nodes` is the whole batch's, as given to the sharded call."""
    world, _ = _world_rank(group)
    sizes = [int(v) for v in torch.as_tensor(num_nodes).reshape(-1).tolist()]
    rows = sizes if per_atom else [1] * len(sizes)
    return _gather_rows(local_out, lpt_shards(sizes, world), rows, world, group, row_dim)


_rank_seed_folded = False


def decorrelate_rank_rng(rank: int) -> None:
    """Fold the rank into this process's default CUDA generator ONCE.  The reference seeds every process identically
    (`seed_everything(cfg.seed)`); with LPT giving equal-shaped shards for uniform-size batches, identically seeded
    ranks would draw the same noise and generate bit-identical molecules (silent duplicates in uniqueness / novelty
    statistics).  Rank 0 keeps the caller's stream, so a 1-GPU run is unchanged."""
    global _rank_seed_folded
    if _rank_seed_folded or rank == 0 or not torch.cuda.is_available():
        _rank_seed_folded = True
        return
    torch.cuda.manual_seed((torch.cuda.initial_seed() + 0x9E3779B97F4A7C15 * rank) % (1 << 63))
    _rank_seed_folded = True


def _world_rank(group=None) -> Tuple[int, int]:
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(group), dist.get_rank(group)
    return 1, 0


def _my_shard(sizes: Sequence[int], group=None):
    """(world size, every rank's molecules, this rank's molecules), after decorrelating this rank's noise stream."""
    world, rank = _world_rank(group)
    decorrelate_rank_rng(rank)
    shards = lpt_shards(sizes, world)
    return world, shards, shards[rank]


def _atom_rows(sizes: Sequence[int], mols: Sequence[int]) -> torch.Tensor:
    """The atoms (rows of the packed batch with molecule sizes `sizes`) of molecules `mols`, ascending: int64 on the host."""
    n = torch.tensor([int(v) for v in sizes], dtype=torch.int64)
    idx = torch.tensor(list(mols), dtype=torch.int64)
    cnt = n[idx]
    first = (torch.cumsum(n, 0) - n)[idx]
    return torch.arange(int(cnt.sum())) + torch.repeat_interleave(first - (torch.cumsum(cnt, 0) - cnt), cnt)


def _take(t: torch.Tensor, rows: torch.Tensor) -> torch.Tensor:
    return t.index_select(0, rows.to(t.device))


def _no_atoms(cfg, frames: int, dev) -> torch.Tensor:
    """The block of a rank without molecules: [0, 3+A(+1)], or [F, 0, 3+A(+1)] with frames."""
    d = 3 + cfg.num_atom_types + int(cfg.include_charges)
    return torch.zeros((frames, 0, d) if frames > 1 else (0, d), device=dev)


def _atoms_out(out, shards, sizes, world, group, frames, mine, gather):
    if not gather:
        return out, mine
    return _gather_rows(out, shards, sizes, world, group, row_dim=int(frames > 1)), mine


def sample_sharded(sampler, num_nodes: torch.Tensor, context: Optional[torch.Tensor] = None,
                   num_timesteps: Optional[int] = None, group=None, gather: bool = True, return_frames: int = 1):
    """Each rank samples its LPT shard with `sampler` (a GCDMSampler); returns (out_full or out_local, my_mols).

    out is [N, 3+A(+1)], or [F, N, 3+A(+1)] for return_frames = F > 1 (frame 0 = the molecules, as `sample` returns it).
    The per-rank noise streams are decorrelated here (see decorrelate_rank_rng).  A rank whose shard is empty (more
    ranks than molecules) skips the chain and contributes a zero-row block, so the final collective still matches."""
    cfg = sampler.cfg
    frames = int(return_frames)
    if frames != 1:
        check_frames(cfg.num_timesteps if num_timesteps is None else int(num_timesteps), frames)
    sizes = [int(v) for v in num_nodes.tolist()]
    world, shards, mine = _my_shard(sizes, group)
    if mine:
        idx = torch.tensor(mine, dtype=torch.long)
        local_nodes = num_nodes.cpu()[idx]
        local_ctx = context.cpu()[idx] if context is not None else None
        frame_arg = {"return_frames": frames} if frames != 1 else {}
        out = sampler.sample(local_nodes, local_ctx, num_timesteps, **frame_arg)[0]
    else:
        out = _no_atoms(cfg, frames, sampler._device())
    return _atoms_out(out, shards, sizes, world, group, frames, mine, gather)


def inpaint_sharded(sampler, molecule: dict, node_mask_fixed: torch.Tensor, num_resamplings: int = 1,
                    jump_length: int = 1, return_frames: int = 1, num_timesteps: Optional[int] = None,
                    context: Optional[torch.Tensor] = None, group=None, gather: bool = True):
    """GCDMSampler.inpaint with the molecules sharded over the ranks; arguments and `out` as inpaint's, returns
    (out_full or out_local, my_mols).

    The whole batch is validated on every rank before anything else, so a bad argument raises the same exception on every
    rank and none is left waiting in the gather.  A shard keeps its molecules' atoms, fixed-atom masks and context rows;
    its batch_index is re-derived from its num_nodes."""
    cfg = sampler.cfg
    frames = int(return_frames)
    check_repaint(int(num_resamplings), int(jump_length), cfg.num_timesteps if num_timesteps is None else int(num_timesteps),
                  frames)
    num_nodes = GCDMSampler._inpaint_inputs(cfg, molecule, node_mask_fixed, context)[0]
    sizes = num_nodes.tolist()
    world, shards, mine = _my_shard(sizes, group)
    if mine:
        rows, idx = _atom_rows(sizes, mine), torch.tensor(mine, dtype=torch.long)
        local = {k: _take(molecule[k], rows) for k in ("x", "one_hot", "charges") if k in molecule}
        local["num_nodes"] = num_nodes[idx]
        local["batch_index"] = torch.repeat_interleave(torch.arange(len(mine)), local["num_nodes"]).to(
            molecule["batch_index"].device)
        out = sampler.inpaint(local, _take(node_mask_fixed, rows), num_resamplings, jump_length, frames, num_timesteps,
                              _take(context, idx) if context is not None else None)
    else:
        out = _no_atoms(cfg, frames, sampler._device())
    return _atoms_out(out, shards, sizes, world, group, frames, mine, gather)


def optimize_sharded(sampler, samples, num_nodes: torch.Tensor, context: Optional[torch.Tensor],
                     num_timesteps: Optional[int] = None, return_frames: int = 1, group=None, gather: bool = True):
    """GCDMSampler.optimize with the molecules sharded over the ranks; `samples` = (x [n_k,3], one_hot [n_k,A]) of every
    molecule, returns (out_full or out_local, my_mols).

    The reference's mean-zero assertion sums the positions of the WHOLE batch: it runs here once, on the full batch and on
    every rank, so whether it raises does not depend on the world size.  Each rank then runs optimize's chain (`sample`
    started from the normalised molecules) on its shard; optimize itself would repeat the assertion on the shard's sum."""
    cfg = sampler.cfg
    if cfg.include_charges:
        raise NotImplementedError("mol_gen_optimize stacks [x | one-hot] only: needs include_charges=False")
    frames = int(return_frames)
    check_frames(cfg.num_timesteps if num_timesteps is None else int(num_timesteps), frames)
    num_nodes = torch.as_tensor(num_nodes)
    z = GCDMSampler._optimize_latent(cfg, samples, num_nodes, sampler._device())
    sizes = [int(v) for v in num_nodes.tolist()]
    world, shards, mine = _my_shard(sizes, group)
    if mine:
        rows, idx = _atom_rows(sizes, mine), torch.tensor(mine, dtype=torch.long)
        out = sampler.sample(num_nodes.cpu()[idx], _take(context, idx) if context is not None else None, num_timesteps,
                             z_init=_take(z, rows), return_frames=frames)[0]
    else:
        out = _no_atoms(cfg, frames, sampler._device())
    return _atoms_out(out, shards, sizes, world, group, frames, mine, gather)


def predict_sharded(classifier, x: torch.Tensor, one_hot: torch.Tensor, num_nodes, group=None, gather: bool = True):
    """PropertyClassifier.predict with the molecules sharded over the ranks: returns (pred [B] in the caller's molecule
    order, or this rank's pred [B_r], my_mols).  The batch is validated on every rank first."""
    nn_ = predict_inputs(x, one_hot, num_nodes)
    sizes = nn_.tolist()
    world, shards, mine = _my_shard(sizes, group)
    if mine:
        rows = _atom_rows(sizes, mine)
        out = classifier.predict(_take(x, rows), _take(one_hot, rows), nn_[torch.tensor(mine, dtype=torch.long)])
    else:
        out = torch.zeros(0, dtype=torch.float32, device=x.device)
    if not gather:
        return out, mine
    return _gather_rows(out, shards, [1] * len(sizes), world, group), mine


def stability_sharded(positions: torch.Tensor, atom_types: torch.Tensor, num_nodes: torch.Tensor, dataset_info: dict,
                      allowed_bonds, group=None, gather: bool = True, margins: Tuple[float, float, float] = (10.0, 5.0, 3.0),
                      limit_bonds_to_one: bool = False):
    """check_molecular_stability_batch with the molecules sharded over the ranks: returns ((molecule_stable bool[B],
    nr_stable_bonds int32[B], n int32[B], per-atom bond counts int32[N]) in the caller's order, or this rank's four
    outputs, my_mols).  The batch is validated on every rank first."""
    nn_ = _stability.stability_inputs(positions, atom_types, num_nodes, dataset_info, allowed_bonds)
    sizes = nn_.tolist()
    world, shards, mine = _my_shard(sizes, group)
    dev = positions.device
    if mine:
        rows = _atom_rows(sizes, mine)
        out = _stability.check_molecular_stability_batch(_take(positions, rows), _take(atom_types, rows),
                                                         nn_[torch.tensor(mine, dtype=torch.long)], dataset_info,
                                                         allowed_bonds, margins, limit_bonds_to_one)
    else:
        z = torch.zeros(0, dtype=torch.int32, device=dev)
        out = (z.bool(), z, z, z)
    if not gather:
        return out, mine
    stable, nr_stable, n, nr_bonds = out
    per_mol = _gather_rows(torch.stack((stable.to(torch.int32), nr_stable, n), dim=1), shards, [1] * len(sizes), world,
                           group)
    return (per_mol[:, 0].bool(), per_mol[:, 1].contiguous(), per_mol[:, 2].contiguous(),
            _gather_rows(nr_bonds, shards, sizes, world, group)), mine


def shard_imbalance(num_nodes: Sequence[int], world_size: int) -> float:
    """max over ranks of the LPT shard cost (sum n^2) divided by the mean: 1.0 = perfectly balanced."""
    shards = lpt_shards(num_nodes, world_size)
    loads = [sum(int(num_nodes[i]) ** 2 for i in s) for s in shards]
    mean = sum(loads) / max(1, world_size)
    return max(loads) / mean if mean > 0 else 1.0


def allreduce_mean_flat_(flat: torch.Tensor, group=None) -> int:
    """In-place mean over the ranks of ONE contiguous buffer (GCDMTrainTail keeps all gradients in one): a single
    all-reduce, no packing.  Returns the number of collectives issued (0 when the world size is 1)."""
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return 0
    dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
    flat.div_(dist.get_world_size(group))
    return 1


def allreduce_mean_(tensors: Sequence[torch.Tensor], group=None, bucket_bytes: int = 64 << 20) -> int:
    """In-place mean over the ranks of `group` of every tensor in `tensors` (the gradients of one step), packed into
    contiguous buckets of at most `bucket_bytes` so that a 2.7 M-parameter model is ONE all-reduce.  All tensors must
    share dtype and device.  Returns the number of collectives issued (0 when the world size is 1)."""
    tensors = [t for t in tensors if t is not None and t.numel() > 0]
    if not tensors:
        return 0
    if not dist.is_available() or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return 0
    world = dist.get_world_size(group)
    dtype, dev = tensors[0].dtype, tensors[0].device
    if any(t.dtype != dtype or t.device != dev for t in tensors):
        raise ValueError("allreduce_mean_: tensors must share dtype and device")
    per = max(1, bucket_bytes // tensors[0].element_size())
    buckets: List[List[torch.Tensor]] = [[]]
    fill = 0
    for t in tensors:
        if buckets[-1] and fill + t.numel() > per:
            buckets.append([])
            fill = 0
        buckets[-1].append(t)
        fill += t.numel()
    for b in buckets:
        flat = torch.cat([t.reshape(-1) for t in b])
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        flat.div_(world)
        o = 0
        for t in b:
            t.copy_(flat[o:o + t.numel()].view_as(t))
            o += t.numel()
    return len(buckets)

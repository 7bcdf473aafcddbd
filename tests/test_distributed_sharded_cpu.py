"""CPU, world_size 2 over gloo: the sharded entry points of bdiff.distributed (inpaint, optimize, sample with frames,
classifier scoring, stability check) return every molecule's rows in the caller's order, with and without the gather.
The per-rank workloads are faked by functions of each molecule's own inputs, so the expected output of any sharding is
the fake run on the whole batch.  Bad arguments must raise on every rank before a collective (gloo's timeout turns a
hang into a failure)."""
import datetime
import os
import sys
from types import SimpleNamespace

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "bio-diffusion_b200"))

A = 5                                          # QM9's atom types (the classifier's input): outputs are [.., 3 + A]
INFO = {"atom_decoder": ["H", "C", "N", "O", "F"]}
ALLOWED = {"H": 1, "C": 4, "N": 3, "O": 2, "F": 1}


def _per_mol(v, batch_index, b):
    return torch.zeros((b,) + v.shape[1:], dtype=v.dtype).index_add_(0, batch_index, v)


class FakeSampler:
    """Stands in for GCDMSampler: outputs [N, 3 + A] (or [F, N, 3 + A]) whose every row is a function of its molecule's
    inputs and the atom's place in it."""
    cfg = SimpleNamespace(num_atom_types=A, include_charges=False, num_context=1, num_timesteps=8,
                          norm_values=(1.0, 4.0, 10.0), norm_biases=(None, -0.5, 0.0))

    def _device(self):
        return torch.device("cpu")

    @staticmethod
    def _frames(out, frames):
        if frames == 1:
            return out
        return torch.stack([out + 1000.0 * k for k in range(frames)])

    def sample(self, num_nodes, context=None, num_timesteps=None, z_init=None, return_frames=1):
        nn_ = num_nodes.cpu()
        bi = torch.repeat_interleave(torch.arange(len(nn_)), nn_)
        first = (torch.cumsum(nn_, 0) - nn_)[bi]
        j = torch.arange(len(bi)) - first
        ctx = context.cpu()[bi, 0] if context is not None else torch.zeros(len(bi))
        zs = z_init.sum(dim=1) if z_init is not None else torch.zeros(len(bi))
        out = torch.stack((nn_[bi].float(), j.float(), ctx, zs, torch.full((len(bi),), float(num_timesteps or 0))), 1)
        out = torch.cat((out, torch.zeros((len(bi), A - 2))), 1)
        return self._frames(out, return_frames), bi, torch.ones(len(bi), dtype=torch.bool)

    def inpaint(self, molecule, node_mask_fixed, num_resamplings=1, jump_length=1, return_frames=1, num_timesteps=None,
                context=None):
        nn_ = torch.as_tensor(molecule["num_nodes"]).cpu()
        bi = molecule["batch_index"].cpu()
        assert torch.equal(bi, torch.repeat_interleave(torch.arange(len(nn_)), nn_))
        x, oh = molecule["x"].cpu(), molecule["one_hot"].cpu()
        mol_x = _per_mol(x.sum(1), bi, len(nn_))[bi]                    # depends on the whole molecule, not its place
        out = torch.stack((x.sum(1), oh.argmax(1).float(), node_mask_fixed.cpu().float(), context.cpu()[bi, 0] + mol_x,
                           torch.full((len(bi),), 10.0 * num_resamplings + jump_length)), 1)
        out = torch.cat((out, oh[:, : A - 2]), 1)
        return self._frames(out, return_frames)


class FakeClassifier:
    def predict(self, x, one_hot, num_nodes):
        nn_ = torch.as_tensor(num_nodes).cpu()
        bi = torch.repeat_interleave(torch.arange(len(nn_)), nn_)
        return _per_mol(x.sum(1) + 3.0 * one_hot.argmax(1), bi, len(nn_)) + 0.5 * nn_


def fake_stability(positions, atom_types, num_nodes, dataset_info, allowed_bonds, margins=None, limit_bonds_to_one=False):
    nn_ = torch.as_tensor(num_nodes).cpu()
    bi = torch.repeat_interleave(torch.arange(len(nn_)), nn_)
    nr_bonds = (atom_types.int() * 2 + (positions[:, 0] > 0).int()).to(torch.int32)
    nr_stable = _per_mol(nr_bonds, bi, len(nn_)).to(torch.int32)
    return nr_stable % 2 == 0, nr_stable, nn_.to(torch.int32), nr_bonds


def make_batch(sizes, seed=0):
    """A packed batch with every molecule's positions centred (optimize's mean-zero requirement)."""
    g = torch.Generator().manual_seed(seed)
    nn_ = torch.tensor(sizes)
    b, n = len(sizes), int(nn_.sum())
    bi = torch.repeat_interleave(torch.arange(b), nn_)
    x = torch.randn((n, 3), generator=g)
    x = x - (_per_mol(x, bi, b) / nn_[:, None].float())[bi]
    types = torch.randint(0, A, (n,), generator=g)
    return dict(x=x, one_hot=torch.eye(A)[types], num_nodes=nn_, batch_index=bi), types, \
        torch.rand(n, generator=g) < 0.4, torch.randn((b, 1), generator=g)


def samples_of(mol):
    out, o = [], 0
    for k in mol["num_nodes"].tolist():
        out.append((mol["x"][o:o + k], mol["one_hot"][o:o + k]))
        o += k
    return out


def run_all(sizes, gather):
    """Every sharded entry point on the same batch: {name: (out, my_mols)}."""
    from bdiff import distributed as D
    mol, types, fixed, ctx = make_batch(sizes)
    s, nn_ = FakeSampler(), mol["num_nodes"]
    res = {}
    for frames in (1, 4):
        res[f"sample_f{frames}"] = D.sample_sharded(s, nn_, ctx, 8, gather=gather, return_frames=frames)
        res[f"inpaint_f{frames}"] = D.inpaint_sharded(s, mol, fixed, 1, 1, frames, 8, ctx, gather=gather)
        res[f"optimize_f{frames}"] = D.optimize_sharded(s, samples_of(mol), nn_, ctx, 8, frames, gather=gather)
    res["inpaint_r2j2"] = D.inpaint_sharded(s, mol, fixed, 2, 2, 1, 8, ctx, gather=gather)
    res["predict"] = D.predict_sharded(FakeClassifier(), mol["x"], mol["one_hot"], nn_, gather=gather)
    res["stability"] = D.stability_sharded(mol["x"], types, nn_, INFO, ALLOWED, gather=gather)
    if not gather:        # the outputs gathered afterwards, as an optimise-score-select loop would
        for k, (out, mine) in list(res.items()):
            if k == "stability":
                res["stability_gathered"] = (
                    [D.gather_shards(out[i], nn_, per_atom=False) for i in range(3)] + [D.gather_shards(out[3], nn_)], mine)
            else:
                per_atom, row_dim = k != "predict", int(k.endswith("_f4"))
                res[k + "_gathered"] = (D.gather_shards(out, nn_, per_atom=per_atom, row_dim=row_dim), mine)
    return res


def expected(sizes):
    """The fakes run on the whole batch (what any sharding must reproduce)."""
    from bdiff.sampler import GCDMSampler
    mol, types, fixed, ctx = make_batch(sizes)
    s, nn_ = FakeSampler(), mol["num_nodes"]
    z = GCDMSampler._optimize_latent(s.cfg, samples_of(mol), nn_, torch.device("cpu"))
    exp = {}
    for frames in (1, 4):
        exp[f"sample_f{frames}"] = s.sample(nn_, ctx, 8, return_frames=frames)[0]
        exp[f"inpaint_f{frames}"] = s.inpaint(mol, fixed, 1, 1, frames, 8, ctx)
        exp[f"optimize_f{frames}"] = s.sample(nn_, ctx, 8, z_init=z, return_frames=frames)[0]
    exp["inpaint_r2j2"] = s.inpaint(mol, fixed, 2, 2, 1, 8, ctx)
    exp["predict"] = FakeClassifier().predict(mol["x"], mol["one_hot"], nn_)
    exp["stability"] = fake_stability(mol["x"], types, nn_, INFO, ALLOWED)
    return exp


def _init(rank, world, port):
    sys.path.insert(0, os.path.join(ROOT, "bio-diffusion_b200"))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=60))
    import bdiff.stability
    bdiff.stability.check_molecular_stability_batch = fake_stability       # the real one needs a GPU


def _worker(rank, world, port, sizes, gather, results):
    _init(rank, world, port)
    results[rank] = run_all(sizes, gather)
    dist.barrier()
    dist.destroy_process_group()


def _rows(t, sizes, mine, per_atom=True, row_dim=0):
    """The rows of molecules `mine` (ascending) of a caller-ordered output."""
    from bdiff.distributed import _atom_rows
    idx = _atom_rows(sizes, mine) if per_atom else torch.tensor(mine, dtype=torch.long)
    return t.index_select(row_dim, idx)


def _spawn(fn, *args):
    mgr = mp.Manager()
    results = mgr.dict()
    mp.spawn(fn, args=args + (results,), nprocs=2, join=True)
    return dict(results)


@pytest.mark.parametrize("sizes,port", [([5, 19, 3, 12, 7, 19, 2], 29611),     # unequal shards
                                        ([6], 29613)])                          # more ranks than molecules
def test_two_rank_sharded_calls_return_the_callers_order(sizes, port):
    results = _spawn(_worker, 2, port, sizes, True)
    exp = expected(sizes)
    for rank in (0, 1):
        for k, want in exp.items():
            got, _ = results[rank][k]
            if k == "stability":
                assert all(torch.equal(a, b) for a, b in zip(got, want)), (rank, k)
                assert got[0].dtype == torch.bool and got[3].shape == (sum(sizes),)
            else:
                assert torch.equal(got, want), (rank, k)
    mine = [results[r]["predict"][1] for r in (0, 1)]
    assert sorted(mine[0] + mine[1]) == list(range(len(sizes)))
    if len(sizes) == 1:
        assert mine[1] == []


@pytest.mark.parametrize("sizes,port", [([5, 19, 3, 12, 7, 19, 2], 29615), ([6], 29617)])
def test_two_rank_local_outputs_and_later_gather(sizes, port):
    """gather=False: each rank holds exactly its own molecules' rows; gather_shards assembles the caller's order."""
    results = _spawn(_worker, 2, port, sizes, False)
    exp = expected(sizes)
    for rank in (0, 1):
        for k, want in exp.items():
            local, mine = results[rank][k]
            full, _ = results[rank][k + "_gathered"]
            if k == "stability":
                for i in range(4):
                    assert torch.equal(local[i], _rows(want[i], sizes, mine, per_atom=i == 3)), (rank, k, i)
                    assert torch.equal(full[i], want[i].to(full[i].dtype)), (rank, k, i)
                continue
            per_atom, row_dim = k != "predict", int(k.endswith("_f4"))
            assert torch.equal(local, _rows(want, sizes, mine, per_atom, row_dim)), (rank, k)
            assert torch.equal(full, want), (rank, k)


def _bad_worker(rank, world, port, results):
    _init(rank, world, port)
    from bdiff import distributed as D
    sizes = [5, 19, 3, 12]
    mol, types, fixed, ctx = make_batch(sizes)
    s, nn_ = FakeSampler(), mol["num_nodes"]
    off_centre = samples_of(mol)
    off_centre[3] = (off_centre[3][0] + 1.0, off_centre[3][1])         # the last molecule is rank 1's; its CoG is not 0
    bad_types = types.clone()
    bad_types[-1] = A
    calls = {
        "inpaint_fixed_mask": lambda: D.inpaint_sharded(s, mol, fixed[:-1], context=ctx),
        "inpaint_no_context": lambda: D.inpaint_sharded(s, mol, fixed),
        "inpaint_frames_with_jumps": lambda: D.inpaint_sharded(s, mol, fixed, 2, 2, 2, 8, ctx),
        "optimize_mean": lambda: D.optimize_sharded(s, off_centre, nn_, ctx, 8),
        "optimize_counts": lambda: D.optimize_sharded(s, samples_of(mol), torch.tensor([5, 19, 3, 11]), ctx, 8),
        "sample_frames": lambda: D.sample_sharded(s, nn_, ctx, 8, return_frames=3),
        "predict_one_hot": lambda: D.predict_sharded(FakeClassifier(), mol["x"], mol["one_hot"][:, :1], nn_),
        "stability_types": lambda: D.stability_sharded(mol["x"], bad_types, nn_, INFO, ALLOWED),
    }
    out = {}
    for name, fn in calls.items():
        try:
            fn()
            out[name] = None
        except Exception as e:       # noqa: BLE001 — the type and message are what is compared
            out[name] = (type(e).__name__, str(e))
    dist.barrier()                   # both ranks get here: no rank was left inside a gather
    results[rank] = out
    dist.destroy_process_group()


def test_invalid_arguments_raise_on_every_rank():
    results = _spawn(_bad_worker, 2, 29619)
    assert set(results) == {0, 1}
    for name, err in results[0].items():
        assert err is not None, name
        assert results[1][name] == err, name
    assert results[0]["optimize_mean"][0] == "AssertionError"


def _old_loop(gathered, shards, num_nodes):
    """gather_results' assembly before the row permutation: a copy per molecule."""
    offsets = [0]
    for n in num_nodes:
        offsets.append(offsets[-1] + int(n))
    out = torch.empty((offsets[-1], gathered[0].shape[1]), dtype=gathered[0].dtype)
    for r, s in enumerate(shards):
        pos = 0
        for i in s:
            n = int(num_nodes[i])
            out[offsets[i]: offsets[i] + n] = gathered[r][pos: pos + n]
            pos += n
    return out


def _layouts():
    g = torch.Generator().manual_seed(3)
    out = [[1], [4, 4], [181, 3, 3, 3], [2, 1]]
    for _ in range(8):
        b = int(torch.randint(1, 40, (1,), generator=g))
        out.append(torch.randint(1, 60, (b,), generator=g).tolist())
    return out


def _gather_worker(rank, world, port, results):
    _init(rank, world, port)
    from bdiff.distributed import gather_results, lpt_shards
    out = []
    for k, sizes in enumerate(_layouts()):
        mine = lpt_shards(sizes, world)[rank]
        g = torch.Generator().manual_seed(1000 * k + rank)
        local = torch.randn((sum(sizes[i] for i in mine), 7), generator=g)
        out.append((local, gather_results(local, mine, sizes, world)))
    results[rank] = out
    dist.barrier()
    dist.destroy_process_group()


def test_gather_equals_the_per_molecule_loop_on_random_layouts():
    from bdiff.distributed import lpt_shards
    results = _spawn(_gather_worker, 2, 29621)
    for k, sizes in enumerate(_layouts()):
        shards = lpt_shards(sizes, 2)
        blocks = [results[r][k][0] for r in (0, 1)]
        want = _old_loop(blocks, shards, sizes)
        for r in (0, 1):
            assert torch.equal(results[r][k][1], want), (k, r)


def test_one_process_sharded_calls_equal_direct_calls():
    """Without torch.distributed (one rank) every entry point is the plain call on the whole batch."""
    import bdiff.stability
    from bdiff import distributed as D
    saved = bdiff.stability.check_molecular_stability_batch
    bdiff.stability.check_molecular_stability_batch = fake_stability
    try:
        sizes = [5, 19, 3, 12, 7]
        exp = expected(sizes)
        for gather in (True, False):
            res = run_all(sizes, gather)
            for k, want in exp.items():
                got, mine = res[k]
                assert mine == list(range(len(sizes)))
                if k == "stability":
                    assert all(torch.equal(a, b) for a, b in zip(got, want)), k
                else:
                    assert torch.equal(got, want), (k, gather)
    finally:
        bdiff.stability.check_molecular_stability_batch = saved

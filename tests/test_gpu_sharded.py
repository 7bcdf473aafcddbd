"""GPU, one rank: every sharded entry point of bdiff.distributed (LPT shard + gather) returns what the plain single-GPU
call returns for the same molecules and seed, element for element.  Tensor mode, which is bit-deterministic for every
molecule size (parity mode's 32-edge tiles sum the pieces of longer rows with atomics).  Every chain runs once before
the seeded pair, so that neither call of the pair captures its CUDA graph first (capture advances the generator
differently from a replay)."""
import os

import pytest
import torch

import classifier_oracle as CO
import gcpnet_oracle as O
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

T = 4
CONFIGS = {"geom": ([12, 30, 7, 44, 19], 2, 1.0), "qm9_cond": ([9, 1, 17, 29, 12, 19], 7, 0.5)}


def _sampler(cname):
    import bdiff
    sizes, seed, scale = CONFIGS[cname]
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named(cname), mode="tensor")
    net.load_state_dict(O.random_state_dict(O.config_named(cname), seed, scale=scale), strict=True)
    net.cuda()
    s = bdiff.GCDMSampler(net)
    g = torch.Generator().manual_seed(3)
    ctx = torch.randn((len(sizes), s.cfg.num_context), generator=g).cuda() if s.cfg.num_context else None
    return s, torch.tensor(sizes), ctx


def _molecules(cfg, sizes, seed=4):
    """Packed molecules with every molecule's positions centred, and a random set of fixed atoms."""
    g = torch.Generator().manual_seed(seed)
    b, n = len(sizes), int(sizes.sum())
    bi = torch.repeat_interleave(torch.arange(b), sizes)
    x = torch.randn((n, 3), generator=g) * 1.5
    x = x - (torch.zeros((b, 3)).index_add_(0, bi, x) / sizes[:, None].float())[bi]
    types = torch.randint(0, cfg.num_atom_types, (n,), generator=g)
    mol = dict(x=x.cuda(), one_hot=torch.eye(cfg.num_atom_types)[types].cuda(), num_nodes=sizes, batch_index=bi.cuda())
    if cfg.include_charges:
        mol["charges"] = torch.randint(1, 10, (n, 1), generator=g).float().cuda()
    return mol, (torch.rand(n, generator=g) < 0.4).cuda()


def _seeded_pair(plain, sharded):
    plain()                                          # captures the graphs of this shape
    torch.manual_seed(5)
    ref = plain()
    torch.manual_seed(5)
    out, mine = sharded()
    return ref, out, mine


@pytest.mark.parametrize("r,j,frames", [(1, 1, 1), (1, 1, 4), (2, 2, 1)])
@pytest.mark.parametrize("cname", list(CONFIGS))
def test_inpaint_sharded_on_one_gpu_equals_inpaint(cname, r, j, frames):
    from bdiff.distributed import inpaint_sharded
    s, sizes, ctx = _sampler(cname)
    mol, fixed = _molecules(s.cfg, sizes)
    ref, out, mine = _seeded_pair(lambda: s.inpaint(mol, fixed, r, j, frames, T, ctx),
                                  lambda: inpaint_sharded(s, mol, fixed, r, j, frames, T, ctx))
    assert mine == list(range(len(sizes)))
    assert out.shape == ref.shape and torch.isfinite(out).all() and torch.equal(out, ref)


@pytest.mark.parametrize("frames", [1, 2])
@pytest.mark.parametrize("cname", list(CONFIGS))
def test_optimize_sharded_on_one_gpu_equals_optimize(cname, frames):
    from bdiff.distributed import optimize_sharded
    s, sizes, ctx = _sampler(cname)
    mol, _ = _molecules(s.cfg, sizes)
    samples, o = [], 0
    for k in sizes.tolist():
        samples.append((mol["x"][o:o + k], mol["one_hot"][o:o + k]))
        o += k
    ref, out, mine = _seeded_pair(lambda: s.optimize(samples, sizes, ctx, T, return_frames=frames)[0],
                                  lambda: optimize_sharded(s, samples, sizes, ctx, T, frames))
    assert mine == list(range(len(sizes))) and torch.equal(out, ref)


@pytest.mark.parametrize("cname", list(CONFIGS))
def test_sample_sharded_frames_on_one_gpu_equal_sample(cname):
    from bdiff.distributed import sample_sharded
    s, sizes, ctx = _sampler(cname)
    ref, out, mine = _seeded_pair(lambda: s.sample(sizes, ctx, T, return_frames=4)[0],
                                  lambda: sample_sharded(s, sizes, ctx, T, return_frames=4))
    assert out.shape[0] == 4 and mine == list(range(len(sizes))) and torch.equal(out, ref)


def test_predict_sharded_on_one_gpu_equals_predict():
    import bdiff
    from bdiff.distributed import predict_sharded
    clf = bdiff.PropertyClassifier(n_layers=7, attention=True, node_attr=0)
    clf.load_state_dict(CO.random_state_dict(9), strict=True)
    clf.cuda().requires_grad_(False)
    sizes = bdiff.sample_num_nodes(bdiff.QM9_N_NODES, 128, seed=4)
    g = torch.Generator().manual_seed(8)
    n = int(sizes.sum())
    x = (torch.randn((n, 3), generator=g) * 1.5).cuda()
    oh = torch.nn.functional.one_hot(torch.randint(0, 5, (n,), generator=g), 5).float().cuda()
    ref = clf.predict(x, oh, sizes)
    out, mine = predict_sharded(clf, x, oh, sizes)
    assert mine == list(range(len(sizes))) and torch.equal(out, ref)
    local, _ = predict_sharded(clf, x, oh, sizes, gather=False)
    assert torch.equal(local, ref)


@pytest.mark.parametrize("name", ["qm9", "geom"])
def test_stability_sharded_on_one_gpu_equals_batch_check(name):
    from bdiff.distributed import stability_sharded
    from bdiff.stability import check_molecular_stability_batch
    fx = torch.load(os.path.join(GOLDEN, "stability.pt"), weights_only=False)[name]
    info = {"atom_decoder": fx["atom_decoder"], "bonds1": fx["bonds"][0], "bonds2": fx["bonds"][1], "bonds3": fx["bonds"][2]}
    args = (fx["x"].cuda(), fx["atom_types"].cuda(), torch.tensor(fx["sizes"]), info, fx["allowed_bonds"])
    ref = check_molecular_stability_batch(*args, fx["margins"])
    out, mine = stability_sharded(*args, margins=fx["margins"])
    assert mine == list(range(len(fx["sizes"])))
    for a, b in zip(out, ref):
        assert a.dtype == b.dtype and torch.equal(a, b)

"""GPU: one GCDMSampler across calls that change the context values, the sizes, the chain kind and the weights.  Every
output of the graph sampler equals, element for element, that of a fresh eager sampler (use_cuda_graph=False) run from
the same seed, and a second call with the same sizes and new context values replays the graph the first one captured:
a captured graph reads only buffers the sampler owns.  Tensor mode, which is bit-deterministic.  The eager samplers run
on a second denoiser with the same weights, so that their plans do not replace the one the graph sampler reuses."""
import pytest
import torch

import gcpnet_oracle as O

pytestmark = pytest.mark.gpu

T = 5


def _net():
    import bdiff
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named("qm9_cond"), mode="tensor")
    net.load_state_dict(O.random_state_dict(O.config_named("qm9_cond"), 7, scale=0.5), strict=True)
    return net.cuda()


def _context(b, seed):
    return torch.randn((b, 1), generator=torch.Generator().manual_seed(seed)).cuda()


def _molecule(cfg, sizes):
    g = torch.Generator().manual_seed(4)
    b, n = len(sizes), int(sizes.sum())
    bi = torch.repeat_interleave(torch.arange(b), sizes)
    x = torch.randn((n, 3), generator=g) * 1.5
    types = torch.randint(0, cfg.num_atom_types, (n,), generator=g)
    mol = dict(x=x.cuda(), one_hot=torch.eye(cfg.num_atom_types)[types].cuda(), num_nodes=sizes, batch_index=bi.cuda())
    return mol, (torch.rand(n, generator=g) < 0.4).cuda()


def test_one_graph_cache_across_calls_equals_eager():
    import bdiff
    net_g, net_e = _net(), _net()
    s = bdiff.GCDMSampler(net_g)

    def both(call, seed):
        torch.manual_seed(seed)
        out = call(s)
        torch.manual_seed(seed)
        ref = call(bdiff.GCDMSampler(net_e, use_cuda_graph=False))
        assert torch.isfinite(out).all() and torch.equal(out, ref)
        return out

    sizes, other = torch.tensor([9, 17, 1, 12]), torch.tensor([19, 5, 11])
    first = both(lambda x: x.sample(sizes, _context(4, 1), T)[0], 3)
    graph = s._graphs[0]
    both(lambda x: x.sample(sizes, _context(4, 2), T)[0], 3)
    assert s._graphs[0] is graph, "new context values must not capture a new graph"
    both(lambda x: x.sample(other, _context(3, 3), T)[0], 4)
    mol, fixed = _molecule(s.cfg, other)
    both(lambda x: x.inpaint(mol, fixed, 2, 2, num_timesteps=T, context=_context(3, 3)), 5)
    assert len(s._graphs) == 2
    with torch.no_grad():
        for net in (net_g, net_e):
            for p in net.parameters():
                p.mul_(0.9)
    updated = both(lambda x: x.sample(sizes, _context(4, 1), T)[0], 3)
    assert not torch.equal(updated, first)

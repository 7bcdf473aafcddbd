"""GPU: GCDMSampler.inpaint (RePaint) and the chain frames of sample / optimize / inpaint against the reference's fixtures
and the CPU oracle, the two new C-ABI ops in isolation, graph replay against the eager loop, and a full-size run.

Bounds are those of test_chain_matches_reference_golden: z_0 and x <= 1e-4 relative, identical atom types (the rounded
charge column, which reaches 1e4 with these untrained weights, <= 1e-4 relative).  The oracle's
own fp32-vs-fp64 gap on these fixtures is <= 4e-7 (make_golden_inpaint.py checks it before writing a fixture)."""
import ctypes as C

import pytest
import torch

import gcpnet_oracle as O
import inpaint_oracle as IO
from conftest import load_golden

pytestmark = pytest.mark.gpu

INPAINT_CASES = ["inpaint_qm9_r2j2_T6", "inpaint_qm9_cond_r3j1_T4_frames", "inpaint_geom_r1j1_T3"]


def make_net(cname, seed, scale=1.0, mode="parity"):
    import bdiff
    ocfg = O.config_named(cname)
    sd = O.random_state_dict(ocfg, seed, scale=scale)
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named(cname), mode=mode)
    net.load_state_dict(sd, strict=True)
    return net.cuda(), ocfg, sd


def rel(a, b):
    return (a.cpu() - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def check_out(ocfg, out, ref, frames_tol=1e-4):
    assert out.shape == ref.shape
    o, r = (out, ref) if ref.dim() == 3 else (out.unsqueeze(0), ref.unsqueeze(0))
    o = o.cpu()
    a = ocfg.num_atom_types
    assert torch.equal(o[0, :, 3:3 + a], r[0, :, 3:3 + a]), "atom types differ"
    if ocfg.include_charges:       # round(10 * h) of |h| ~ 1e3: the rounding may flip where the value is not exact
        assert rel(o[0, :, 3 + a:], r[0, :, 3 + a:]) <= 1e-4, "charges differ"
    assert rel(o[0, :, :3], r[0, :, :3]) <= 1e-4, f"x rel diff {rel(o[0, :, :3], r[0, :, :3]):.3e}"
    if r.shape[0] > 1:
        assert rel(o[1:], r[1:]) <= frames_tol, f"frames rel diff {rel(o[1:], r[1:]):.3e}"


def molecule_cuda(fx):
    return {k: fx[k].cuda() for k in ("x", "one_hot", "charges", "num_nodes", "batch_index")}


@pytest.mark.parametrize("mode", ["parity", "tensor"])
@pytest.mark.parametrize("name", INPAINT_CASES)
def test_inpaint_matches_reference_golden(name, mode):
    """The fixture's CPU noise stream replayed on the GPU; z_0 (the last denoiser input) and the output."""
    import bdiff
    fx = load_golden(name)
    net, ocfg, _ = make_net(fx["config"], fx["weight_seed"], fx["weight_scale"], mode)
    sampler = bdiff.GCDMSampler(net)
    ctx = fx["context"].cuda() if fx["context"] is not None else None
    torch.manual_seed(fx["noise_seed"])
    out = sampler.inpaint(molecule_cuda(fx), fx["node_mask_fixed"].cuda(), fx["num_resamplings"], fx["jump_length"],
                          fx["return_frames"], fx["steps"], ctx, noise=lambda s: torch.randn(s).cuda())
    z0 = sampler._static["z"]
    assert rel(z0, fx["z_0"]) <= 1e-4, f"z_0 rel diff {rel(z0, fx['z_0']):.3e}"
    check_out(ocfg, out, fx["out"])


def test_sample_frames_match_reference_golden():
    import bdiff
    fx = load_golden("chain_frames_qm9_T6")
    net, ocfg, _ = make_net(fx["config"], fx["weight_seed"], fx["weight_scale"])
    sampler = bdiff.GCDMSampler(net)
    torch.manual_seed(fx["noise_seed"])
    out, _, _ = sampler.sample(torch.tensor(fx["sizes"]), num_timesteps=fx["steps"], return_frames=fx["return_frames"],
                               noise=lambda s: torch.randn(s).cuda())
    check_out(ocfg, out, fx["out"])
    # the default stays [N, D] and the frames path does not disturb a later plain chain
    torch.manual_seed(fx["noise_seed"])
    plain, _, _ = sampler.sample(torch.tensor(fx["sizes"]), num_timesteps=fx["steps"], noise=lambda s: torch.randn(s).cuda())
    assert plain.shape == fx["out"].shape[1:]


def test_optimize_frames_match_oracle():
    import bdiff
    net, ocfg, sd = make_net("geom", 7, 0.5)
    g = torch.Generator().manual_seed(3)
    sizes = [30, 21]
    bi = torch.repeat_interleave(torch.arange(2), torch.tensor(sizes))
    n = bi.shape[0]
    mask = torch.ones(n, dtype=torch.bool)
    _, x = O.centralize(torch.randn((n, 3), generator=g) * 1.5, bi, mask, 2)
    one_hot = torch.nn.functional.one_hot(torch.randint(0, ocfg.num_atom_types, (n,), generator=g), ocfg.num_atom_types).float()
    z_init = O.normalize_samples(ocfg, x, one_hot, mask)
    ref = IO.sample_chain_frames(sd, ocfg, torch.tensor(sizes), O.SeededNoise(8), 4, 2, z_init=z_init)
    noise = O.SeededNoise(8)
    samples = [(x[:30], one_hot[:30]), (x[30:], one_hot[30:])]
    out, _, _ = bdiff.GCDMSampler(net).optimize(samples, torch.tensor(sizes), num_timesteps=4, return_frames=2,
                                                noise=lambda s: noise(s).cuda())
    check_out(ocfg, out, ref)


def test_frames_graph_equals_eager():
    """sample with frames: the captured graph (frame write inside) and the eager loop agree bit-wise on the device RNG."""
    import bdiff
    net, _, _ = make_net("qm9", 7, mode="tensor")
    nn_ = torch.tensor([19, 7, 12])
    s_graph = bdiff.GCDMSampler(net)
    s_graph.sample(nn_, num_timesteps=6, return_frames=3)                  # capture
    outs = []
    for s in (s_graph, bdiff.GCDMSampler(net, use_cuda_graph=False)):
        torch.manual_seed(4)
        outs.append(s.sample(nn_, num_timesteps=6, return_frames=3)[0])
    assert outs[0].shape == (3, 38, 9) and torch.equal(outs[0], outs[1])


def test_all_free_inpaint_equals_sample():
    """No fixed atom, r = j = 1: with the unknown-part draws fed by sample()'s draws, inpaint IS sample (tensor mode)."""
    import bdiff
    net, ocfg, _ = make_net("qm9", 7, mode="tensor")
    sizes = [19, 7, 12]
    steps = 5
    n, f = sum(sizes), ocfg.num_h
    gen = O.SeededNoise(17)
    rec = []

    def record(shape):
        t = gen(shape)
        rec.append(t)
        return t.cuda()

    sampler = bdiff.GCDMSampler(net)
    ref, _, _ = sampler.sample(torch.tensor(sizes), num_timesteps=steps, noise=record)
    assert len(rec) == 2 * (steps + 2)
    junk = O.SeededNoise(99)
    stream = rec[:2]
    for k in range(steps):
        stream += [junk((n, 3)), junk((n, f))] + rec[2 + 2 * k: 4 + 2 * k]
    stream += rec[-2:]
    replay = O.RecordedNoise(stream)
    mol = dict(x=torch.randn(n, 3), one_hot=torch.eye(ocfg.num_atom_types)[torch.arange(n) % ocfg.num_atom_types],
               charges=torch.ones(n, 1), num_nodes=torch.tensor(sizes),
               batch_index=torch.repeat_interleave(torch.arange(3), torch.tensor(sizes)))
    out = sampler.inpaint(mol, torch.zeros(n, dtype=torch.bool), num_timesteps=steps, noise=lambda s: replay(s).cuda())
    assert replay.i == len(stream)
    assert torch.equal(out, ref)


@pytest.mark.parametrize("cname,sizes,fixed_spec", [
    ("qm9", [12, 7, 19, 5], {1: "none", 2: "all", 3: "none"}),
    ("geom", [181, 20], {1: "none"}),
])
def test_edge_case_batches_match_oracle(cname, sizes, fixed_spec):
    """Molecules without fixed atoms (also the last one), a fully fixed molecule and a 181-atom GEOM molecule."""
    import bdiff
    net, ocfg, sd = make_net(cname, 7, 0.5)
    g = torch.Generator().manual_seed(5)
    nmol = len(sizes)
    bi = torch.repeat_interleave(torch.arange(nmol), torch.tensor(sizes))
    n = bi.shape[0]
    x = torch.randn((n, 3), generator=g) * 1.5
    one_hot = torch.nn.functional.one_hot(torch.randint(0, ocfg.num_atom_types, (n,), generator=g), ocfg.num_atom_types).float()
    charges = torch.randint(1, 10, (n, 1), generator=g).float() if ocfg.include_charges else torch.zeros((n, 0))
    fixed = torch.rand(n, generator=g) < 0.4
    off = 0
    for k, m in enumerate(sizes):
        spec = fixed_spec.get(k)
        if spec is not None:
            fixed[off:off + m] = spec == "all"
        off += m
    steps, r, j = 4, 2, 2
    ref = IO.inpaint_chain(sd, ocfg, x, one_hot, charges, torch.tensor(sizes), fixed, O.SeededNoise(6), r, j, 1, steps)
    noise = O.SeededNoise(6)
    mol = dict(x=x.cuda(), one_hot=one_hot.cuda(), charges=charges.cuda(), num_nodes=torch.tensor(sizes), batch_index=bi)
    out = bdiff.GCDMSampler(net).inpaint(mol, fixed.cuda(), r, j, num_timesteps=steps, noise=lambda s: noise(s).cuda())
    check_out(ocfg, out, ref)


def _plan(net, sizes):
    nmol = len(sizes)
    bi = torch.repeat_interleave(torch.arange(nmol), torch.tensor(sizes))
    mask = torch.ones(bi.shape[0], dtype=torch.bool)
    net.plan(bi.cuda(), mask.cuda(), nmol)
    return bi, mask, nmol


def test_repaint_combine_and_renoise_ops_match_oracle():
    """bdiff_repaint_combine and bdiff_renoise one op at a time (row read at a device index) against the oracle."""
    from bdiff import _lib
    net, ocfg, _ = make_net("geom", 7)
    sizes = [181, 9, 30, 4]
    bi, mask, nmol = _plan(net, sizes)
    lib, h, stream = _lib.load(), net._handle, net._stream()
    n, f = bi.shape[0], ocfg.num_h
    g = torch.Generator().manual_seed(12)
    _, zx = O.centralize(torch.randn((n, 3), generator=g), bi, mask, nmol)
    z = torch.cat((zx, torch.randn((n, f), generator=g)), -1)
    xh0 = torch.randn((n, 3 + f), generator=g) * 2
    fixed = torch.rand(n, generator=g) < 0.3
    fixed[181:190] = False                             # a molecule without fixed atoms
    fixed[-4:] = True                                  # a fully fixed one
    nx, nh = torch.randn((n, 3), generator=g), torch.randn((n, f), generator=g)
    table = torch.tensor([[0.3, 0.7], [0.8125, 0.5819]])
    idx = torch.tensor(1, dtype=torch.int32)

    def p(t):
        return C.c_void_p(t.data_ptr())

    zd, xd, fd, nxd, nhd, td, idd = (t.cuda().contiguous() for t in (z, xh0, fixed.to(torch.uint8), nx, nh, table, idx))
    _lib.check(h, lib.bdiff_repaint_combine(h, stream, p(zd), p(xd), p(fd), p(nxd), p(nhd), p(td), p(idd)), "combine")
    zk = IO.known_part(ocfg, xh0, 0.8125, 0.5819, bi, mask, nmol, O.RecordedNoise([nx, nh]))
    ref = IO.combine(zk, z, fixed, bi, nmol)
    assert rel(zd, ref) <= 1e-6, f"combine rel diff {rel(zd, ref):.3e}"
    assert torch.equal(zd.cpu()[~fixed], z[~fixed])     # free rows untouched
    cog = torch.zeros((nmol, 3)).index_add_(0, bi, zd.cpu()[:, :3])
    assert cog.abs().max().item() < 1e-4                # the combination keeps every molecule CoG-free

    jt = torch.tensor([[0.5, 0.25, 0.0, 0.0], [0.97, 0.243, 0.4, 0.6]])
    zd2 = z.cuda().contiguous()
    jtd = jt.cuda()
    _lib.check(h, lib.bdiff_renoise(h, stream, p(zd2), p(nxd), p(nhd), p(jtd), p(idd)), "renoise")
    ref = IO.renoise(ocfg, z, 0.97, 0.243, bi, mask, nmol, O.RecordedNoise([nx, nh]))
    assert rel(zd2, ref) <= 1e-6, f"renoise rel diff {rel(zd2, ref):.3e}"


def test_inpaint_graph_replay_equals_eager():
    """r=2, j=2 on the device RNG: the two replayed graphs and the eager loop agree bit-wise."""
    import bdiff
    net, ocfg, _ = make_net("qm9", 7, mode="tensor")
    sizes = [19, 7, 12, 19]
    n = sum(sizes)
    g = torch.Generator().manual_seed(2)
    mol = dict(x=torch.randn((n, 3), generator=g).cuda(),
               one_hot=torch.eye(ocfg.num_atom_types)[torch.randint(0, ocfg.num_atom_types, (n,), generator=g)].cuda(),
               charges=torch.randint(1, 10, (n, 1), generator=g).float().cuda(), num_nodes=torch.tensor(sizes),
               batch_index=torch.repeat_interleave(torch.arange(4), torch.tensor(sizes)).cuda())
    fixed = (torch.rand(n, generator=g) < 0.4).cuda()
    s_graph = bdiff.GCDMSampler(net)
    s_graph.inpaint(mol, fixed, 2, 2, num_timesteps=6)                     # capture
    assert len(s_graph._graphs) == 2                                      # the denoise op and the jump back
    outs = []
    for s in (s_graph, bdiff.GCDMSampler(net, use_cuda_graph=False)):
        torch.manual_seed(11)
        outs.append((s.inpaint(mol, fixed, 2, 2, num_timesteps=6), s._static["z"].clone()))
    assert torch.isfinite(outs[0][0]).all()
    assert torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][0], outs[1][0])


def test_inpaint_full_size_qm9_b128():
    """QM9 B=128 x 19 atoms, T=1000, r = j = 1, tensor mode: finite, CoG-free per molecule, no NaN-guard hits."""
    import bdiff
    net, ocfg, _ = make_net("qm9", 7, mode="tensor")
    b, nat = 128, 19
    n = b * nat
    g = torch.Generator().manual_seed(9)
    bi = torch.repeat_interleave(torch.arange(b), torch.full((b,), nat))
    types = torch.randint(0, ocfg.num_atom_types, (n,), generator=g)
    mol = dict(x=(torch.randn((n, 3), generator=g) * 1.5).cuda(),
               one_hot=torch.eye(ocfg.num_atom_types)[types].cuda(),
               charges=torch.randint(1, 10, (n, 1), generator=g).float().cuda(), num_nodes=torch.full((b,), nat),
               batch_index=bi.cuda())
    fixed = (torch.arange(n) % nat) < 5                 # the first 5 atoms of every molecule
    sampler = bdiff.GCDMSampler(net)
    out = sampler.inpaint(mol, fixed.cuda(), num_timesteps=1000)
    assert out.shape == (n, 3 + ocfg.num_h) and torch.isfinite(out).all()
    cog = torch.zeros((b, 3), device="cuda").index_add_(0, bi.cuda(), out[:, :3])
    assert cog.abs().max().item() < 5e-2
    assert sampler.nan_guard_count() == 0

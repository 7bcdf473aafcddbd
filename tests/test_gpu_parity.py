"""GPU parity tests proper: the CUDA path (through the C ABI) vs the reference's golden outputs and the oracle.

Tolerances (parity mode, fp32 FFMA): integer work bit-exact; per-forward max-abs <= 5e-5 * max(1, |ref|_max)
(the measured fp32-vs-fp64 floor of the reference itself is ~1e-6..7e-6, SURVEY.md §8c); short chains 1e-3
relative on z_0 with identical atom types.
"""
import pytest
import torch

import gcpnet_oracle as O
from conftest import load_golden

pytestmark = pytest.mark.gpu

FWD_CASES = ["qm9_small_masked", "qm9_tiny_sizes", "qm9_b4_n19", "qm9_cond", "geom_mixed", "geom_max181"]


def make_net(cname, seed, dev="cuda", scale=1.0):
    import bdiff
    ocfg = O.config_named(cname)
    sd = O.random_state_dict(ocfg, seed, scale=scale)
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named(cname))
    net.load_state_dict(sd, strict=True)
    return net.to(dev), ocfg, sd


def relerr(a, b):
    return (a - b).abs().max().item() / max(1.0, b.abs().max().item())


def test_library_loaded_is_in_tree():
    import bdiff
    lib = bdiff.load_library()
    assert "bio-diffusion_b200/bdiff/libbdiff_sm90.so" in lib._name


def test_edge_index_kat_bit_exact():
    import bdiff
    fx = load_golden("kat_edge_index")
    net, _, _ = make_net("qm9", 7)
    for mask, key in ((fx["mask"], "edge_index"), (torch.ones_like(fx["mask"]), "edge_index_nomask")):
        bi = fx["batch_index"].cuda()
        mk = mask.cuda()
        net.plan(bi, mk)
        ei = net.edge_index()
        assert ei.dtype == torch.int64 and torch.equal(ei.cpu(), fx[key])


@pytest.mark.parametrize("name", FWD_CASES)
def test_forward_matches_reference_golden(name):
    fx = load_golden(name)
    net, ocfg, sd = make_net(fx["config"], fx["weight_seed"])
    ctx = fx["context"].cuda() if fx["context"] is not None else None
    out = net.denoise(fx["batch_index"].cuda(), fx["mask"].cuda(), fx["xh"].cuda(), fx["t"].cuda(), ctx).cpu()
    ref = fx["net_out"]
    assert relerr(out, ref) <= 5e-5, f"net_out rel err {relerr(out, ref):.3e}"
    assert net.edge_index().shape[1] == fx["num_edges"]
    if "edge_index" in fx:
        assert torch.equal(net.edge_index().cpu(), fx["edge_index"])
        assert (net.debug_tap("f_ij").cpu().reshape(-1, 3, 3) - fx["f_ij"]).abs().max().item() <= 2e-6
        assert relerr(net.debug_tap("e").cpu(), fx["e"]) <= 1e-5
        assert relerr(net.debug_tap("xi").cpu().reshape(fx["xi"].shape), fx["xi"]) <= 1e-5
        last = fx["layers"][-1]
        assert relerr(net.debug_tap("h").cpu(), last["h"]) <= 5e-5
        assert relerr(net.debug_tap("chi").cpu().reshape(last["chi"].shape), last["chi"]) <= 5e-5
        assert relerr(net.debug_tap("x").cpu(), last["x"]) <= 5e-5


def test_forward_drop_in_contract():
    """forward(batch, xh, t) -> (batch, net_out) with the reference's attribute-bag Batch."""
    fx = load_golden("qm9_b4_n19")
    net, _, _ = make_net("qm9", fx["weight_seed"])

    class Bag:
        pass

    b = Bag()
    b.batch, b.mask, b.props_context = fx["batch_index"].cuda(), fx["mask"].cuda(), None
    xh = fx["xh"].cuda()
    xh_before = xh.clone()
    with torch.inference_mode():
        rb, out = net(b, xh, fx["t"].cuda())
    assert rb is b and torch.equal(xh, xh_before)
    assert relerr(out.cpu(), fx["net_out"]) <= 5e-5
    # second call with the same Batch tensors reuses the plan
    key = net._plan_key
    with torch.no_grad():
        net(b, xh, fx["t"].cuda())
    assert net._plan_key == key
    # under autograd with trainable parameters the module runs the training pass: the output carries a grad_fn instead of
    # being silently detached (ADVICE r1); tests/test_gpu_train.py checks the gradients
    _, out_g = net(b, xh, fx["t"].cuda())
    assert out_g.grad_fn is not None and relerr(out_g.detach().cpu(), fx["net_out"]) <= 5e-5


def test_forward_is_deterministic_and_batch_composable():
    net, ocfg, sd = make_net("qm9", 3)
    g = torch.Generator().manual_seed(9)
    sizes = [19] * 16 + [5, 29, 11]
    bi = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes)).cuda()
    n = bi.shape[0]
    mask = torch.ones(n, dtype=torch.bool, device="cuda")
    xh = torch.randn((n, 9), generator=g).cuda()
    t = torch.rand((n, 1), generator=g).cuda()
    o1 = net.denoise(bi, mask, xh, t)
    o2 = net.denoise(bi, mask, xh, t)
    assert torch.equal(o1, o2), "two runs on the same input must be bit-identical"
    ref = O.denoiser_forward(sd, ocfg, bi.cpu(), mask.cpu(), xh.cpu(), t.cpu())
    assert relerr(o1.cpu(), ref) <= 5e-5


def test_se3_equivariance_on_device():
    net, ocfg, sd = make_net("geom", 5)
    g = torch.Generator().manual_seed(2)
    sizes = [44, 23]
    bi = torch.repeat_interleave(torch.arange(2), torch.tensor(sizes))
    n = bi.shape[0]
    mask = torch.ones(n, dtype=torch.bool)
    xh = torch.randn((n, 3 + ocfg.num_h), generator=g)
    _, xc = O.centralize(xh[:, :3], bi, mask, 2)
    q, _ = torch.linalg.qr(torch.randn((3, 3), generator=g))
    if torch.det(q) < 0:
        q[:, 0] = -q[:, 0]
    t = torch.full((n, 1), 0.4)
    o1 = net.denoise(bi.cuda(), mask.cuda(), torch.cat((xc, xh[:, 3:]), -1).cuda(), t.cuda()).cpu()
    o2 = net.denoise(bi.cuda(), mask.cuda(), torch.cat((xc @ q.T, xh[:, 3:]), -1).cuda(), t.cuda()).cpu()
    scale = max(1.0, o1.abs().max().item())
    assert (o2[:, :3] - o1[:, :3] @ q.T).abs().max().item() <= 2e-5 * scale
    assert (o2[:, 3:] - o1[:, 3:]).abs().max().item() <= 2e-5 * scale


@pytest.mark.parametrize("name", ["chain_qm9_T6", "chain_qm9_cond_T4", "chain_geom_T3"])
def test_chain_matches_reference_golden(name):
    """Same CPU noise stream as the reference run that produced the fixture, replayed on the GPU."""
    import bdiff
    fx = load_golden(name)
    net, ocfg, sd = make_net(fx["config"], fx["weight_seed"], scale=fx.get("weight_scale", 1.0))
    torch.manual_seed(fx["noise_seed"])          # CPU generator: identical draws to the reference's
    sampler = bdiff.GCDMSampler(net)
    ctx = fx["context"].cuda() if fx["context"] is not None else None
    out, bi, mask, z0 = sampler.sample(torch.tensor(fx["sizes"]), ctx, num_timesteps=fx["steps"],
                                       noise=lambda s: torch.randn(s).cuda(), return_z0=True)
    rel = (z0.cpu() - fx["z_0"]).abs().max().item() / fx["z_0"].abs().max().item()
    assert rel < 1e-4, f"z_0 rel diff {rel:.3e}"
    a = ocfg.num_atom_types
    assert torch.equal(out[:, 3:3 + a].cpu(), fx["out"][:, 3:3 + a])
    relx = (out[:, :3].cpu() - fx["out"][:, :3]).abs().max().item() / fx["out"][:, :3].abs().max().item()
    assert relx < 1e-4


@pytest.mark.parametrize("scale,tol", [(0.5, 2e-5), (1.0, 1e-3)])
@pytest.mark.parametrize("cname,sizes", [("qm9", [19, 7, 12]), ("qm9_cond", [9, 14]), ("geom", [30, 44])])
def test_reverse_steps_teacher_forced_vs_oracle(cname, sizes, scale, tol):
    """Every reverse step checked in isolation: the GPU step starts from the ORACLE's z_t, so round-off is not
    amplified across steps.  With 0.5-scaled weights the step is well conditioned (tolerance 2e-5); with full-size
    random weights the untrained net drives |z| to 1e5 and one step alone amplifies fp32 round-off to ~1e-4
    (the oracle's own fp32-vs-fp64 difference is of that order), so the tolerance there is 1e-3."""
    import bdiff
    net, ocfg, sd = make_net(cname, 7, scale=scale)
    steps = 5
    nmol = len(sizes)
    num_nodes = torch.tensor(sizes)
    bi = torch.repeat_interleave(torch.arange(nmol), num_nodes)
    n = bi.shape[0]
    mask = torch.ones(n, dtype=torch.bool)
    g = torch.Generator().manual_seed(21)
    ctx_b = torch.randn((nmol, ocfg.num_context), generator=g) if ocfg.num_context else None
    ctx = ctx_b[bi] if ctx_b is not None else None
    gamma = O.gamma_table(ocfg.num_timesteps, ocfg.noise_precision, ocfg.schedule_power)
    noise = O.SeededNoise(33)
    z = O.combined_noise(noise, ocfg, bi, mask, nmol)
    sampler = bdiff.GCDMSampler(net)
    for r, s in enumerate(reversed(range(steps))):
        nx, nh = noise((n, 3)), noise((n, ocfg.num_h))
        replay = O.RecordedNoise([nx, nh])
        z_next = O.reverse_step(sd, ocfg, gamma, s, s + 1, z, bi, mask, ctx, replay, steps, nmol)
        z_gpu = sampler.reverse_step_once(z.cuda(), r, steps, bi.cuda(), mask.cuda(), nx.cuda(), nh.cuda(),
                                          ctx.cuda() if ctx is not None else None, nmol).cpu()
        rel = (z_gpu - z_next).abs().max().item() / z_next.abs().max().item()
        assert rel < tol, f"step {r}: rel diff {rel:.3e}"
        z = z_next


def test_cuda_graph_chain_equals_eager_chain():
    """The captured-graph sampler and the eager loop consume the same device RNG stream and agree bit-wise."""
    import bdiff
    net, ocfg, sd = make_net("qm9", 7)
    nn_ = torch.tensor([19, 7, 12, 19])
    outs = []
    for use_graph in (False, True):
        torch.manual_seed(11)
        s = bdiff.GCDMSampler(net, use_cuda_graph=use_graph)
        out, _, _, z0 = s.sample(nn_, num_timesteps=5, return_z0=True)
        outs.append((out.clone(), z0.clone()))
    assert torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][0], outs[1][0])


def test_full_size_properties_qm9_b128():
    """BASELINE config[1] size: finite, CoG-free velocity, masked-free batch, reproducible, permutation of
    molecule ORDER changes nothing but the orientation boundary rows (SURVEY.md fact 2)."""
    net, ocfg, sd = make_net("qm9", 7)
    g = torch.Generator().manual_seed(4)
    b, nat = 128, 19
    bi = torch.repeat_interleave(torch.arange(b), torch.full((b,), nat)).cuda()
    n = b * nat
    mask = torch.ones(n, dtype=torch.bool, device="cuda")
    xh = torch.randn((n, 9), generator=g)
    _, xc = O.centralize(xh[:, :3], bi.cpu(), mask.cpu(), b)
    xh = torch.cat((xc, xh[:, 3:]), -1).cuda()
    t = torch.full((n, 1), 0.5, device="cuda")
    out = net.denoise(bi, mask, xh, t)
    assert torch.isfinite(out).all()
    cog = torch.zeros((b, 3), device="cuda").index_add_(0, bi, out[:, :3])
    assert cog.abs().max().item() < 1e-4
    assert net.edge_index().shape[1] == b * nat * nat
    # linearity check of the sampler algebra is in test_chain_*; here: the oracle on a 4-molecule slice
    sl = slice(0, 4 * nat)
    ref = O.denoiser_forward(sd, ocfg, bi[sl].cpu(), mask[sl].cpu(), xh[sl].cpu(), t[sl].cpu())
    # all rows except the last atom of the slice see the same neighbours as in the full batch
    assert relerr(out[sl][:3 * nat].cpu(), ref[:3 * nat]) <= 5e-5


@pytest.mark.parametrize("name", ["nll_qm9", "nll_geom"])
def test_eval_nll_on_device_matches_reference(name):
    """GCDMEvalNLL (two denoiser calls through the C ABI + torch bookkeeping on the GPU) vs the reference's terms.
    The CPU noise stream of the fixture is replayed; tolerance 1e-4 relative on every term and on the NLL."""
    import bdiff
    fx = load_golden(name)
    net, ocfg, sd = make_net(fx["config"], fx["weight_seed"], scale=fx["weight_scale"])
    ev = bdiff.GCDMEvalNLL(net, fx["histogram"])
    torch.manual_seed(fx["rng_seed"])
    t_int = torch.randint(1, ocfg.num_timesteps + 1, size=(len(fx["sizes"]), 1))      # same first draw as the reference
    assert torch.equal(t_int.squeeze(-1), fx["terms"]["t_int"])
    nll, terms = ev(fx["batch_index"].cuda(), fx["mask"].cuda(), fx["x"].cuda(), fx["one_hot"].cuda(),
                    fx["charges"].cuda(), None, t_int=t_int, noise=lambda s: torch.randn(s))
    for k, ref in fx["terms"].items():
        if k == "t_int":
            continue
        assert torch.allclose(terms[k].cpu(), ref, rtol=1e-4, atol=1e-4), (k, terms[k].cpu(), ref)
    assert torch.allclose(nll.cpu(), fx["nll"], rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("autograd", [False, True])
@pytest.mark.parametrize("name", ["train_qm9", "train_geom"])
def test_training_loss_on_device_matches_reference(name, autograd):
    """GCDMTrainLoss (one denoiser call through the C ABI, t == 0 molecule included) vs the reference in .train() mode;
    the fixture's t_int and CPU noise stream are replayed; tolerance 1e-4 relative on every term and on the loss.
    autograd=False: value from the sampler kernels; True: from the training pass (loss carries a grad_fn)."""
    import bdiff
    fx = load_golden(name)
    net, ocfg, sd = make_net(fx["config"], fx["weight_seed"], scale=fx["weight_scale"])
    tl = bdiff.GCDMTrainLoss(net, fx["histogram"])
    torch.manual_seed(fx["rng_seed"])
    with torch.set_grad_enabled(autograd):
        loss, terms = tl(fx["batch_index"].cuda(), fx["mask"].cuda(), fx["x"].cuda(), fx["one_hot"].cuda(),
                         fx["charges"].cuda(), None, t_int=fx["terms"]["t_int"].reshape(-1, 1), noise=lambda s: torch.randn(s))
    assert loss.requires_grad == autograd
    loss, terms = loss.detach(), {k: v.detach() for k, v in terms.items()}
    for k, ref in fx["terms"].items():
        if k == "t_int":
            continue
        assert torch.allclose(terms[k].cpu(), ref, rtol=1e-4, atol=1e-4), (k, terms[k].cpu(), ref)
    assert torch.allclose(loss.cpu(), fx["nll"], rtol=1e-4, atol=1e-3)


@pytest.mark.parametrize("name", ["optimize_qm9_cond_T4", "optimize_geom_T3"])
def test_optimize_chain_matches_reference_golden(name):
    """GCDMSampler.optimize (= mol_gen_optimize: the chain started from given molecules) vs the reference, CPU noise
    stream replayed; identical atom types, coordinates <= 1e-4 relative."""
    import bdiff
    fx = load_golden(name)
    net, ocfg, sd = make_net(fx["config"], fx["weight_seed"], scale=fx["weight_scale"])
    sampler = bdiff.GCDMSampler(net)
    samples, o = [], 0
    for k in fx["sizes"]:
        samples.append((fx["x"][o:o + k], fx["one_hot"][o:o + k]))
        o += k
    ctx = fx["context"].cuda() if fx["context"] is not None else None
    torch.manual_seed(fx["noise_seed"])
    out, bi, mask = sampler.optimize(samples, torch.tensor(fx["sizes"]), ctx, num_timesteps=fx["steps"],
                                     noise=lambda s: torch.randn(s).cuda())
    a = ocfg.num_atom_types
    assert torch.equal(out[:, 3:3 + a].cpu(), fx["out"][:, 3:3 + a])
    relx = (out[:, :3].cpu() - fx["out"][:, :3]).abs().max().item() / fx["out"][:, :3].abs().max().item()
    assert relx < 1e-4, relx


def test_sample_sharded_on_one_gpu_equals_sample():
    """bdiff.distributed.sample_sharded (the N>1 entry point: LPT shards + one gather) with a world of one rank returns what
    GCDMSampler.sample returns for the same molecules and seed (VERDICT r1 item 3)."""
    import bdiff
    from bdiff.distributed import sample_sharded
    # tensor mode: bit-deterministic for every molecule size (parity mode's 32-edge tiles sum the pieces of rows longer than
    # 32 atoms with atomics, so two runs of a 44-atom molecule agree to ~1e-7 only)
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named("geom"), mode="tensor")
    net.load_state_dict(O.random_state_dict(O.config_named("geom"), 2), strict=True)
    net.cuda()
    sizes = torch.tensor([12, 30, 7, 44, 19])
    s = bdiff.GCDMSampler(net)
    s.sample(sizes, num_timesteps=4)                 # captures the step graph (capture advances the generator differently)
    torch.manual_seed(5)
    ref, _, _ = s.sample(sizes, num_timesteps=4)
    torch.manual_seed(5)
    out, mine = sample_sharded(s, sizes, num_timesteps=4)
    assert mine == list(range(5)) and torch.equal(out, ref)

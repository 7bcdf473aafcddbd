"""GPU: the denoiser's training pass (bdiff_train_forward / bdiff_train_backward behind torch.autograd) — SURVEY.md §8 a20.

Parity targets:
  * forward: the reference's net_out fixtures (same 5e-5 bar as the sampler's parity mode);
  * gradients: tests/golden/grad_*.pt = loss.backward() through the UNMODIFIED reference in .train() mode (fingerprints of
    every parameter tensor: L2 norm, sum, 8 strided entries), bar 2e-4 of the tensor's norm — the same bar the oracle meets;
  * gradients on larger batches: torch.autograd through the forward oracle on the CPU, every parameter, 2e-4 of max|ref|.
Plus bit-reproducibility, the one-tape guard, the TF32 option and a few optimiser steps end to end."""
import pytest
import torch

import gcpnet_oracle as O
from conftest import load_golden

pytestmark = pytest.mark.gpu


def make_net(cname, seed, scale=1.0, mode="parity"):
    import bdiff
    ocfg = O.config_named(cname)
    sd = O.random_state_dict(ocfg, seed, scale=scale)
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named(cname), mode=mode)
    net.load_state_dict(sd, strict=True)
    return net.cuda(), ocfg, sd


def relerr(a, b):
    return (a - b).abs().max().item() / max(1.0, b.abs().max().item())


@pytest.mark.parametrize("name", ["qm9_small_masked", "qm9_tiny_sizes", "qm9_cond", "geom_mixed", "geom_max181"])
def test_train_forward_matches_reference_golden(name):
    fx = load_golden(name)
    net, ocfg, sd = make_net(fx["config"], fx["weight_seed"])
    ctx = fx["context"].cuda() if fx.get("context") is not None else None
    args = (fx["batch_index"].cuda(), fx["mask"].cuda(), fx["xh"].cuda(), fx["t"].cuda(), ctx)
    out = net.denoise_train(*args)
    assert out.requires_grad and out.grad_fn is not None
    assert relerr(out.detach().cpu(), fx["net_out"]) <= 5e-5
    # the sampler kernels (fp32 parity mode) on the same inputs, same flattened parameters
    with torch.no_grad():
        inf = net.denoise(*args)
    assert relerr(out.detach(), inf) <= 2e-5
    # parameters are now views of one flat buffer and still hold the loaded values
    for k, p in net.named_parameters():
        assert torch.equal(p.detach().cpu(), sd[k]), k


@pytest.mark.parametrize("name", ["grad_qm9", "grad_geom"])
def test_gradients_match_reference_fingerprints(name):
    """loss.mean().backward() of GCDMTrainLoss == loss.backward() through the unmodified reference, every parameter."""
    import bdiff
    fx = load_golden(name)
    net, ocfg, sd = make_net(fx["config"], fx["weight_seed"], scale=fx["weight_scale"])
    tl = bdiff.GCDMTrainLoss(net, fx["histogram"])
    torch.manual_seed(fx["rng_seed"])
    loss, terms = tl(fx["batch_index"].cuda(), fx["mask"].cuda(), fx["x"].cuda(), fx["one_hot"].cuda(),
                     fx["charges"].cuda(), None, t_int=fx["terms"]["t_int"].reshape(-1, 1), noise=lambda s: torch.randn(s))
    assert loss.requires_grad
    assert torch.allclose(loss.detach().cpu(), fx["nll"], rtol=1e-4, atol=1e-3)
    loss.mean().backward()
    names = [k for k, _ in net.named_parameters()]
    assert set(names) == set(fx["grads"].keys())
    worst, worst_key = 0.0, None
    for k, p in net.named_parameters():
        assert p.grad is not None, k
        ref = fx["grads"][k]
        f = p.grad.detach().double().reshape(-1).cpu()
        scale = max(ref["norm"], 1e-12)
        err = max(abs(float(f.norm()) - ref["norm"]) / scale, abs(float(f.sum()) - ref["sum"]) / scale,
                  float((f[ref["idx"]].float() - ref["vals"]).abs().max()) / scale)
        if err > worst:
            worst, worst_key = err, k
    assert worst < 2e-4, (worst_key, worst)


def _autograd_case(cname, sizes, masked, seed=5):
    cfg = O.config_named(cname)
    g = torch.Generator().manual_seed(seed)
    bi = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
    n = bi.shape[0]
    mask = torch.ones(n, dtype=torch.bool)
    for i in masked:
        mask[i] = False
    xh = torch.randn((n, 3 + cfg.num_h), generator=g)
    t = torch.rand((len(sizes), 1), generator=g)[bi]
    ctx = torch.randn((n, cfg.num_context), generator=g) * mask[:, None] if cfg.num_context else None
    d_out = torch.randn((n, 3 + cfg.num_h), generator=g)
    return cfg, bi, mask, xh, t, ctx, d_out


@pytest.mark.parametrize("cname,sizes,masked", [("qm9", [19, 7, 12, 1, 25], [3, 30]), ("qm9_cond", [9, 14, 19], [0]),
                                                ("geom", [44, 30, 3], [50])])
def test_backward_matches_autograd_through_oracle(cname, sizes, masked):
    """The training pass (forward and every parameter's gradient) against autograd through the oracle."""
    cfg, bi, mask, xh, t, ctx, d_out = _autograd_case(cname, sizes, masked)
    net, _, sd = make_net(cname, 21, scale=0.7)
    sda = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    out_a = O.denoiser_forward(sda, cfg, bi, mask, xh, t, ctx)
    (out_a * d_out).sum().backward()
    out = net.denoise_train(bi.cuda(), mask.cuda(), xh.cuda(), t.cuda(), ctx.cuda() if ctx is not None else None)
    assert relerr(out.detach().cpu(), out_a.detach()) <= 5e-5
    (out * d_out.cuda()).sum().backward()
    worst, worst_key = 0.0, None
    for k, p in net.named_parameters():
        ref = sda[k].grad
        err = (p.grad.cpu() - ref).abs().max().item() / max(ref.abs().max().item(), 1e-12)
        if err > worst:
            worst, worst_key = err, k
    assert worst < 2e-4, (worst_key, worst)
    # a second backward pass over a fresh tape gives bit-identical gradients (no atomics anywhere), and autograd
    # accumulates: p.grad doubles
    g1 = [p.grad.clone() for p in net.parameters()]
    out2 = net.denoise_train(bi.cuda(), mask.cuda(), xh.cuda(), t.cuda(), ctx.cuda() if ctx is not None else None)
    assert torch.equal(out2.detach(), out.detach())
    (out2 * d_out.cuda()).sum().backward()
    for p, a in zip(net.parameters(), g1):
        assert torch.equal(p.grad, a + a)


def test_forward_seam_under_autograd_and_one_tape_guard():
    import bdiff
    cfg, bi, mask, xh, t, ctx, d_out = _autograd_case("qm9", [5, 9], [])
    net, _, _ = make_net("qm9", 3)

    class Bag:
        pass

    b = Bag()
    b.batch, b.mask, b.props_context, b.num_graphs = bi.cuda(), mask.cuda(), None, 2
    rb, out = net(b, xh.cuda(), t.cuda())                     # reference seam: forward(batch, xh, t) under autograd
    assert rb is b and out.grad_fn is not None
    with torch.no_grad():
        _, out_ng = net(b, xh.cuda(), t.cuda())               # sampler kernels
    assert out_ng.grad_fn is None and relerr(out.detach(), out_ng) <= 2e-5
    _, out_b = net(b, xh.cuda(), t.cuda())                    # a second tape replaces the first
    with pytest.raises(RuntimeError, match="ONE training tape"):
        out.sum().backward()
    out_b.sum().backward()
    assert all(p.grad is not None for p in net.parameters())
    # frozen parameters: no gradient requested -> sampler path, no grad_fn
    for p in net.parameters():
        p.requires_grad_(False)
    _, out_f = net(b, xh.cuda(), t.cuda())
    assert out_f.grad_fn is None


def test_tf32_gradients_close_to_fp32():
    cfg, bi, mask, xh, t, ctx, d_out = _autograd_case("geom", [30, 21], [])
    net, _, _ = make_net("geom", 4, scale=0.7)
    args = (bi.cuda(), mask.cuda(), xh.cuda(), t.cuda(), None)
    (net.denoise_train(*args) * d_out.cuda()).sum().backward()
    ref = torch.cat([p.grad.reshape(-1) for p in net.parameters()]).clone()
    for p in net.parameters():
        p.grad = None
    net.set_train_precision(tf32=True)
    (net.denoise_train(*args) * d_out.cuda()).sum().backward()
    got = torch.cat([p.grad.reshape(-1) for p in net.parameters()])
    rel = ((got - ref).norm() / ref.norm()).item()
    assert rel < 2e-2, rel
    net.set_train_precision(tf32=False)


def test_training_steps_end_to_end_reduce_the_loss():
    """GCDMTrainLoss -> backward -> GCDMTrainTail.step (clip + AdamW(amsgrad) + EMA kernels) on a fixed batch / t / noise:
    the objective goes down, the sampler kernels see the updated weights, the EMA moves."""
    import bdiff
    from bdiff.optim import GCDMTrainTail
    fx = load_golden("train_geom")
    net, ocfg, sd = make_net(fx["config"], fx["weight_seed"], scale=fx["weight_scale"])
    net.flatten_parameters()
    opt = GCDMTrainTail(net.parameters(), lr=2e-4)
    tl = bdiff.GCDMTrainLoss(net, fx["histogram"])
    batch = (fx["batch_index"].cuda(), fx["mask"].cuda(), fx["x"].cuda(), fx["one_hot"].cuda(), fx["charges"].cuda(), None)
    t_int = torch.tensor([[311], [500], [42]])

    def objective():
        torch.manual_seed(77)
        return tl(*batch, t_int=t_int, noise=lambda s: torch.randn(s))[0].mean()

    losses = []
    for _ in range(4):
        opt.zero_grad()
        loss = objective()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    with torch.no_grad():
        final = float(objective())
    assert all(l == l for l in losses) and final < losses[0], (losses, final)
    w0 = sd["interaction_layers.0.feedforward_network.0.scalar_out.2.weight"]
    p = dict(net.named_parameters())["interaction_layers.0.feedforward_network.0.scalar_out.2.weight"]
    assert not torch.equal(p.detach().cpu(), w0)
    assert p.data_ptr() == net._flat.data_ptr() + 4 * net._layout["interaction_layers.0.feedforward_network.0.scalar_out.2.weight"][0]
    assert opt.report()["step"] == 4

"""GPU: saving, resuming and converting training runs (bdiff/checkpoint.py, GCDMTrainTail.state_dict / swap_ema).

Resume and the EMA swap must be bit-exact (torch.equal).  Imports and exports are compared with torch.optim.AdamW and
TrainTailOracle at test_gpu_optim.py's tolerance (2e-6 relative on parameters and EMA)."""
import pytest
import torch

import gcpnet_oracle as O
import optim_oracle as OO
from checkpoint_synth import EMA_DECAY, layout, synth_checkpoint
from conftest import load_golden

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def deterministic_torch_ops():
    """GCDMTrainLoss sums per molecule with torch's index_add_, which accumulates with atomics on CUDA unless
    deterministic algorithms are requested; bit-exact comparisons of whole training steps need them."""
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True, warn_only=True)
    yield
    torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def fresh(cname, seed=7, scale=0.5, queue_len=50, mode="parity"):
    import bdiff
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named(cname), mode=mode)
    net.load_state_dict(O.random_state_dict(O.config_named(cname), seed, scale=scale), strict=True)
    net.cuda()
    net.flatten_parameters()
    return net, bdiff.GCDMTrainTail(net.parameters(), queue_len=queue_len)


def train_batch():
    fx = load_golden("train_qm9")
    return fx, (fx["batch_index"].cuda(), fx["mask"].cuda(), fx["x"].cuda(), fx["one_hot"].cuda(), fx["charges"].cuda(), None)


def run_steps(net, opt, k):
    import bdiff
    fx, batch = train_batch()
    tl = bdiff.GCDMTrainLoss(net, fx["histogram"])
    losses = []
    for _ in range(k):
        opt.zero_grad()
        loss = tl(*batch)[0].mean()            # t and the noise from the device generator
        loss.backward()
        opt.step()
        losses.append(loss.detach().clone())
    return losses


def snapshot(net, opt):
    sd = opt.state_dict()
    return [p.detach().clone() for p in net.parameters()], sd


def assert_runs_equal(a, b):
    (pa, sa), (pb, sb) = a, b
    assert all(torch.equal(x, y) for x, y in zip(pa, pb))
    for k in ("exp_avg", "exp_avg_sq", "max_exp_avg_sq", "ema"):
        assert all(torch.equal(x, y) for x, y in zip(sa[k], sb[k])), k
    assert torch.equal(sa["state"], sb["state"])


def test_resume_is_bit_exact(tmp_path):
    import bdiff
    torch.manual_seed(11)
    net, opt = fresh("qm9", queue_len=3)
    straight = run_steps(net, opt, 6)
    ref = snapshot(net, opt)
    ref_report = opt.report()
    assert ref_report["step"] == 6

    torch.manual_seed(11)
    net, opt = fresh("qm9", queue_len=3)
    first = run_steps(net, opt, 3)
    torch.save(bdiff.training_state(net, opt, extra={"epoch": 0}), tmp_path / "run.pt")
    del net, opt
    torch.manual_seed(999)                      # the saved generator state must win
    net, opt = fresh("qm9", seed=3, queue_len=3)
    flat, table, grads = net._flat, opt.table, [p.grad for p in net.parameters()]
    extra = bdiff.load_training_state(torch.load(tmp_path / "run.pt", weights_only=False), net, opt)
    assert extra == {"epoch": 0}
    assert net._flat is flat and opt.table is table and all(p.grad is g for p, g in zip(net.parameters(), grads))
    assert all(p.data_ptr() == flat.data_ptr() + 4 * net._layout[n][0] for n, p in net.named_parameters())
    second = run_steps(net, opt, 3)
    assert all(torch.equal(x, y) for x, y in zip(straight, first + second))
    assert_runs_equal(ref, snapshot(net, opt))
    assert opt.report() == ref_report


def test_load_rejects_mismatches_and_loads_nothing():
    import bdiff
    net, opt = fresh("geom", queue_len=3)
    sd = opt.state_dict()
    other_net, other = fresh("geom", seed=5, queue_len=4)
    before = snapshot(other_net, other)
    with pytest.raises(ValueError, match="queue_len"):
        other.load_state_dict(sd)
    with pytest.raises(ValueError, match="queue_len"):
        bdiff.load_training_state(bdiff.training_state(net, opt), other_net, other)
    assert_runs_equal(before, snapshot(other_net, other))
    bad = dict(sd, shapes=sd["shapes"][:-1])
    with pytest.raises(ValueError, match="tensors"):
        opt.load_state_dict(bad)


def _reference_ordered(cname, names, tensors):
    """Tensors in the tail's order -> CPU copies in the reference's parameters() order (dynamics only)."""
    by = dict(zip(names, tensors))
    return [by[k[len("ddpm.dynamics_network."):]].detach().cpu() for k in layout(cname)["parameters"][:-1]]


def test_import_then_one_step_matches_adamw_ema_and_oracle():
    import bdiff
    cname = "geom"
    ckpt, params = synth_checkpoint(cname, steps=3, seed=1)
    net, opt = fresh(cname, seed=2)
    bdiff.from_reference_checkpoint(ckpt, net, opt)
    names = [n for n, _ in net.named_parameters()]
    g = torch.Generator().manual_seed(8)
    grads = [torch.randn(p.shape, generator=g) * 0.01 for p in net.parameters()]

    # torch AdamW continuing the checkpoint's own state, on the reference-ordered parameters
    torch_params = [torch.nn.Parameter(p.detach().clone(), requires_grad=p.requires_grad) for p in params]
    adam = torch.optim.AdamW(torch_params, lr=1e-4, weight_decay=1e-12, amsgrad=True)
    adam.load_state_dict(ckpt["optimizer_states"][0])
    for p, gr in zip(torch_params[:-1], _reference_ordered(cname, names, grads)):
        p.grad = gr.clone()
    adam.step()
    # the oracle of the whole tail, seeded with the imported state and a fresh clip queue
    oracle = OO.TrainTailOracle(list(net.parameters()))
    sd0 = opt.state_dict()
    oracle.m = [t.cpu() for t in sd0["exp_avg"]]
    oracle.v = [t.cpu() for t in sd0["exp_avg_sq"]]
    oracle.vmax = [t.cpu() for t in sd0["max_exp_avg_sq"]]
    oracle.ema = [t.cpu() for t in sd0["ema"]]
    oracle.p = [p.detach().cpu() for p in net.parameters()]
    oracle.step_count = 3
    ema_ref = [e.clone() for e in oracle.ema]
    oracle.step(grads)

    opt.zero_grad()
    for p, gr in zip(net.parameters(), grads):
        p.grad.copy_(gr)
    opt.step()
    rep = opt.report()
    assert rep["step"] == 4 and rep["history"][-1] == 3000.0
    assert abs(rep["limit"] - oracle.last["limit"]) <= 2e-6 * oracle.last["limit"]
    got = _reference_ordered(cname, names, list(net.parameters()))
    for a, b in zip(got, torch_params[:-1]):
        assert torch.allclose(a, b.detach(), rtol=2e-6, atol=1e-8)
    for i, p in enumerate(net.parameters()):
        assert torch.allclose(p.detach().cpu(), oracle.p[i], rtol=2e-6, atol=1e-8)
        e = ema_ref[i] - (ema_ref[i] - oracle.p[i]) * (1.0 - EMA_DECAY)
        assert torch.allclose(opt.ema[i].cpu(), e, rtol=2e-6, atol=1e-8)
        assert torch.allclose(opt.ema[i].cpu(), oracle.ema[i], rtol=2e-6, atol=1e-8)


def test_export_loads_into_adamw_and_continues_alike():
    import bdiff
    cname = "geom"
    ckpt, params = synth_checkpoint(cname, steps=2, seed=3)
    net, opt = fresh(cname, seed=2)
    bdiff.from_reference_checkpoint(ckpt, net, opt)
    run_steps_geom(net, opt, 2)
    out, ema_ckpt = bdiff.to_reference_checkpoint(ckpt, net, opt, epoch=3, global_step=4)
    assert out["global_step"] == 4 and float(out["optimizer_states"][0]["state"][0]["step"]) == 4.0

    names = [n for n, _ in net.named_parameters()]
    torch_params = [torch.nn.Parameter(out["state_dict"][k].clone(), requires_grad=k != "ddpm.gamma.gamma")
                    for k in layout(cname)["parameters"]]
    adam = torch.optim.AdamW(torch_params, lr=1e-4, weight_decay=1e-12, amsgrad=True)
    adam.load_state_dict(out["optimizer_states"][0])
    g = torch.Generator().manual_seed(9)
    grads = [torch.randn(p.shape, generator=g) * 0.01 for p in net.parameters()]
    for p, gr in zip(torch_params[:-1], _reference_ordered(cname, names, grads)):
        p.grad = gr.clone()
    adam.step()
    opt.zero_grad()
    for p, gr in zip(net.parameters(), grads):
        p.grad.copy_(gr)
    opt.step()
    assert not opt.report()["clipped"]
    for a, b in zip(_reference_ordered(cname, names, list(net.parameters())), torch_params[:-1]):
        assert torch.allclose(a, b.detach(), rtol=2e-6, atol=1e-8)


def _fwd_inputs(fx):
    n = fx["x"].shape[0]
    g = torch.Generator().manual_seed(1)
    xh = torch.randn((n, 3 + fx["one_hot"].shape[1]), generator=g) * fx["mask"][:, None]
    t = torch.full((n, 1), 0.3)
    return fx["batch_index"].cuda(), fx["mask"].cuda(), xh.cuda(), t.cuda()


def test_export_companion_equals_a_net_holding_ema_parameters():
    import bdiff
    cname = "geom"
    ckpt, _ = synth_checkpoint(cname, steps=1, seed=6)     # the template only: its random weights are not trained
    net, opt = fresh(cname, seed=2)
    run_steps_geom(net, opt, 2)
    _, ema_ckpt = bdiff.to_reference_checkpoint(ckpt, net, opt)
    prefix = "ddpm.dynamics_network."
    # tensor mode: its forward is bit-identical from run to run (parity mode's is not guaranteed to be)
    companion = bdiff.GCPNetDynamicsB200(config=net.cfg, mode="tensor")
    companion.load_state_dict({k[len(prefix):]: v for k, v in ema_ckpt["state_dict"].items() if k.startswith(prefix)},
                              strict=True)
    held = bdiff.GCPNetDynamicsB200(config=net.cfg, mode="tensor")
    held.load_state_dict({n: e.cpu() for (n, _), e in zip(net.named_parameters(), opt.ema_parameters())}, strict=True)
    companion.cuda()
    held.cuda()
    fx = load_golden("train_geom")
    with torch.no_grad():
        a, b = companion.denoise(*_fwd_inputs(fx)), held.denoise(*_fwd_inputs(fx))
    assert torch.isfinite(a).all() and torch.equal(a, b)


def run_steps_geom(net, opt, k, seed=4):
    import bdiff
    fx = load_golden("train_geom")
    batch = (fx["batch_index"].cuda(), fx["mask"].cuda(), fx["x"].cuda(), fx["one_hot"].cuda(), fx["charges"].cuda(), None)
    tl = bdiff.GCDMTrainLoss(net, fx["histogram"])
    torch.manual_seed(seed)
    losses = []
    for _ in range(k):
        opt.zero_grad()
        loss = tl(*batch)[0].mean()
        loss.backward()
        opt.step()
        losses.append(loss.detach().clone())
    return losses


def test_ema_swap_is_exact_and_does_not_change_training():
    import bdiff
    cname = "geom"
    net, opt = fresh(cname, seed=2, mode="tensor")
    run_steps_geom(net, opt, 2, seed=1)
    fx = load_golden("train_geom")
    before = [p.detach().clone() for p in net.parameters()]
    ema_before = [e.clone() for e in opt.ema_parameters()]
    held = bdiff.GCPNetDynamicsB200(config=net.cfg, mode="tensor")
    held.load_state_dict({n: e.cpu() for (n, _), e in zip(net.named_parameters(), opt.ema_parameters())}, strict=True)
    held.cuda()
    with torch.no_grad():
        plain = net.denoise(*_fwd_inputs(fx))
        with opt.ema_applied():
            with pytest.raises(bdiff.BdiffError):
                opt.step()
            inside = net.denoise(*_fwd_inputs(fx))
        after = net.denoise(*_fwd_inputs(fx))
        expect = held.denoise(*_fwd_inputs(fx))
    assert torch.equal(inside, expect)
    assert torch.equal(after, plain)
    assert all(torch.equal(p.detach(), q) for p, q in zip(net.parameters(), before))
    assert all(torch.equal(e, q) for e, q in zip(opt.ema_parameters(), ema_before))
    swapped = run_steps_geom(net, opt, 2, seed=5)
    end_swapped = snapshot(net, opt)

    net2, opt2 = fresh(cname, seed=2, mode="tensor")
    run_steps_geom(net2, opt2, 2, seed=1)
    plain_losses = run_steps_geom(net2, opt2, 2, seed=5)
    assert all(torch.equal(a, b) for a, b in zip(swapped, plain_losses))
    assert_runs_equal(end_swapped, snapshot(net2, opt2))

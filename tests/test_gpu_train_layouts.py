"""The training step of the denoiser (bdiff_train_forward / bdiff_train_backward, then GCDMTrainTail) on every batch
layout of layout_catalogue.py, on batches whose shape changes from step to step, and over a short run.

Cases: every catalogue layout except `two_mids` and `mid_phases` (they exist for the megakernel's mid tiles; the training
pass has no tiles, and their float64 autograd would need 17-32 GB), plus the longest GEOM row `geom [181, 3]` and a QM9
training-size batch of 64 molecules drawn from the dataset's size histogram with about 10 % of the atoms masked.
`TRAIN_RISKS` lists what the backward can get wrong on a batch (an empty reduction when E = 0, a molecule without or with
one active atom, `act_idx` not the identity, orientation rows that cross molecule borders, long rows, every config, a
realistic batch size); a CPU test checks that the sweep reaches all of it.

Per case, net_out and every parameter's gradient of sum(net_out * d_out) are compared with torch.autograd through the
oracle in float64 (guard_empty=True, see test_gpu_tc_layouts.py): net_out within 5e-5 of max(1, |ref|max), each gradient
within 2e-4 of its max|ref|, exactly zero where the reference tensor is (the edge parameters when E = 0), all finite,
and a second forward and backward bit-identical.  Weights are the random ones of seed 21 at scale 0.7, 0.5 on rows of 128
atoms or more (the untrained network amplifies round-off with the row length) and on `SMALL_WEIGHTS`.  The oracle's own
float32 gradients miss its float64 ones by at most (worst tensor, scaled as above; measured on the CPU):

    scale 0.7   ascending_1_to_29 1.4e-5   empty_mols_qm9 8.5e-6   empty_mols_geom 4.4e-5   sparse_mask_qm9 9.1e-6
                sparse_mask_geom 4.2e-6    node_tile_edges 2.3e-6  tiny_1 8.1e-6            all_masked 7.8e-8
                cond_masked 6.1e-6         fuzz_qm9_0 2.0e-5       fuzz_qm9_1 2.8e-6        fuzz_qm9_2 3.1e-6
                fuzz_geom_0 6.4e-6         fuzz_geom_1 4.5e-5      fuzz_geom_2 2.5e-6
    scale 0.5   row_is_tile 3.2e-6         cut_1_127 5.0e-6        geom_181_3 3.0e-6        tiny_2 3.3e-6
                qm9_train_64 1.7e-5

so each stays within a quarter of the 2e-4 bar.  The worst tensor is nearly always the one-element bias of a scalar message
attention, a sum over all edges that cancels; at scale 0.7 it misses by 6.5e-5 on tiny_2 and 2.6e-4 on qm9_train_64,
which is why those two run at 0.5.  The float64 reference of a case is computed once per session (the largest take
7-15 s and 7-10 GB on the CPU).
"""
import numpy as np
import pytest
import torch

import gcpnet_oracle as O
from layout_catalogue import LAYOUTS, Layout, _inputs, _offsets, layout_paths

WEIGHT_SEED = 21
OUT_TOL = 5e-5      # net_out, as the training forward of test_gpu_train.py
GRAD_TOL = 2e-4     # every gradient tensor, of its max|ref| (test_gpu_train.py::test_backward_matches_autograd_through_oracle)
TF32_TOL = 2e-2     # relative norm of all gradients with TF32 GEMMs (test_gpu_train.py::test_tf32_gradients_close_to_fp32)


def _qm9_training_batch():
    """64 QM9 molecules drawn from the dataset's size histogram, about 10 % of the atoms masked."""
    from bdiff.datasets import QM9_N_NODES, sample_num_nodes
    sizes = [int(s) for s in sample_num_nodes(QM9_N_NODES, 64, seed=64)]
    rng = np.random.default_rng(64)
    masked = sorted(int(i) for i in np.nonzero(rng.random(sum(sizes)) < 0.1)[0])
    return Layout("qm9_train_64", "qm9", sizes, masked)


CASES = [c for c in LAYOUTS if c.name not in ("two_mids", "mid_phases")] + [
    Layout("geom_181_3", "geom", [181, 3]),
    _qm9_training_batch(),
]
BY_NAME = {c.name: c for c in CASES}

TRAIN_RISKS = {"E = 0", "E = 1", "empty molecule", "one active atom", "masked atom between active ones",
               "first or last atom of a molecule masked", "row of 129+ atoms", "config qm9", "config qm9_cond",
               "config geom", "B >= 64"}


def _edges(c: Layout) -> int:
    m, o = c.mask(), _offsets(c.sizes)
    return sum(int(m[o[k]:o[k + 1]].sum()) ** 2 for k in range(len(c.sizes)))


# cases whose float32 oracle misses the float64 one by more than a quarter of GRAD_TOL at scale 0.7 (see above)
SMALL_WEIGHTS = {"tiny_2", "qm9_train_64"}


def _scale(c: Layout) -> float:
    return 0.5 if max(c.sizes) >= 128 or c.name in SMALL_WEIGHTS else 0.7


def train_risks(c: Layout):
    """What of TRAIN_RISKS a case reaches."""
    mask, o = c.mask().numpy(), _offsets(c.sizes)
    risks = {f"config {c.config}"}
    e = _edges(c)
    if e == 0:
        risks.add("E = 0")
    if e == 1:
        risks.add("E = 1")
    if len(c.sizes) >= 64:
        risks.add("B >= 64")
    for k in range(len(c.sizes)):
        act = mask[o[k]:o[k + 1]]
        idx = np.nonzero(act)[0]
        if len(idx) == 0:
            risks.add("empty molecule")
            continue
        if len(idx) == 1 and len(act) > 1:
            risks.add("one active atom")
        if idx[-1] - idx[0] + 1 > len(idx):
            risks.add("masked atom between active ones")
        if not act[0] or not act[-1]:
            risks.add("first or last atom of a molecule masked")
        if len(idx) >= 129:
            risks.add("row of 129+ atoms")
    return risks


def test_train_sweep_reaches_every_risk():
    """CPU: the sweep reaches every backward risk class, and the QM9 training batch is what it says."""
    union = set()
    for c in CASES:
        r = train_risks(c)
        print(f"{c.name:20s} {c.config:8s} B={len(c.sizes):3d} N={c.n:5d} E={_edges(c):6d}: {', '.join(sorted(r))}")
        union |= r
    assert TRAIN_RISKS <= union, f"no case reaches {TRAIN_RISKS - union}"
    c = BY_NAME["qm9_train_64"]
    assert len(c.sizes) == 64 and 0.05 < len(c.masked) / c.n < 0.15
    assert "row cut once" in layout_paths(c.sizes, c.mask().numpy(), c.config)
    assert O.config_named("qm9_cond").num_context > 0 and _inputs(BY_NAME["cond_masked"])[4] is not None


# ------------------------------------------------------------------------------------------------ oracle
def _d_out(c: Layout) -> torch.Tensor:
    g = torch.Generator().manual_seed(7 + sum(map(ord, c.name)))
    return torch.randn((c.n, 3 + O.config_named(c.config).num_h), generator=g)


def oracle_grads(sd, config, inputs, d_out, dtype=torch.float64):
    """net_out and d sum(net_out * d_out) / d theta for every parameter, by torch.autograd through the oracle; `config`
    is a shipped configuration's name or an OracleConfig."""
    ocfg = O.config_named(config) if isinstance(config, str) else config
    leaves = {k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    out = O.denoiser_forward(leaves, ocfg, *inputs, dtype=dtype, guard_empty=True)
    grads = torch.autograd.grad(out, list(leaves.values()), d_out.to(dtype), allow_unused=True)
    return out.detach(), {k: (g if g is not None else torch.zeros_like(v)) for (k, v), g in zip(leaves.items(), grads)}


_REF = {}


def _reference(c: Layout):
    if c.name not in _REF:
        sd = O.random_state_dict(O.config_named(c.config), WEIGHT_SEED, scale=_scale(c))
        _REF[c.name] = oracle_grads(sd, c.config, _inputs(c), _d_out(c))
    return _REF[c.name]


def scaled_gradient_error(name, got, ref):
    """max|got - ref| / max|ref| of one tensor; a tensor the reference has exactly zero must be exactly zero.
    (Single entries are not held to that: on degenerate geometry, such as the two atoms of tiny_2, which the centring
    places exactly opposite each other in float64, some frame features vanish in float64 and not in float32.)"""
    got = got.detach().cpu().double()
    assert torch.isfinite(got).all(), f"{name}: non-finite gradient"
    top = ref.abs().max().item()
    if top == 0:
        bad = int((got != 0).sum())
        assert bad == 0, f"{name}: {bad} entries are nonzero where the reference gradient is exactly zero"
        return 0.0
    return (got - ref).abs().max().item() / top


def check_gradients(what, names, grads, ref_grads, tol=GRAD_TOL):
    worst, worst_key = 0.0, None
    for k, g in zip(names, grads):
        err = scaled_gradient_error(f"{what}/{k}", g, ref_grads[k])
        if err > worst:
            worst, worst_key = err, k
    print(f"{what}: worst scaled gradient error {worst:.3e} ({worst_key})")
    assert worst <= tol, f"{what}: {worst_key} scaled gradient error {worst:.3e} > {tol:.0e}"
    return worst


# ------------------------------------------------------------------------------------------------ GPU side
def _net(config, scale):
    import bdiff
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named(config), mode="parity")
    net.load_state_dict(O.random_state_dict(O.config_named(config), WEIGHT_SEED, scale=scale), strict=True)
    return net.cuda()


def _cuda_args(c: Layout):
    return tuple(a.cuda() if a is not None else None for a in _inputs(c))


def train_pass(net, args, d_out):
    """One training forward and backward: (net_out, [gradient of every parameter in named_parameters() order])."""
    out = net.denoise_train(*args)
    grads = torch.autograd.grad(out, list(net.parameters()), d_out)
    return out.detach(), [g.clone() for g in grads]


def _relerr(a, b):
    return (a.detach().cpu().double() - b).abs().max().item() / max(1.0, b.abs().max().item())


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.name for c in CASES])
def test_backward_layout_matches_fp64_autograd(name):
    c = BY_NAME[name]
    ref_out, ref_grads = _reference(c)
    net = _net(c.config, _scale(c))
    args, d_out = _cuda_args(c), _d_out(c).cuda()
    out, grads = train_pass(net, args, d_out)
    assert torch.isfinite(out).all()
    err = _relerr(out, ref_out)
    assert err <= OUT_TOL, f"{name}: net_out scaled error {err:.3e}"
    names = [k for k, _ in net.named_parameters()]
    check_gradients(name, names, grads, ref_grads)
    out2, grads2 = train_pass(net, args, d_out)
    assert torch.equal(out2, out), f"{name}: second training forward differs"
    for k, a, b in zip(names, grads, grads2):
        assert torch.equal(a, b), f"{name}/{k}: second backward differs"


@pytest.mark.gpu
def test_tf32_gradients_on_a_training_batch():
    c = BY_NAME["qm9_train_64"]
    _, ref_grads = _reference(c)
    net = _net(c.config, _scale(c))
    net.set_train_precision(tf32=True)
    _, grads = train_pass(net, _cuda_args(c), _d_out(c).cuda())
    got = torch.cat([g.reshape(-1).cpu().double() for g in grads])
    ref = torch.cat([ref_grads[k].reshape(-1) for k, _ in net.named_parameters()])
    rel = ((got - ref).norm() / ref.norm()).item()
    print(f"qm9_train_64 TF32: relative gradient norm error {rel:.3e}")
    assert rel <= TF32_TOL, rel


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["qm9", "geom"])
def test_one_net_across_changing_batch_shapes(config):
    """One net runs the largest case of its config, the others from smallest to largest, then the largest again; every
    forward and backward is bit-identical to a fresh net's on the same case (the tape layout, the arena growth and the
    re-pointed gradient slots of ensure_train would show)."""
    cases = sorted((c for c in CASES if c.config == config), key=_edges)
    order = [cases[-1]] + cases[:-1] + [cases[-1]]
    fresh = {}
    for c in cases:
        fresh[c.name] = train_pass(_net(config, 0.5), _cuda_args(c), _d_out(c).cuda())
    net = _net(config, 0.5)
    alive = []       # the plan is cached by the address of batch_index / mask: keep every input alive so none is reused
    for c in order:
        alive.append((_cuda_args(c), _d_out(c).cuda()))
        out, grads = train_pass(net, *alive[-1])
        assert torch.equal(out, fresh[c.name][0]), f"{c.name}: net_out differs after the net served other batches"
        for (k, _), a, b in zip(net.named_parameters(), grads, fresh[c.name][1]):
            assert torch.equal(a, b), f"{c.name}/{k}: gradient differs after the net served other batches"


@pytest.mark.gpu
def test_sampler_forward_between_training_forward_and_backward():
    """A sampler forward on the same batch leaves the tape alone; one on another batch re-plans, and the backward of the
    earlier training forward must refuse rather than use the new plan; a new training pass then works."""
    a, b = BY_NAME["ascending_1_to_29"], BY_NAME["empty_mols_qm9"]
    args_a, d_a, args_b = _cuda_args(a), _d_out(a).cuda(), _cuda_args(b)
    ref_out, ref_grads = train_pass(_net("qm9", 0.7), args_a, d_a)
    net = _net("qm9", 0.7)
    params = list(net.parameters())
    out = net.denoise_train(*args_a)
    with torch.no_grad():
        net.denoise(*args_a)
    grads = torch.autograd.grad(out, params, d_a)
    assert torch.equal(out.detach(), ref_out)
    for g, r in zip(grads, ref_grads):
        assert torch.equal(g, r), "a sampler forward on the same batch changed the gradients"
    out = net.denoise_train(*args_a)
    with torch.no_grad():
        net.denoise(*args_b)
    with pytest.raises(RuntimeError, match="current plan"):
        torch.autograd.grad(out, params, d_a)
    out, grads = train_pass(net, args_a, d_a)
    assert torch.equal(out, ref_out)
    for g, r in zip(grads, ref_grads):
        assert torch.equal(g, r)


def _small_batch(step):
    rng = np.random.default_rng(500 + step)
    sizes = [int(s) for s in rng.integers(1, 14, size=int(rng.integers(2, 6)))]
    masked = sorted(int(i) for i in np.nonzero(rng.random(sum(sizes)) < 0.1)[0])
    return Layout(f"step_{step}", "qm9", sizes, masked)


@pytest.mark.gpu
def test_short_training_run_teacher_forced():
    """Ten steps of training forward, backward and GCDMTrainTail.step, each on a different small batch.  Every step is
    checked on its own: the gradients against float64 autograd at the GPU's current weights, the update against
    TrainTailOracle fed the GPU's own gradients, and the sampler forward against the oracle at the updated weights.
    With the default learning rate (1e-4) a step moves net_out by 1-5 % of its scale, and the oracle's own float32
    gradients stay within 6e-6 of the float64 ones at every step (at 1e-3 the weights run away within eight steps and the
    one-element attention biases lose their accuracy)."""
    import optim_oracle as OO
    from bdiff.optim import GCDMTrainTail
    net = _net("qm9", 0.5)
    net.flatten_parameters()
    names = [k for k, _ in net.named_parameters()]
    params = list(net.parameters())
    opt = GCDMTrainTail(params)
    orc = OO.TrainTailOracle([p.detach().cpu() for p in params])
    for step in range(10):
        c = _small_batch(step)
        inputs, d_out = _inputs(c), _d_out(c)
        args = tuple(x.cuda() if x is not None else None for x in inputs)
        sd = {k: p.detach().cpu() for k, p in zip(names, params)}
        ref_out, ref_grads = oracle_grads(sd, "qm9", inputs, d_out)
        opt.zero_grad()
        out = net.denoise_train(*args)
        (out * d_out.cuda()).sum().backward()
        assert _relerr(out, ref_out) <= OUT_TOL, f"step {step}: net_out"
        grads = [p.grad.detach().cpu() for p in params]
        check_gradients(f"step {step} {c.sizes}", names, grads, ref_grads)
        opt.step()
        o = orc.step(grads)
        rep = opt.report()
        assert abs(rep["norm"] - o["norm"]) <= 2e-6 * o["norm"]
        assert abs(rep["limit"] - o["limit"]) <= 2e-6 * o["limit"]
        assert rep["clipped"] == (o["norm"] > o["limit"]) and abs(rep["coef"] - o["coef"]) <= 2e-6
        for k, p, q, e, f in zip(names, params, orc.p, opt.ema_parameters(), orc.ema):
            assert torch.allclose(p.detach().cpu(), q, rtol=2e-6, atol=1e-8), f"step {step}: parameter {k}"
            assert torch.allclose(e.cpu(), f, rtol=2e-6, atol=1e-8), f"step {step}: EMA of {k}"
        # the sampler kernels see the updated weights
        sd_new = {k: p.detach().cpu().double() for k, p in zip(names, params)}
        ref_new = O.denoiser_forward(sd_new, O.config_named("qm9"), *inputs, dtype=torch.float64, guard_empty=True)
        with torch.no_grad():
            sampled = net.denoise(*args)
        assert _relerr(sampled, ref_new) <= OUT_TOL, f"step {step}: sampler forward after the update"
        assert _relerr(out, ref_new) > 10 * OUT_TOL, f"step {step}: the update did not move net_out"
    assert opt.report()["step"] == 10

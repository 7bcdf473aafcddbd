"""The CUDA denoiser on the configurations of config_catalogue.py: the generic edge embedding, node embeddings past
K = 64, projections of up to 28 rows, 2 to 19 context columns, 1 to 64 layers, against the float64 oracle.

Per entry: parity mode on each of its layouts and tensor mode on each when the entry's (e_hidden, xi_hidden) is a
tensor pair, every molecule's x and h blocks within 5e-5 (parity) / 1e-4 (tensor) of max(1, |ref|max) of that block, as
test_gpu_tc_layouts.py; the training pass (denoise_train, bdiff_train_backward) on the entry's first layout, as
test_gpu_train_layouts.py (net_out 5e-5, each gradient 2e-4 of its max|ref|); teacher-forced reverse steps and a short
conditional chain.  The oracle runs with guard_empty=True (see test_gpu_tc_layouts.py).

The oracle's own float32 result misses its float64 one by at most (forward: worst block over the entry's layouts;
gradients: worst tensor on the training layout with the test's d_out; measured on the CPU):

    entry            scale  forward  gradient        entry            scale  forward  gradient
    hin2             0.7    2.3e-7   3.7e-6          qm9_c2           0.7    1.3e-6   3.4e-5
    hin28_e16x16     0.7    3.1e-7   1.8e-6          qm9_l1           0.7    3.0e-7   2.1e-5
    hin25_e64x4_l1   0.7    2.9e-7   2.1e-6          geom_l12         0.7    1.6e-6   3.3e-6
    e4x4_l1          0.7    2.4e-7   2.4e-6          geom_l64         0.4    9.1e-7   3.2e-5
    e32x12_c3        0.7    1.9e-7   2.6e-6          geom_hin28       0.7    9.2e-7   7.7e-6

so each stays within a quarter of its bars at the 0.7 of test_gpu_train_layouts.py, except the 64-layer entry: its
gradient gap is 1.8e-4 at 0.7 and 3e-5 .. 9e-5 at 0.5 depending on d_out (the worst tensor is a one-element attention
bias, a sum over all edges that cancels), so it runs at 0.4.
"""
import pytest
import torch

import gcpnet_oracle as O
from config_catalogue import BY_NAME, CONFIGS, ConfigCase
from layout_catalogue import BY_NAME as LAYOUTS, _active_mol_rows, _inputs, _offsets
from test_gpu_train_layouts import GRAD_TOL, OUT_TOL, check_gradients, oracle_grads, train_pass

pytestmark = pytest.mark.gpu

TENSOR_TOL = 1e-4
PARITY_TOL = 5e-5
STEP_TOL = 2e-5      # one teacher-forced reverse step at weight scale 0.5 (test_gpu_parity.py)

FORWARD = [(c.name, lay) for c in CONFIGS for lay in c.layouts]
TENSOR = [(c.name, lay) for c in CONFIGS if c.tensor for lay in c.layouts]


def _net(c: ConfigCase, mode: str, scale=None):
    import bdiff
    net = bdiff.GCPNetDynamicsB200(config=c.denoiser(), mode=mode)
    net.load_state_dict(O.random_state_dict(c.oracle(), c.seed, scale=c.scale if scale is None else scale), strict=True)
    return net.cuda()


_ORACLE = {}


def _oracle(c: ConfigCase, lay) -> torch.Tensor:
    key = (c.name, lay.name)
    if key not in _ORACLE:
        sd = O.random_state_dict(c.oracle(), c.seed, scale=c.scale)
        _ORACLE[key] = O.denoiser_forward(sd, c.oracle(), *_inputs(lay, c.oracle()), dtype=torch.float64,
                                          guard_empty=True)
    return _ORACLE[key]


def _cuda_args(c: ConfigCase, lay):
    return tuple(a.cuda() if a is not None else None for a in _inputs(lay, c.oracle()))


def _check_per_molecule(c: ConfigCase, lay, out: torch.Tensor, tol: float, what: str):
    """x and h of every molecule with an active atom against the oracle, each scaled by max(1, |ref|max) of its block."""
    ref = _oracle(c, lay)
    out = out.detach().cpu().double()
    assert out.shape == ref.shape
    assert torch.isfinite(out).all(), f"{c.name}/{lay.name}/{what}: non-finite output"
    keep, o = _active_mol_rows(lay), _offsets(lay.sizes)
    worst = (0.0, None)
    for k in range(len(lay.sizes)):
        if not keep[o[k]]:
            continue
        for blk, cols in (("x", slice(0, 3)), ("h", slice(3, None))):
            r, y = ref[o[k]:o[k + 1], cols], out[o[k]:o[k + 1], cols]
            err = (y - r).abs().max().item() / max(1.0, r.abs().max().item())
            worst = max(worst, (err, (k, blk)), key=lambda e: e[0])
    print(f"{c.name}/{lay.name}/{what}: worst per-molecule scaled error {worst[0]:.3e} at {worst[1]}")
    assert worst[0] <= tol, f"{c.name}/{lay.name}/{what}: molecule {worst[1]} scaled error {worst[0]:.3e} > {tol:.0e}"


# ------------------------------------------------------------------------------------------------ forward
@pytest.mark.parametrize("name,layout", FORWARD)
def test_parity_forward_matches_fp64_oracle(name, layout):
    c, lay = BY_NAME[name], LAYOUTS[layout]
    _check_per_molecule(c, lay, _net(c, "parity").denoise(*_cuda_args(c, lay)), PARITY_TOL, "parity")


@pytest.mark.parametrize("name,layout", TENSOR)
def test_tensor_forward_matches_fp64_oracle(name, layout):
    """k_layers_tc: within 1e-4, a rerun bit-identical, and the rows of empty molecules as parity mode has them."""
    c, lay = BY_NAME[name], LAYOUTS[layout]
    net, args = _net(c, "tensor"), _cuda_args(c, lay)
    out = net.denoise(*args)
    assert torch.equal(out, net.denoise(*args)), f"{name}/{layout}: tensor mode must be run-to-run deterministic"
    _check_per_molecule(c, lay, out, TENSOR_TOL, "tensor")
    keep = _active_mol_rows(lay).cuda()
    if not keep.all():
        par = _net(c, "parity").denoise(*args)
        d = (out[~keep] - par[~keep]).abs().max().item()
        assert torch.isfinite(par).all() and d <= TENSOR_TOL * max(1.0, par[~keep].abs().max().item()), d


# ------------------------------------------------------------------------------------------------ training
def _d_out(c: ConfigCase, lay) -> torch.Tensor:
    return torch.randn((lay.n, 3 + c.oracle().num_h), generator=torch.Generator().manual_seed(c.seed))


_REF = {}


def _train_reference(c: ConfigCase):
    if c.name not in _REF:
        lay = LAYOUTS[c.layouts[0]]
        sd = O.random_state_dict(c.oracle(), c.seed, scale=c.scale)
        _REF[c.name] = oracle_grads(sd, c.oracle(), _inputs(lay, c.oracle()), _d_out(c, lay))
    return _REF[c.name]


def _relerr(a, b):
    return (a.detach().cpu().double() - b).abs().max().item() / max(1.0, b.abs().max().item())


@pytest.mark.parametrize("name", [c.name for c in CONFIGS])
def test_training_pass_matches_fp64_autograd(name):
    c = BY_NAME[name]
    lay = LAYOUTS[c.layouts[0]]
    ref_out, ref_grads = _train_reference(c)
    net = _net(c, "parity")
    args, d_out = _cuda_args(c, lay), _d_out(c, lay).cuda()
    out, grads = train_pass(net, args, d_out)
    assert torch.isfinite(out).all()
    err = _relerr(out, ref_out)
    print(f"{name}: training net_out scaled error {err:.3e}")
    assert err <= OUT_TOL, f"{name}: net_out scaled error {err:.3e}"
    names = [k for k, _ in net.named_parameters()]
    check_gradients(name, names, grads, ref_grads)
    out2, grads2 = train_pass(net, args, d_out)
    assert torch.equal(out2, out), f"{name}: second training forward differs"
    for k, a, b in zip(names, grads, grads2):
        assert torch.equal(a, b), f"{name}/{k}: second backward differs"


def test_tf32_training_pass_on_hin28():
    """TF32 GEMMs on the widest node input.  There is no fixed bar: net_out and the relative norm of all gradients (the
    measure of test_gpu_train_layouts.py) must stay within 10x the fp32 bars.  The worst single tensor is printed; on an
    H100 SXM (700 W) it was 3.6e-3 of its max|ref| (edge embedding vector_down_frames, a 1 x 1 weight summed over all
    edges), against 3e-7 .. 3e-6 in fp32."""
    c = BY_NAME["hin28_e16x16"]
    lay = LAYOUTS[c.layouts[0]]
    ref_out, ref_grads = _train_reference(c)
    net = _net(c, "parity")
    net.set_train_precision(tf32=True)
    out, grads = train_pass(net, _cuda_args(c, lay), _d_out(c, lay).cuda())
    err = _relerr(out, ref_out)
    names = [k for k, _ in net.named_parameters()]
    worst = check_gradients(f"{c.name} TF32", names, grads, ref_grads, tol=float("inf"))
    got = torch.cat([g.reshape(-1).cpu().double() for g in grads])
    ref = torch.cat([ref_grads[k].reshape(-1) for k in names])
    rel = ((got - ref).norm() / ref.norm()).item()
    print(f"{c.name} TF32: net_out {err:.3e}, gradient norm {rel:.3e}, worst gradient tensor {worst:.3e}")
    assert err <= 10 * OUT_TOL, err
    assert rel <= 10 * GRAD_TOL, rel


# ------------------------------------------------------------------------------------------------ sampler
@pytest.mark.parametrize("name,mode,sizes", [("qm9_c2", "tensor", [19, 7, 12]), ("geom_hin28", "tensor", [30, 44]),
                                             ("e32x12_c3", "parity", [9, 14])])
def test_reverse_steps_teacher_forced_vs_oracle(name, mode, sizes):
    """As test_gpu_parity.py: every step starts from the oracle's z_t, weights at scale 0.5."""
    import bdiff
    c = BY_NAME[name]
    ocfg = c.oracle()
    sd = O.random_state_dict(ocfg, c.seed, scale=0.5)
    net = bdiff.GCPNetDynamicsB200(config=c.denoiser(), mode=mode)
    net.load_state_dict(sd, strict=True)
    net.cuda()
    steps, nmol = 5, len(sizes)
    bi = torch.repeat_interleave(torch.arange(nmol), torch.tensor(sizes))
    n = bi.shape[0]
    mask = torch.ones(n, dtype=torch.bool)
    g = torch.Generator().manual_seed(21)
    ctx = torch.randn((nmol, ocfg.num_context), generator=g)[bi] if ocfg.num_context else None
    gamma = O.gamma_table(ocfg.num_timesteps, ocfg.noise_precision, ocfg.schedule_power)
    noise = O.SeededNoise(33)
    z = O.combined_noise(noise, ocfg, bi, mask, nmol)
    sampler = bdiff.GCDMSampler(net)
    for r, s in enumerate(reversed(range(steps))):
        nx, nh = noise((n, 3)), noise((n, ocfg.num_h))
        z_next = O.reverse_step(sd, ocfg, gamma, s, s + 1, z, bi, mask, ctx, O.RecordedNoise([nx, nh]), steps, nmol)
        z_gpu = sampler.reverse_step_once(z.cuda(), r, steps, bi.cuda(), mask.cuda(), nx.cuda(), nh.cuda(),
                                          ctx.cuda() if ctx is not None else None, nmol).cpu()
        rel = (z_gpu - z_next).abs().max().item() / z_next.abs().max().item()
        print(f"{name}/{mode} step {r}: {rel:.3e}")
        assert rel < STEP_TOL, f"{name}/{mode} step {r}: rel diff {rel:.3e}"
        z = z_next


def test_conditional_chain_two_context_columns_graph_equals_eager():
    c = BY_NAME["qm9_c2"]
    net = _net(c, "tensor", scale=0.5)
    num_nodes = torch.tensor([19, 7, 12, 3])
    context = torch.randn((4, 2), generator=torch.Generator().manual_seed(3))
    outs = []
    for use_graph in (False, True):
        import bdiff
        torch.manual_seed(11)
        out, _, _, z0 = bdiff.GCDMSampler(net, use_cuda_graph=use_graph).sample(num_nodes, context=context,
                                                                                num_timesteps=4, return_z0=True)
        assert torch.isfinite(out).all() and torch.isfinite(z0).all()
        outs.append((out.clone(), z0.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])

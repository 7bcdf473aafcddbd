"""GPU tests of the tensor-core (wgmma) path = `mode="tensor"`, the mode bench.py times.

Arithmetic of that mode: every dense GEMM runs on the 5th-gen tensor cores with SPLIT-bf16 operands — activations and
weights are each the sum of two bf16 numbers (>= 16 significant bits), products evaluated as
A_hi.W_hi + A_lo.W_hi + A_hi.W_lo with fp32 accumulation — and ex2/rcp activations (~2 ulp).  Stated
tolerances (the reference's arithmetic is fp32, configs/trainer/default.yaml:15-16):
  * hardware self test vs an fp64 matmul: 3e-5 relative (plain bf16 operands: 2.4e-3);
  * one denoiser forward vs the reference golden output: max-abs <= 1e-4 * max(1, |ref|) on all six fixtures
    (parity/FFMA mode: 5e-5; the reference's own fp32-vs-fp64 floor is ~1e-6);
  * short reference chains (recorded noise): z_0 and coordinates within 1e-3 relative, identical atom types;
  * two runs of the same forward are BIT-identical (fixed-order aggregation, no floating-point atomics whose order
    matters);
  * the T=1000 chain bench.py times: per-step moments of z and the final atom-type histogram against the parity-mode
    chain on the same device noise stream (test_tensor_chain_T1000_moments).
"""
import ctypes as C

import pytest
import torch

import gcpnet_oracle as O
from conftest import load_golden

pytestmark = pytest.mark.gpu

FWD_TOL = 1e-4
CHAIN_TOL = 1e-3


@pytest.mark.parametrize("variant", [0, 2])
def test_wgmma_selftest_split_matches_fp64_matmul(variant):
    """variant 0: edge-tile layout (hi / lo A blocks, 3 products); variant 2: node-tile R5 layout (2 row views, 4 products)."""
    import bdiff
    lib = bdiff.load_library()
    g = torch.Generator().manual_seed(0)
    a = torch.randn((128, 128), generator=g).cuda()
    w = torch.randn((320, 128), generator=g).cuda()
    c = torch.zeros((128, 336), device="cuda")
    rc = lib.bdiff_selftest_split(C.c_void_p(torch.cuda.current_stream().cuda_stream), variant, C.c_void_p(a.data_ptr()),
                                  C.c_void_p(w.data_ptr()), C.c_void_p(c.data_ptr()))
    assert rc == 0
    aa = a.double()
    if variant & 2:
        aa = aa[:32].repeat(4, 1)        # every row quarter holds the complete product of the 32 rows
    ref = aa @ w.double().t()
    ref[:, 288:] = -ref[:, 288:]
    err = (c[:, :320].double() - ref).abs().max().item() / ref.abs().max().item()
    print(f"split-bf16 wgmma self test variant {variant}: rel err vs fp64 {err:.3e}")
    assert err < 3e-5, f"wgmma self test rel err {err:.3e}"
    r = torch.arange(128, device="cuda", dtype=torch.float32)[:, None] * 8 + torch.arange(8, device="cuda")[None, :]
    assert torch.equal(c[:, 320:328], 1000 + r) and torch.equal(c[:, 328:336], r)      # accumulator-scratch pair exchange


def make_net(cname, seed, mode, scale=1.0):
    import bdiff
    ocfg = O.config_named(cname)
    sd = O.random_state_dict(ocfg, seed, scale=scale)
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named(cname), mode=mode)
    net.load_state_dict(sd, strict=True)
    return net.cuda(), ocfg, sd


@pytest.mark.parametrize("name", ["qm9_small_masked", "qm9_tiny_sizes", "qm9_b4_n19", "qm9_cond", "geom_mixed",
                                  "geom_max181"])
def test_tensor_forward_matches_reference(name):
    fx = load_golden(name)
    net, ocfg, sd = make_net(fx["config"], fx["weight_seed"], "tensor")
    ctx = fx["context"].cuda() if fx["context"] is not None else None
    args = (fx["batch_index"].cuda(), fx["mask"].cuda(), fx["xh"].cuda(), fx["t"].cuda(), ctx)
    out = net.denoise(*args)
    out2 = net.denoise(*args)
    assert torch.equal(out, out2), "tensor mode must be run-to-run deterministic"
    out = out.cpu()
    ref = fx["net_out"]
    scale = max(1.0, ref.abs().max().item())
    max_abs = (out - ref).abs().max().item()
    rms = (out - ref).pow(2).mean().sqrt().item()
    print(f"{name}: tensor-mode max|diff| {max_abs:.3e}, rms {rms:.3e} (|ref|max {ref.abs().max().item():.3g})")
    assert torch.isfinite(out).all()
    assert max_abs <= FWD_TOL * scale


def test_rejected_plan_leaves_the_previous_batch_intact():
    """A batch the planner rejects (unsorted batch_index) changes no plan state: the next forward on the batch planned
    before is bit-identical to the one before the rejection."""
    import bdiff
    net, ocfg, _ = make_net("qm9", 7, "tensor")
    g = torch.Generator().manual_seed(3)
    bi = torch.repeat_interleave(torch.arange(4), torch.tensor([5, 9, 3, 19])).cuda()
    n = bi.shape[0]
    mask = torch.ones(n, dtype=torch.bool, device="cuda")
    xh = torch.randn((n, 3 + ocfg.num_h), generator=g).cuda()
    t = torch.full((n, 1), 0.5, device="cuda")
    first = net.denoise(bi, mask, xh, t)
    unsorted = bi.clone()
    unsorted[4], unsorted[5] = 1, 0
    with pytest.raises(bdiff.BdiffError, match="batch_index must be sorted"):
        net.denoise(unsorted, mask, xh, t)
    assert torch.equal(net.denoise(bi, mask, xh, t), first)


@pytest.mark.parametrize("b", [128, 300])
def test_tensor_and_parity_modes_agree_full_size(b):
    """QM9 B=128 (BASELINE config) and B=300 (more 32-node tiles than SMs): tensor mode vs parity mode on the same input,
    both on the GPU; bdiff_profile_forward fails if a dependency wait of the megakernel ever timed out."""
    g = torch.Generator().manual_seed(4)
    nat = 19
    n = b * nat
    bi = torch.repeat_interleave(torch.arange(b), torch.full((b,), nat)).cuda()
    mask = torch.ones(n, dtype=torch.bool, device="cuda")
    xh = torch.randn((n, 9), generator=g)
    _, xc = O.centralize(xh[:, :3], bi.cpu(), mask.cpu(), b)
    xh = torch.cat((xc, xh[:, 3:]), -1).cuda()
    t = torch.full((n, 1), 0.5, device="cuda")
    outs = {}
    for mode in ("parity", "tensor"):
        net, _, _ = make_net("qm9", 7, mode)
        outs[mode] = net.denoise(bi, mask, xh, t)
        if mode == "tensor":
            prof, out2 = net.profile_forward(bi, mask, xh, t)
            assert "layers_fused" in prof
            assert torch.equal(out2, outs[mode])
    d = (outs["tensor"] - outs["parity"])
    scale = max(1.0, outs["parity"].abs().max().item())
    print(f"full-size tensor vs parity: max {d.abs().max().item():.3e} rms {d.pow(2).mean().sqrt().item():.3e}")
    assert d.abs().max().item() <= FWD_TOL * scale


def test_tensor_geom_histogram_batch_matches_parity():
    """GEOM-Drugs shapes incl. rows longer than one 128-edge tile (n = 130..181: `mid` tiles) and tiny molecules."""
    sizes = torch.tensor([181, 3, 130, 44, 129, 61, 150, 12, 181, 30])
    b = len(sizes)
    g = torch.Generator().manual_seed(11)
    bi = torch.repeat_interleave(torch.arange(b), sizes).cuda()
    n = int(sizes.sum())
    mask = torch.ones(n, dtype=torch.bool, device="cuda")
    xh = torch.randn((n, 3 + 16), generator=g)
    _, xc = O.centralize(xh[:, :3], bi.cpu(), mask.cpu(), b)
    xh = torch.cat((xc, xh[:, 3:]), -1).cuda()
    t = torch.full((n, 1), 0.3, device="cuda")
    outs = {}
    for mode in ("parity", "tensor"):
        net, _, _ = make_net("geom", 3, mode)
        outs[mode] = net.denoise(bi, mask, xh, t)
        if mode == "tensor":
            assert torch.equal(net.denoise(bi, mask, xh, t), outs[mode])
    d = (outs["tensor"] - outs["parity"])
    scale = max(1.0, outs["parity"].abs().max().item())
    print(f"geom mixed sizes tensor vs parity: max {d.abs().max().item():.3e} (scale {scale:.3g})")
    assert d.abs().max().item() <= FWD_TOL * scale


@pytest.mark.parametrize("name", ["chain_qm9_T6", "chain_qm9_cond_T4", "chain_geom_T3"])
def test_tensor_chain_matches_reference_chain(name):
    """A whole sampling chain in tensor mode (CUDA-graph-free here: recorded noise) against the reference's chain with the
    same recorded noise: z_0 / coordinates within 1e-3 relative, identical argmax atom types."""
    import bdiff
    fx = load_golden(name)
    net, ocfg, sd = make_net(fx["config"], fx["weight_seed"], "tensor", scale=fx.get("weight_scale", 1.0))
    torch.manual_seed(fx["noise_seed"])
    sampler = bdiff.GCDMSampler(net)
    ctx = fx["context"].cuda() if fx["context"] is not None else None
    out, bi, mask, z0 = sampler.sample(torch.tensor(fx["sizes"]), ctx, num_timesteps=fx["steps"],
                                       noise=lambda s: torch.randn(s).cuda(), return_z0=True)
    rel = (z0.cpu() - fx["z_0"]).abs().max().item() / fx["z_0"].abs().max().item()
    a = ocfg.num_atom_types
    same = (out[:, 3:3 + a].cpu() == fx["out"][:, 3:3 + a]).all(dim=-1).float().mean().item()
    relx = (out[:, :3].cpu() - fx["out"][:, :3]).abs().max().item() / fx["out"][:, :3].abs().max().item()
    print(f"{name}: tensor chain z_0 rel {rel:.3e}, x rel {relx:.3e}, identical atom types {100 * same:.1f} %")
    assert rel < CHAIN_TOL and relx < CHAIN_TOL and same == 1.0


def test_tensor_chain_T1000_moments():
    """The chain bench.py times (QM9 unconditional, B=128 x 19 atoms, T=1000, CUDA-graph step, bench.py's seed-7 weights) in
    tensor mode against the parity-mode chain on the SAME device noise stream (same seed, same draw order).  An untrained
    denoiser amplifies round-off along the chain (SURVEY.md §8c: a 1e-6 perturbation of z_T moves final coordinates by ~1e-4
    relative) and lets |h| grow without bound, so long chains are compared through per-step moments of z (overflow-safe
    ones: mean|x|, max|x|, mean h, mean|h|) and the final atom-type histogram:
      x moments at every step within 2 % of the parity chain's; the h moments of this untrained network grow by ~17 decades
      along the chain (|h| ~ 1e17 at the end, in the reference's fp32 arithmetic too), so their per-step round-off compounds
      multiplicatively and they are compared on a log scale: |log10(tensor / parity)| <= 0.05 at every step;
      final atom-type histogram within 2 % of the atoms, everything finite, no NaN-guard hits."""
    import bdiff
    b, nat, steps = 128, 19, 1000
    sizes = torch.full((b,), nat)
    res = {}
    for mode in ("parity", "tensor"):
        net, ocfg, _ = make_net("qm9", 7, mode)
        sampler = bdiff.GCDMSampler(net)
        torch.manual_seed(123)
        out, bi, mask = sampler.sample(sizes, num_timesteps=steps, record_moments=True)
        res[mode] = (out.cpu(), sampler.last_moments.cpu().double(), sampler.nan_guard_count())
    out_p, mom_p, nan_p = res["parity"]
    out_t, mom_t, nan_t = res["tensor"]
    assert torch.isfinite(out_t).all() and torch.isfinite(mom_t).all() and torch.isfinite(mom_p).all()
    assert nan_t == 0 and nan_p == 0
    dev = (mom_t - mom_p).abs() / mom_p.abs().clamp_min(1e-2)
    worst = dev.max(dim=0)
    print(f"T=1000 moments [mean|x|, max|x|, mean h, mean|h|]: worst relative deviation per column {worst.values.tolist()} "
          f"at steps {worst.indices.tolist()}; final parity moments {mom_p[-1].tolist()}", flush=True)
    a = 5
    hist_p = out_p[:, 3:3 + a].sum(0)
    hist_t = out_t[:, 3:3 + a].sum(0)
    same = (out_p[:, 3:3 + a] == out_t[:, 3:3 + a]).all(-1).float().mean().item()
    relx = (out_t[:, :3] - out_p[:, :3]).abs().max().item() / out_p[:, :3].abs().max().item()
    print(f"atom-type histogram parity {hist_p.tolist()} tensor {hist_t.tolist()}; identical atom types {100 * same:.2f} %, "
          f"final coordinates rel diff {relx:.3e}", flush=True)
    logdev = (mom_t[:, 2:].abs().clamp_min(1e-2).log10() - mom_p[:, 2:].abs().clamp_min(1e-2).log10()).abs()
    print(f"T=1000 h moments: worst |log10 ratio| {logdev.max(dim=0).values.tolist()}", flush=True)
    assert (dev[:, :2] <= 0.02).all()
    assert (logdev <= 0.05).all()
    assert (hist_p - hist_t).abs().max().item() <= 0.02 * b * nat

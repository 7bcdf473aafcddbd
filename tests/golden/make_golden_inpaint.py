"""Generate the inpainting and chain-frame fixtures in tests/golden/ from the reference.

Build-container only: imports /root/reference through oracle/ref_shim.py.  The reference's own `inpaint` never runs
(variational_diffusion.py:1650 reads `num_denoise_steps` before assignment; :1177 indexes a [B,1] tensor with an [N]
node mask, so every jump back fails unless N == B).  Both methods are therefore re-created IN MEMORY from their own
source with exactly one asserted substring replaced each (inspect.getsource -> str.replace -> exec in the module's
globals); nothing from the reference is written anywhere, the fixtures hold only inputs and outputs.  As in
make_golden.py the weights are regenerated from `random_state_dict(cfg, 7, scale=0.5)` and only their checksum is kept.
Every molecule has at least one fixed atom, which keeps the fixtures inside the reference's domain.

Before a fixture is written, the CPU oracle (tests/inpaint_oracle.py) is run on it in fp32 and fp64: the fp32 oracle
must match the reference and the fp64-vs-fp32 gap shows that the chain is well conditioned (relative to each block's
maximum: x, one-hot/charge columns, and the frames).

Run:  python tests/golden/make_golden_inpaint.py
"""
import inspect
import os
import sys
import textwrap
import warnings

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.dirname(HERE))
warnings.filterwarnings("ignore")
import ref_shim  # noqa: E402
import gcpnet_oracle as O  # noqa: E402
import inpaint_oracle as IO  # noqa: E402
from make_golden import WEIGHT_SEED, weight_checksum  # noqa: E402

FIXES = {
    "inpaint": ("s_array_self_cond = torch.full((num_samples, 1), fill_value=0, device=z.device) / num_denoise_steps",
                "s_array_self_cond = None"),
    "sample_p_zt_given_zs": ("mu = alpha_t_given_s[node_mask] * zs", "mu = alpha_t_given_s[batch_index] * zs"),
}


def patch_reference():
    """Replace the two faulty lines of the reference in memory (see the module docstring)."""
    from src.models.components import variational_diffusion as vd
    cls = vd.EquivariantVariationalDiffusion
    for name, (old, new) in FIXES.items():
        src = textwrap.dedent(inspect.getsource(getattr(cls, name)))
        assert src.count(old) == 1, f"{name}: expected exactly one occurrence of {old!r}"
        ns = {}
        exec(compile(src.replace(old, new), f"<patched {name}>", "exec"), vd.__dict__, ns)
        setattr(cls, name, ns[name])


def ddpm_with_weights(cname, scale=0.5):
    ddpm, _ = ref_shim.build_reference_ddpm(cname, seed=0)
    cfg = O.config_named(cname)
    sd = O.random_state_dict(cfg, WEIGHT_SEED, scale=scale)
    ddpm.dynamics_network.load_state_dict(sd, strict=True)
    return ddpm, cfg, sd


def molecule_inputs(cfg, sizes, seed, fully_fixed=()):
    g = torch.Generator().manual_seed(seed)
    nmol = len(sizes)
    num_nodes = torch.tensor(sizes)
    bi = torch.repeat_interleave(torch.arange(nmol), num_nodes)
    n = bi.shape[0]
    x = torch.randn((n, 3), generator=g) * 1.5
    one_hot = torch.nn.functional.one_hot(torch.randint(0, cfg.num_atom_types, (n,), generator=g), cfg.num_atom_types).float()
    charges = torch.randint(1, 10, (n, 1), generator=g).float() if cfg.include_charges else torch.zeros((n, 0))
    fixed = torch.rand(n, generator=g) < 0.4
    off = 0
    for k, m in enumerate(sizes):
        if k in fully_fixed:
            fixed[off:off + m] = True
        elif not fixed[off:off + m].any():
            fixed[off] = True
        off += m
    ctx = torch.randn((nmol, cfg.num_context), generator=g) if cfg.num_context else None
    return dict(num_nodes=num_nodes, batch_index=bi, x=x, one_hot=one_hot, charges=charges), fixed, ctx


def blocks(cfg, out):
    a = cfg.num_atom_types
    return {"x": out[..., :3], "h": out[..., 3:]} if out.dim() == 2 else \
        {"x": out[0, :, :3], "types": out[0, :, 3:3 + a], "frames": out[1:]}


def check_oracle(cfg, sd, ref_out, run):
    """fp32 oracle vs the reference, and fp64 vs fp32 oracle, relative to each block's maximum."""
    o32 = run(sd, torch.float32)
    o64 = run({k: v.double() for k, v in sd.items()}, torch.float64)
    a = cfg.num_atom_types
    types = (slice(None), slice(3, 3 + a)) if ref_out.dim() == 2 else (0, slice(None), slice(3, 3 + a))
    assert torch.equal(o32[types], ref_out[types]), "oracle atom types differ from the reference"
    rep = {}
    for name, r in blocks(cfg, ref_out).items():
        m = max(r.abs().max().item(), 1e-30)
        rep[name] = ((blocks(cfg, o32)[name] - r).abs().max().item() / m,
                     (blocks(cfg, o64)[name].float() - blocks(cfg, o32)[name]).abs().max().item() / m)
    for name, (vs_ref, cond) in rep.items():
        print(f"    {name:7s} oracle32-vs-ref {vs_ref:.2e}  oracle64-vs-32 {cond:.2e}")
        assert vs_ref <= 1e-4 and cond <= 1e-4, name
    return rep


def seeded(seed, dtype):
    g = O.SeededNoise(seed)
    return lambda shape: g(shape).to(dtype)


def inpaint_case(cname, sizes, steps, r, j, frames, seed, fully_fixed=()):
    ddpm, cfg, sd = ddpm_with_weights(cname)
    mol, fixed, ctx = molecule_inputs(cfg, sizes, seed, fully_fixed)
    zs = []
    hook = ddpm.dynamics_network.register_forward_pre_hook(lambda m, args: zs.append(args[1].clone()))
    ref_mol = dict(mol)
    if not cfg.include_charges:
        ref_mol["charges"] = torch.zeros((mol["x"].shape[0], 1))
    torch.manual_seed(seed)
    out = ddpm.inpaint(ref_mol, fixed, num_resamplings=r, jump_length=j, return_frames=frames, num_timesteps=steps,
                       context=ctx)
    hook.remove()
    calls = len(zs)
    print(f"  {cname} r={r} j={j} T={steps} F={frames}: {calls} denoiser calls, out {tuple(out.shape)}")

    def run(sd_, dtype):
        return IO.inpaint_chain(sd_, cfg, mol["x"].to(dtype), mol["one_hot"].to(dtype), mol["charges"].to(dtype),
                                mol["num_nodes"], fixed, seeded(seed, dtype), r, j, frames, steps,
                                ctx.to(dtype) if ctx is not None else None)

    rep = check_oracle(cfg, sd, out, run)
    return dict(config=cname, sizes=list(sizes), steps=steps, num_resamplings=r, jump_length=j, return_frames=frames,
                noise_seed=seed, weight_seed=WEIGHT_SEED, weight_scale=0.5, weight_checksum=weight_checksum(sd),
                schedule=IO.repaint_schedule(r, j, steps), denoiser_calls=calls, context=ctx, node_mask_fixed=fixed,
                z_0=zs[-1], out=out.clone(), oracle_report=rep, **mol)


def chain_frames_case(cname, sizes, steps, frames, seed):
    ddpm, cfg, sd = ddpm_with_weights(cname)
    torch.manual_seed(seed)
    out, bi, mask = ddpm.mol_gen_sample(num_samples=len(sizes), num_nodes=torch.tensor(sizes), device="cpu",
                                        num_timesteps=steps, return_frames=frames)
    print(f"  {cname} mol_gen_sample T={steps} F={frames}: out {tuple(out.shape)}")

    def run(sd_, dtype):
        return IO.sample_chain_frames(sd_, cfg, torch.tensor(sizes), seeded(seed, dtype), steps, frames)

    rep = check_oracle(cfg, sd, out, run)
    return dict(config=cname, sizes=list(sizes), steps=steps, return_frames=frames, noise_seed=seed,
                weight_seed=WEIGHT_SEED, weight_scale=0.5, weight_checksum=weight_checksum(sd), out=out.clone(),
                oracle_report=rep)


def schedules_case():
    ddpm, _ = ref_shim.build_reference_ddpm("qm9", seed=0)
    table = {}
    for r in (1, 2, 3, 5, 10):
        for j in (1, 2, 3, 10):
            for T in (1, 4, 6, 10, 1000):
                table[(r, j, T)] = list(ddpm.get_repaint_schedule(r, j, T))
    return dict(schedules=table)


def main():
    only = sys.argv[1:]
    ref_shim.install()
    patch_reference()
    fixtures = {
        "inpaint_qm9_r2j2_T6": lambda: inpaint_case("qm9", [19, 7, 12], 6, 2, 2, 1, 131, fully_fixed=(1,)),
        "inpaint_qm9_cond_r3j1_T4_frames": lambda: inpaint_case("qm9_cond", [9, 14], 4, 3, 1, 2, 132),
        "inpaint_geom_r1j1_T3": lambda: inpaint_case("geom", [30, 44], 3, 1, 1, 1, 133),
        "chain_frames_qm9_T6": lambda: chain_frames_case("qm9", [19, 7, 12], 6, 3, 134),
        "repaint_schedules": schedules_case,
    }
    for name, make in fixtures.items():
        if only and name not in only:
            continue
        print(name)
        fx = make()
        path = os.path.join(HERE, name + ".pt")
        torch.save(fx, path)
        print(f"{name:34s} {os.path.getsize(path) / 1024:8.1f} KiB")


if __name__ == "__main__":
    main()

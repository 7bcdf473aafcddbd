"""CPU: the inpainting / chain-frame oracle against the reference's fixtures, the RePaint schedule and program tables of
bdiff.schedule, and the argument errors of GCDMSampler.inpaint / sample / optimize (raised before any device work)."""
import pytest
import torch

import gcpnet_oracle as O
import inpaint_oracle as IO
from conftest import load_golden

INPAINT_CASES = ["inpaint_qm9_r2j2_T6", "inpaint_qm9_cond_r3j1_T4_frames", "inpaint_geom_r1j1_T3"]


def weights(fx):
    cfg = O.config_named(fx["config"])
    sd = O.random_state_dict(cfg, fx["weight_seed"], scale=fx["weight_scale"])
    tot = sum(float(v.double().sum()) for v in sd.values())
    sq = sum(float((v.double() ** 2).sum()) for v in sd.values())
    assert torch.allclose(torch.tensor([tot, sq], dtype=torch.float64), fx["weight_checksum"]), "weight generator drifted"
    return cfg, sd


def compare(cfg, out, ref):
    """Identical atom types; every other block <= 1e-4 relative to its own maximum."""
    a = cfg.num_atom_types
    if ref.dim() == 2:
        out, ref = out.unsqueeze(0), ref.unsqueeze(0)
    assert out.shape == ref.shape
    assert torch.equal(out[0, :, 3:3 + a], ref[0, :, 3:3 + a])
    if cfg.include_charges:       # round(10 * h): may flip where |h| reaches 1e3 with these untrained weights
        rel = (out[0, :, 3 + a:] - ref[0, :, 3 + a:]).abs().max().item() / ref[0, :, 3 + a:].abs().max().item()
        assert rel <= 1e-4, f"charges rel diff {rel:.3e}"
    rel = (out[0, :, :3] - ref[0, :, :3]).abs().max().item() / ref[0, :, :3].abs().max().item()
    assert rel <= 1e-4, f"x rel diff {rel:.3e}"
    if ref.shape[0] > 1:
        rel = (out[1:] - ref[1:]).abs().max().item() / ref[1:].abs().max().item()
        assert rel <= 1e-4, f"frames rel diff {rel:.3e}"


@pytest.mark.parametrize("name", INPAINT_CASES)
def test_inpaint_oracle_matches_reference(name):
    fx = load_golden(name)
    cfg, sd = weights(fx)
    noise = O.SeededNoise(fx["noise_seed"])
    out = IO.inpaint_chain(sd, cfg, fx["x"], fx["one_hot"], fx["charges"], fx["num_nodes"], fx["node_mask_fixed"], noise,
                           fx["num_resamplings"], fx["jump_length"], fx["return_frames"], fx["steps"], fx["context"])
    compare(cfg, out, fx["out"])


def test_chain_frames_oracle_matches_reference():
    fx = load_golden("chain_frames_qm9_T6")
    cfg, sd = weights(fx)
    out = IO.sample_chain_frames(sd, cfg, torch.tensor(fx["sizes"]), O.SeededNoise(fx["noise_seed"]), fx["steps"],
                                 fx["return_frames"])
    compare(cfg, out, fx["out"])


def test_repaint_schedules_match_reference():
    from bdiff.schedule import repaint_schedule
    table = load_golden("repaint_schedules")["schedules"]
    assert len(table) == 100
    for (r, j, T), ref in table.items():
        assert repaint_schedule(r, j, T) == ref, (r, j, T)
        assert IO.repaint_schedule(r, j, T) == ref, (r, j, T)
        assert sum(ref) == T + j * (len(ref) - 1)       # every jump back re-walks jump_length steps


def _terms(g, s, t, T, model_T=1000):
    gs = g[torch.round(torch.tensor(s / T, dtype=torch.float32) * model_T).long()].double()
    gt = g[torch.round(torch.tensor(t / T, dtype=torch.float32) * model_T).long()].double()
    a2s, a2t = torch.sigmoid(-gs), torch.sigmoid(-gt)
    alpha_ts = torch.sqrt(a2t / a2s)
    return dict(alpha_ts=alpha_ts, sigma_ts=torch.sqrt(1 - alpha_ts ** 2), alpha_s=torch.sqrt(a2s),
                sigma_s=torch.sqrt(torch.sigmoid(gs)), sigma_t=torch.sqrt(torch.sigmoid(gt)))


@pytest.mark.parametrize("r,j,T,F", [(2, 2, 6, 1), (3, 1, 4, 2), (10, 10, 1000, 1), (1, 1, 50, 5), (5, 3, 10, 1)])
def test_repaint_program_tables(r, j, T, F):
    """The unrolled program against an independent walk of inpaint's loop and alpha / sigma computed in fp64."""
    from bdiff.schedule import gamma_table, repaint_program, step_coefficient_table
    g = gamma_table()
    prog = repaint_program(g, r, j, T, F)
    sched = IO.repaint_schedule(r, j, T)
    s, ops, jumps = T - 1, [], []
    for i, nd in enumerate(sched):
        for jj in range(nd):
            writes = (nd > j or i == len(sched) - 1) and (s * F) % T == 0
            ops.append((s, (s * F) // T if writes else F, jj == nd - 1 and i < len(sched) - 1))
            if ops[-1][2]:
                jumps.append((s, s + j))
                s += j
            s -= 1
    assert len(prog["jump_after"]) == len(ops) == sum(sched) and prog["num_jumps"] == len(jumps)
    assert prog["s_of_op"] == [o[0] for o in ops] and prog["jump_after"] == [o[2] for o in ops]
    assert prog["slot"].tolist() == [o[1] for o in ops]
    if F > 1:
        assert sorted(set(prog["slot"].tolist()) - {F}) == list(range(F))   # every frame is written at least once
    plain = step_coefficient_table(g, T)
    for k, (s_op, _, _) in enumerate(ops):
        assert torch.equal(prog["rev"][k], plain[T - 1 - s_op])              # gathered from the plain chain's table
        ref = _terms(g, s_op, s_op + 1, T)
        assert torch.allclose(prog["known"][k].double(), torch.stack((ref["alpha_s"], ref["sigma_s"])), rtol=1e-5, atol=1e-7)
    for k, (s_j, t_j) in enumerate(jumps):
        ref = _terms(g, s_j, t_j, T)
        assert torch.allclose(prog["jump"][k, :2].double(), torch.stack((ref["alpha_ts"], ref["sigma_ts"])), rtol=1e-4,
                              atol=1e-6)
        assert prog["jump"][k, 2].item() == pytest.approx(s_j / T) and prog["jump"][k, 3].item() == pytest.approx(t_j / T)


def test_step_coefficient_table_is_the_factored_formula():
    """step_coefficient_table is now built from transition_terms; its rows are the p(z_s | z_t) coefficients."""
    from bdiff.schedule import gamma_table, step_coefficient_table
    g = gamma_table()
    tab = step_coefficient_table(g, 20)
    for r, s in enumerate(reversed(range(20))):
        ref = _terms(g, s, s + 1, 20)
        c_eps = (1 - ref["alpha_ts"] ** 2) / ref["alpha_ts"] / ref["sigma_t"]
        sig = ref["sigma_ts"] * ref["sigma_s"] / ref["sigma_t"]
        assert torch.allclose(tab[r, :3].double(), torch.stack((ref["alpha_ts"], c_eps, sig)), rtol=1e-4, atol=1e-6)


def _cpu_sampler(cname):
    import bdiff
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named(cname))
    return bdiff.GCDMSampler(net)


def _molecule(cfg, sizes):
    nn_ = torch.tensor(sizes)
    n = int(nn_.sum())
    mol = dict(x=torch.zeros(n, 3), one_hot=torch.zeros(n, cfg.num_atom_types), num_nodes=nn_,
               batch_index=torch.repeat_interleave(torch.arange(len(sizes)), nn_))
    if cfg.include_charges:
        mol["charges"] = torch.zeros(n, 1)
    return mol, torch.zeros(n, dtype=torch.bool)


@pytest.mark.parametrize("kwargs,match", [
    (dict(num_resamplings=0), "num_resamplings"),
    (dict(jump_length=0), "jump_length"),
    (dict(num_timesteps=0), "num_timesteps"),
    (dict(return_frames=0), "return_frames"),
    (dict(return_frames=7, num_timesteps=6), "return_frames"),
    (dict(return_frames=4, num_timesteps=6), "does not divide"),
    (dict(return_frames=2, jump_length=2, num_timesteps=6), "jump_length == 1"),
])
def test_inpaint_argument_errors(kwargs, match):
    s = _cpu_sampler("qm9")
    mol, fixed = _molecule(s.cfg, [3, 4])
    with pytest.raises(ValueError, match=match):
        s.inpaint(mol, fixed, **kwargs)


def test_inpaint_shape_errors():
    s = _cpu_sampler("qm9")
    mol, fixed = _molecule(s.cfg, [3, 4])
    for key, bad in (("x", torch.zeros(7, 2)), ("one_hot", torch.zeros(7, 4)), ("charges", torch.zeros(6, 1)),
                     ("batch_index", torch.zeros(7, dtype=torch.long)), ("num_nodes", torch.tensor([3, 5]))):
        with pytest.raises(ValueError):
            s.inpaint(dict(mol, **{key: bad}), fixed, num_timesteps=2)
    for key in ("x", "charges"):
        m = dict(mol)
        del m[key]
        with pytest.raises(ValueError):
            s.inpaint(m, fixed, num_timesteps=2)
    with pytest.raises(ValueError):
        s.inpaint(mol, torch.zeros(6, dtype=torch.bool), num_timesteps=2)
    with pytest.raises(ValueError, match="context"):
        s.inpaint(mol, fixed, num_timesteps=2, context=torch.zeros(2, 1))
    sc = _cpu_sampler("qm9_cond")
    mol, fixed = _molecule(sc.cfg, [3, 4])
    with pytest.raises(ValueError, match="context"):
        sc.inpaint(mol, fixed, num_timesteps=2)
    with pytest.raises(ValueError, match="context"):
        sc.inpaint(mol, fixed, num_timesteps=2, context=torch.zeros(3, 1))


def test_inpaint_without_gpu_is_an_error_not_a_fallback():
    import bdiff
    s = _cpu_sampler("qm9")
    mol, fixed = _molecule(s.cfg, [3, 4])
    with pytest.raises(bdiff.BdiffError):
        s.inpaint(mol, fixed, num_timesteps=2)


@pytest.mark.parametrize("frames,steps", [(0, 6), (4, 6), (7, 6)])
def test_sample_and_optimize_frame_errors(frames, steps):
    s = _cpu_sampler("qm9")
    with pytest.raises(ValueError):
        s.sample(torch.tensor([3]), num_timesteps=steps, return_frames=frames)
    g = _cpu_sampler("geom")
    with pytest.raises(ValueError):
        g.optimize([(torch.zeros(3, 3), torch.zeros(3, 16))], torch.tensor([3]), num_timesteps=steps, return_frames=frames)

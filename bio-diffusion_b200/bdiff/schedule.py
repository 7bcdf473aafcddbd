"""Noise schedule of the variational diffusion process (host side, tiny).

Restates reference src/models/components/variational_diffusion.py:68-107,206-255 (polynomial schedule, gamma
lookup table) and :316-367,1219-1253 (per-step coefficients) so the sampler does not depend on the reference.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F


def gamma_table(num_timesteps: int = 1000, precision: float = 1e-5, schedule: str = "polynomial_2") -> torch.Tensor:
    """gamma[0..T] (float32), built in float64 numpy exactly like PredefinedNoiseSchedule."""
    if not schedule.startswith("polynomial"):
        raise NotImplementedError(f"noise schedule '{schedule}' (shipped configs use polynomial_2)")
    power = float(schedule.split("_")[1])
    steps = num_timesteps + 1
    x = np.linspace(0, steps, steps)
    alphas2 = (1 - np.power(x / steps, power)) ** 2
    alphas2 = np.concatenate([np.ones(1), alphas2], axis=0)
    step = np.clip(alphas2[1:] / alphas2[:-1], a_min=0.001, a_max=1.0)
    alphas2 = np.cumprod(step, axis=0)
    alphas2 = (1 - 2 * precision) * alphas2 + precision
    sigmas2 = 1 - alphas2
    return torch.tensor(-(np.log(alphas2) - np.log(sigmas2))).float()


def transition_terms(gamma: torch.Tensor, s_int: torch.Tensor, t_int: torch.Tensor, sample_steps: int) -> dict:
    """sigma / alpha terms between the grid points s_int < t_int of a `sample_steps`-step chain (float32 index tensors).

    s/sample_steps, t/sample_steps index gamma via round(t * T) (variational_diffusion.py:252-255, 1336-1339);
    sigma_and_alpha_t_given_s (:342-367), sigma (:318-323), alpha (:327-332).  All arithmetic in float32 like the
    reference.  Returns a dict of 1-D tensors: s, t, alpha_ts, sigma2_ts, sigma_ts, alpha_s, sigma_s, sigma_t.
    """
    T = gamma.shape[0] - 1
    s = s_int / sample_steps
    t = t_int / sample_steps
    g_s = gamma[torch.round(s * T).long()]
    g_t = gamma[torch.round(t * T).long()]
    sigma2_ts = -torch.expm1(F.softplus(g_s) - F.softplus(g_t))
    alpha_ts = torch.exp(0.5 * (F.logsigmoid(-g_t) - F.logsigmoid(-g_s)))
    return dict(s=s, t=t, alpha_ts=alpha_ts, sigma2_ts=sigma2_ts, sigma_ts=torch.sqrt(sigma2_ts),
                alpha_s=torch.sqrt(torch.sigmoid(-g_s)), sigma_s=torch.sqrt(torch.sigmoid(g_s)),
                sigma_t=torch.sqrt(torch.sigmoid(g_t)))


def _reverse_rows(k: dict) -> torch.Tensor:
    """{alpha_ts, c_eps, sigma, t} of p(z_s | z_t) (variational_diffusion.py:1247-1253)."""
    c_eps = k["sigma2_ts"] / k["alpha_ts"] / k["sigma_t"]
    sigma = k["sigma_ts"] * k["sigma_s"] / k["sigma_t"]
    return torch.stack((k["alpha_ts"], c_eps, sigma, k["t"]), dim=1).contiguous()


def step_coefficient_table(gamma: torch.Tensor, sample_steps: int) -> torch.Tensor:
    """Rows {alpha_ts, c_eps, sigma, t} for s = sample_steps-1 .. 0 (row r is the r-th reverse step)."""
    s_int = torch.arange(sample_steps - 1, -1, -1, dtype=torch.float32)
    return _reverse_rows(transition_terms(gamma, s_int, s_int + 1, sample_steps))


def check_frames(num_timesteps: int, return_frames: int) -> None:
    """The frame-count rule of mol_gen_sample / inpaint (variational_diffusion.py:1309-1310, 1606-1607)."""
    if not 0 < return_frames <= num_timesteps:
        raise ValueError(f"return_frames must be in [1, num_timesteps={num_timesteps}], got {return_frames}")
    if num_timesteps % return_frames:
        raise ValueError(f"return_frames={return_frames} does not divide num_timesteps={num_timesteps}")


def frame_slot(s: int, num_timesteps: int, return_frames: int) -> int:
    """Frame index written after the step that lands on grid point s (variational_diffusion.py:1353-1360), or -1."""
    return (s * return_frames) // num_timesteps if (s * return_frames) % num_timesteps == 0 else -1


def chain_frame_slots(num_timesteps: int, return_frames: int) -> torch.Tensor:
    """int64 frame slot per reverse step of a plain chain (s = T-1 .. 0); -1 maps to the dummy slot `return_frames`."""
    slots = [frame_slot(s, num_timesteps, return_frames) for s in reversed(range(num_timesteps))]
    return torch.tensor([return_frames if v < 0 else v for v in slots], dtype=torch.int64)


def repaint_schedule(resamplings: int, jump_length: int, num_timesteps: int) -> list:
    """get_repaint_schedule (variational_diffusion.py:1549-1578): denoising steps of each segment before a jump back."""
    if resamplings < 1 or jump_length < 1 or num_timesteps < 1:
        raise ValueError(f"num_resamplings, jump_length and num_timesteps must be >= 1 "
                         f"(got {resamplings}, {jump_length}, {num_timesteps})")
    curr_t, sched = 0, []
    while curr_t < num_timesteps:
        if curr_t + jump_length < num_timesteps:
            if sched:
                sched[-1] += jump_length
                sched.extend([jump_length] * (resamplings - 1))
            else:
                sched.extend([jump_length] * resamplings)
            curr_t += jump_length
        else:
            residual = num_timesteps - curr_t
            if sched:
                sched[-1] += residual
            else:
                sched.append(residual)
            curr_t += residual
    return list(reversed(sched))


def check_repaint(resamplings: int, jump_length: int, num_timesteps: int, return_frames: int) -> None:
    """The argument rules of inpaint (variational_diffusion.py:1606-1608)."""
    if resamplings < 1 or jump_length < 1 or num_timesteps < 1:
        raise ValueError(f"num_resamplings, jump_length and num_timesteps must be >= 1 "
                         f"(got {resamplings}, {jump_length}, {num_timesteps})")
    check_frames(num_timesteps, return_frames)
    if jump_length > 1 and return_frames > 1:
        raise ValueError("chain visualisation (return_frames > 1) is only defined for jump_length == 1")


def repaint_program(gamma: torch.Tensor, resamplings: int, jump_length: int, num_timesteps: int,
                    return_frames: int = 1) -> dict:
    """Unrolls the RePaint schedule of inpaint (variational_diffusion.py:1646-1751) into device-ready tables.

    Every denoise op moves z from t = s+1 to s; the last op of every segment but the final one is followed by a jump
    back from s to t = s + jump_length (after which s = t; every op ends with s -= 1).  Returns
      rev    [ops, 4]  {alpha_ts, c_eps, sigma, t} of the op's reverse step (rows of step_coefficient_table)
      known  [ops, 2]  {alpha_s, sigma_s}: z_known = alpha_s * xh0 + sigma_s * eps (:1659-1667, :910-931)
      jump   [jumps, 4] {alpha_t|s, sigma_t|s, s, t}: z_t = alpha_t|s * z_s + sigma_t|s * eps (:1730-1749, :1163-1201)
      slot   [ops] int64 frame index of the op (:1720-1728), `return_frames` = no frame (dummy slot)
      jump_after [ops] bool, s_of_op [ops] int (host-side)
    """
    check_repaint(resamplings, jump_length, num_timesteps, return_frames)
    sched = repaint_schedule(resamplings, jump_length, num_timesteps)
    s = num_timesteps - 1
    op_s, slots, jump_after, jumps = [], [], [], []
    for i, nd in enumerate(sched):
        last_seg = i == len(sched) - 1
        for jj in range(nd):
            op_s.append(s)
            slot = frame_slot(s, num_timesteps, return_frames) if (nd > jump_length or last_seg) else -1
            slots.append(return_frames if slot < 0 else slot)
            jump = jj == nd - 1 and not last_seg
            jump_after.append(jump)
            if jump:
                jumps.append((s, s + jump_length))
                s = s + jump_length
            s -= 1
    s_int = torch.tensor(op_s, dtype=torch.float32)
    k = transition_terms(gamma, s_int, s_int + 1, num_timesteps)
    # reverse-step rows are gathered from the plain chain's table, so that an op is bit-identical to sample()'s step
    rev = step_coefficient_table(gamma, num_timesteps)[num_timesteps - 1 - torch.tensor(op_s, dtype=torch.int64)]
    prog = dict(schedule=sched, s_of_op=op_s, jump_after=jump_after, rev=rev.contiguous(),
                known=torch.stack((k["alpha_s"], k["sigma_s"]), dim=1).contiguous(),
                slot=torch.tensor(slots, dtype=torch.int64))
    if jumps:
        js = torch.tensor([a for a, _ in jumps], dtype=torch.float32)
        jt = torch.tensor([b for _, b in jumps], dtype=torch.float32)
        kj = transition_terms(gamma, js, jt, num_timesteps)
        prog["jump"] = torch.stack((kj["alpha_ts"], kj["sigma_ts"], kj["s"], kj["t"]), dim=1).contiguous()
    else:
        prog["jump"] = torch.zeros((1, 4))      # never read; keeps the device pointer valid
    prog["num_jumps"] = len(jumps)
    return prog


def decode_coefficients(gamma: torch.Tensor) -> torch.Tensor:
    """{1/alpha_0, sigma_0, sigma_x, 0} for p(x,h | z_0) (variational_diffusion.py:559-577, 860-885)."""
    g0 = gamma[0]
    sigma_x = torch.exp(0.5 * g0)
    sigma_0 = torch.sqrt(torch.sigmoid(g0))
    alpha_0 = torch.sqrt(torch.sigmoid(-g0))
    return torch.stack((1.0 / alpha_0, sigma_0, sigma_x, torch.zeros(()))).contiguous()

"""CPU restatement of RePaint inpainting and of chain frames (torch, no reference import), for the tests.

Cites /root/reference/src/models/components/variational_diffusion.py.  `inpaint_chain` is
EquivariantVariationalDiffusion.inpaint (:1580-1789) with the two repairs that make it run:
  1. the dead self-conditioning line (:1650) that reads `num_denoise_steps` before assignment is dropped
     (self-conditioning is off in every shipped configuration);
  2. the jump back, sample_p_zt_given_zs (:1163-1201), takes alpha_t|s per molecule (`[batch_index]`, as sample_normal
     does with sigma at :837) where :1177 indexes it with the node mask;
and one extension: a molecule without fixed atoms is sampled freely (shift 0, no row overwritten), where the reference's
`scatter(..., reduce="mean")` without dim_size errors or zero-fills.  Builds on oracle/gcpnet_oracle.py.
"""
from __future__ import annotations

from typing import List, Optional

import torch

import gcpnet_oracle as O


def repaint_schedule(resamplings: int, jump_length: int, num_timesteps: int) -> List[int]:
    """get_repaint_schedule (:1549-1578): denoising steps per segment, in execution order."""
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


def gamma_at(cfg: O.OracleConfig, gamma: torch.Tensor, s_int: int, num_timesteps: int) -> torch.Tensor:
    """PredefinedNoiseSchedule.forward (:252-255) at s_int / num_timesteps (float32 like the reference)."""
    s = torch.tensor(s_int / num_timesteps, dtype=torch.float32)
    return gamma[torch.round(s * cfg.num_timesteps).long()]


def unnormalize_z(cfg: O.OracleConfig, z: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """unnormalize_z (:762-792) with unnormalize (:735-760)."""
    mf = mask.to(z.dtype)[:, None]
    a = cfg.num_atom_types
    parts = [z[:, :3] * cfg.norm_values[0], (z[:, 3:3 + a] * cfg.norm_values[1] + cfg.norm_biases[1]) * mf]
    if cfg.include_charges:
        parts.append((z[:, 3 + a:] * cfg.norm_values[2] + cfg.norm_biases[2]) * mf)
    return torch.cat(parts, dim=-1)


def _finish(cfg, x, h_cat, h_int, batch_index, mask, nmol, cog_fix: bool):
    if cog_fix:                                                  # CoG drift fix (:1391-1402, :1768-1778)
        tot = torch.zeros((nmol, 3), dtype=x.dtype).index_add_(0, batch_index, x)
        if tot.abs().max().item() > 5e-2:
            _, x = O.centralize(x, batch_index, mask, nmol)
    parts = [x, h_cat.to(x.dtype)] + ([h_int.to(x.dtype)] if cfg.include_charges else [])
    return torch.cat(parts, dim=-1)


def sample_chain_frames(sd, cfg: O.OracleConfig, num_nodes: torch.Tensor, randn, num_timesteps: int,
                        return_frames: int, context: Optional[torch.Tensor] = None,
                        z_init: Optional[torch.Tensor] = None) -> torch.Tensor:
    """mol_gen_sample (:1280-1412) / mol_gen_optimize (:1414-1546, with z_init) with return_frames: [F, N, D] (or
    [N, D] for F = 1).  Frame k = unnormalize_z of the latent after the step landing on s = k*T/F; frame 0 is
    overwritten by the decoded molecules; no CoG fix when F > 1."""
    T = num_timesteps
    nmol = int(num_nodes.shape[0])
    batch_index = torch.repeat_interleave(torch.arange(nmol), num_nodes)
    mask = torch.ones_like(batch_index, dtype=torch.bool)
    ctx = context[batch_index] * mask.float()[:, None] if context is not None else None
    gamma = O.gamma_table(cfg.num_timesteps, cfg.noise_precision, cfg.schedule_power)
    z = O.combined_noise(randn, cfg, batch_index, mask, nmol) if z_init is None else z_init.clone()
    out = torch.zeros((return_frames,) + tuple(z.shape), dtype=z.dtype)
    for s in reversed(range(T)):
        z = O.reverse_step(sd, cfg, gamma, s, s + 1, z, batch_index, mask, ctx, randn, T, nmol)
        if (s * return_frames) % T == 0:                         # (:1353-1360)
            out[(s * return_frames) // T] = unnormalize_z(cfg, z, mask)
    x, h_cat, h_int = O.decode_z0(sd, cfg, gamma, z, batch_index, mask, ctx, randn, nmol)
    out[0] = _finish(cfg, x, h_cat, h_int, batch_index, mask, nmol, return_frames == 1)
    return out.squeeze(0)


def centre_on_fixed(x: torch.Tensor, batch_index: torch.Tensor, fixed: torch.Tensor, nmol: int) -> torch.Tensor:
    """x minus the mean of the fixed atoms' x of its molecule (:1624-1633); 0 for a molecule without fixed atoms."""
    ff = fixed.to(x.dtype)
    tot = torch.zeros((nmol, 3), dtype=x.dtype).index_add_(0, batch_index, x * ff[:, None])
    cnt = torch.zeros(nmol, dtype=x.dtype).index_add_(0, batch_index, ff)
    return x - (tot / cnt.clamp(min=1)[:, None])[batch_index]


def known_part(cfg, xh0, alpha_s, sigma_s, batch_index, mask, nmol, randn):
    """compute_noised_representation (:910-931) with the combined noise of :795-819."""
    eps = O.combined_noise(randn, cfg, batch_index, mask, nmol)
    return alpha_s * xh0 + sigma_s * eps


def combine(z_known: torch.Tensor, z_unknown: torch.Tensor, fixed: torch.Tensor, batch_index: torch.Tensor,
            nmol: int) -> torch.Tensor:
    """Move z_known.x so that its fixed atoms share z_unknown's fixed-atom centre, then take fixed rows from z_known
    (:1694-1713).  Molecules without fixed atoms: shift 0, nothing taken from z_known."""
    ff = fixed.to(z_known.dtype)
    cnt = torch.zeros(nmol, dtype=z_known.dtype).index_add_(0, batch_index, ff).clamp(min=1)[:, None]
    com_noised = torch.zeros((nmol, 3), dtype=z_known.dtype).index_add_(0, batch_index, z_known[:, :3] * ff[:, None]) / cnt
    com_denoised = torch.zeros((nmol, 3), dtype=z_known.dtype).index_add_(0, batch_index, z_unknown[:, :3] * ff[:, None]) / cnt
    zk = z_known.clone()
    zk[:, :3] = zk[:, :3] + (com_denoised - com_noised)[batch_index]
    return torch.where(fixed[:, None], zk, z_unknown)


def renoise(cfg, z, alpha_ts, sigma_ts, batch_index, mask, nmol, randn):
    """sample_p_zt_given_zs (:1163-1201) with alpha_t|s per molecule (repair 2): alpha*z + sigma*eps, x re-centred."""
    zt = alpha_ts * z + sigma_ts * O.combined_noise(randn, cfg, batch_index, mask, nmol)
    _, zx = O.centralize(zt[:, :3], batch_index, mask, nmol)
    return torch.cat((zx, zt[:, 3:]), dim=-1)


def inpaint_chain(sd, cfg: O.OracleConfig, x: torch.Tensor, one_hot: torch.Tensor, charges: Optional[torch.Tensor],
                  num_nodes: torch.Tensor, fixed: torch.Tensor, randn, num_resamplings: int = 1, jump_length: int = 1,
                  return_frames: int = 1, num_timesteps: Optional[int] = None,
                  context: Optional[torch.Tensor] = None) -> torch.Tensor:
    """inpaint (:1580-1789) with repairs 1 and 2 and free sampling of molecules without fixed atoms.  Draw order of
    `randn`: z_T; per denoise op the known part, then the unknown part; per jump one pair; the final decode."""
    T = cfg.num_timesteps if num_timesteps is None else num_timesteps
    assert 0 < return_frames <= T and T % return_frames == 0                 # (:1606-1608)
    assert jump_length == 1 or return_frames == 1
    nmol = int(num_nodes.shape[0])
    batch_index = torch.repeat_interleave(torch.arange(nmol), num_nodes)
    mask = torch.ones_like(batch_index, dtype=torch.bool)                    # no padding mask (:1638)
    ctx = context[batch_index] if context is not None else None              # (:1614-1615)
    parts = [x, one_hot] + ([charges.reshape(-1, 1)] if cfg.include_charges else [])
    xh0 = torch.cat([p.to(x.dtype) for p in parts], dim=-1)                  # NOT normalised (:1617-1622)
    xh0 = torch.cat((centre_on_fixed(xh0[:, :3], batch_index, fixed, nmol), xh0[:, 3:]), dim=-1)
    gamma = O.gamma_table(cfg.num_timesteps, cfg.noise_precision, cfg.schedule_power)
    z = O.combined_noise(randn, cfg, batch_index, mask, nmol).to(x.dtype)   # z_T (:1635-1640)
    out = torch.zeros((return_frames,) + tuple(z.shape), dtype=z.dtype)
    s = T - 1
    sched = repaint_schedule(num_resamplings, jump_length, T)
    for i, nd in enumerate(sched):
        for jj in range(nd):
            g_s = gamma_at(cfg, gamma, s, T)
            z_known = known_part(cfg, xh0, torch.sqrt(torch.sigmoid(-g_s)), torch.sqrt(torch.sigmoid(g_s)),
                                 batch_index, mask, nmol, randn)                 # (:1659-1667)
            z_unknown = O.reverse_step(sd, cfg, gamma, s, s + 1, z, batch_index, mask, ctx, randn, T, nmol)
            z = combine(z_known, z_unknown, fixed, batch_index, nmol)        # (:1694-1713)
            if nd > jump_length or i == len(sched) - 1:                      # (:1720-1728)
                if (s * return_frames) % T == 0:
                    out[(s * return_frames) // T] = unnormalize_z(cfg, z, mask)
            if jj == nd - 1 and i < len(sched) - 1:                          # jump back (:1730-1749)
                t = s + jump_length
                g_t = gamma_at(cfg, gamma, t, T)
                a_ts, _, _ = O.step_coefficients(g_s, g_t)
                sigma_ts = torch.sqrt(-torch.expm1(torch.nn.functional.softplus(g_s) - torch.nn.functional.softplus(g_t)))
                z = renoise(cfg, z, a_ts, sigma_ts, batch_index, mask, nmol, randn)
                s = t
            s -= 1
    xo, h_cat, h_int = O.decode_z0(sd, cfg, gamma, z, batch_index, mask, ctx, randn, nmol)     # (:1753-1762)
    out[0] = _finish(cfg, xo, h_cat, h_int, batch_index, mask, nmol, return_frames == 1)
    return out.squeeze(0)

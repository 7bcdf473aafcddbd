"""CPU oracle: a functional restatement of the GCPNet denoiser + GCDM reverse-diffusion step.

TEST INFRASTRUCTURE — NOT PRODUCT CODE.  Only `tests/`, `__graft_entry__.smoke()` and
`bench.py`'s `cpu_baseline` / `--impl reference` legs may import this module, and only as the
checker (or the timed CPU baseline), never as something the product path routes through.

Parity pinning: the reference repository holds no golden vectors for this path (SURVEY.md §4), so the
oracle is pinned against the reference ITSELF: `oracle/check_against_reference.py` imports the
unmodified reference modules (under `oracle/ref_shim.py`, build container only) and compares every
stage of this restatement with them; `tests/golden/make_golden.py` stores reference outputs as
fixtures that `tests/test_oracle_golden.py` re-checks anywhere (no /root/reference needed).

Everything is plain torch on CPU tensors, written as pure functions over a `state_dict` that uses
the reference's parameter names.  `dtype` may be float32 (default, like the reference) or float64
(used to measure the fp32 round-off floor).  Citations are to files under /root/reference/.

Scope restated (SURVEY.md §8a): a2 edge index, a3 orientations, a4 edge features, a5 centralize,
a6 localize, a7 embedding, a8 GCP2, a9 scalarize, a10 safe_norm, a11 message passing, a12 interaction
layer + coordinate update, a13 projection, a16-a19 sampler step / chain / final decode.
Only the options the shipped configs select are restated (GCP2, vector_gate, no frame_gate, no
norm/dropout, residual message GCPs, scalar message attention, no self-conditioning).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------------------------
# configuration
# ----------------------------------------------------------------------------------------------
@dataclass
class OracleConfig:
    """Dims of one shipped configuration (SURVEY.md §8 table)."""
    num_atom_types: int = 5
    include_charges: bool = True
    num_context: int = 0           # len(module_cfg.conditioning)
    num_layers: int = 9            # model_cfg.num_encoder_layers
    h_hidden: int = 256
    chi_hidden: int = 32
    e_hidden: int = 64
    xi_hidden: int = 16
    bottleneck: int = 4
    num_message_layers: int = 4
    num_timesteps: int = 1000
    noise_precision: float = 1e-5
    schedule_power: float = 2.0    # "polynomial_2"
    norm_values: Tuple[float, float, float] = (1.0, 4.0, 10.0)
    norm_biases: Tuple[Optional[float], float, float] = (None, 0.0, 0.0)

    @property
    def num_h(self) -> int:        # F in xh = [x(3) | h(F)]
        return self.num_atom_types + int(self.include_charges)

    @property
    def h_in(self) -> int:         # node scalar input dim: F + time + context (gcpnet.py:947-977)
        return self.num_h + 1 + self.num_context


def config_named(name: str) -> OracleConfig:
    if name == "qm9":
        return OracleConfig()
    if name == "qm9_cond":
        return OracleConfig(num_atom_types=5, include_charges=False, num_context=1,
                            norm_values=(1.0, 8.0, 1.0))
    if name == "geom":
        return OracleConfig(num_atom_types=16, include_charges=False, num_layers=4,
                            e_hidden=16, xi_hidden=8)
    raise ValueError(name)


# ----------------------------------------------------------------------------------------------
# graph + geometry primitives
# ----------------------------------------------------------------------------------------------
def fully_connected_edge_index(batch_index: torch.Tensor, mask: Optional[torch.Tensor]) -> torch.Tensor:
    """Block-diagonal complete digraph with self loops, masked nodes dropped, (row, col)-sorted.

    Restates GCPNetDynamics.get_fully_connected_edge_index (gcpnet.py:1054-1066) without the dense
    N x N adjacency: for each molecule, every ordered pair of its unmasked atoms.  int64 [2, E].
    """
    bi = batch_index.cpu().numpy()
    keep = np.ones_like(bi, dtype=bool) if mask is None else mask.cpu().numpy().astype(bool)
    rows: List[np.ndarray] = []
    cols: List[np.ndarray] = []
    # molecule ids are sorted/contiguous on every caller of the path, but do not rely on it:
    for m in np.unique(bi):
        members = np.nonzero(bi == m)[0]          # all atoms of molecule m, ascending
        act = members[keep[members]]
        if act.size == 0:
            continue
        rows.append(np.repeat(act, act.size))
        cols.append(np.tile(act, act.size))
    if not rows:
        return torch.zeros((2, 0), dtype=torch.int64)
    r = np.concatenate(rows)
    c = np.concatenate(cols)
    order = np.lexsort((c, r))                    # torch.where(adj) enumerates row-major
    return torch.from_numpy(np.stack([r[order], c[order]]).astype(np.int64))


def _unit(v: torch.Tensor) -> torch.Tensor:
    """v / ||v|| with 0/0 -> 0 (helper.py:15-24, `_normalize`)."""
    return torch.nan_to_num(v / torch.linalg.vector_norm(v, dim=-1, keepdim=True))


def orientations(x: torch.Tensor) -> torch.Tensor:
    """chi[i] = (unit(x[i+1]-x[i]), unit(x[i-1]-x[i])) over the CONCATENATED atom list.

    protein_graph_dataset.py:217-225 via edm_dataset.py:72-74.  The neighbour may belong to another
    molecule (SURVEY.md fact 2); first/last rows get a zero vector.  [N, 2, 3].
    """
    n = x.shape[0]
    out = torch.zeros((n, 2, 3), dtype=x.dtype)
    if n > 1:
        d = x[1:] - x[:-1]
        out[:-1, 0] = _unit(d)
        out[1:, 1] = _unit(-d)
    return torch.nan_to_num(out)


def edge_features(x: torch.Tensor, ei: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """e = ||x_r - x_c||^2 [E,1];  xi = unit(x_r - x_c) [E,1,3]  (edm_dataset.py:22-38)."""
    d = x[ei[0]] - x[ei[1]]
    e = torch.nan_to_num((d * d).sum(dim=1, keepdim=True))
    xi = torch.nan_to_num(_unit(d).unsqueeze(1))
    return e, xi


def centralize(x: torch.Tensor, batch_index: torch.Tensor, mask: torch.Tensor,
               num_mols: Optional[int] = None, guard_empty: bool = False) -> Tuple[torch.Tensor, torch.Tensor]:
    """x - mask * (sum_mol x / sum_mol mask)   (components/__init__.py:46-98, edm=True branch).

    A molecule without active atoms has the centroid 0/0 = NaN, as in the reference; guard_empty=True makes it 0
    instead (what the CUDA path computes, DESIGN.md §2)."""
    b = int(batch_index.max().item()) + 1 if num_mols is None else num_mols
    mf = mask.to(x.dtype)
    cnt = torch.zeros(b, dtype=x.dtype).index_add_(0, batch_index, mf)
    tot = torch.zeros((b, x.shape[1]), dtype=x.dtype).index_add_(0, batch_index, x)
    cen = tot / (cnt.clamp(min=1) if guard_empty else cnt).unsqueeze(-1)
    return cen, x - cen[batch_index] * mf.unsqueeze(-1)


def localize(xc: torch.Tensor, ei: torch.Tensor) -> torch.Tensor:
    """Edge frames f_ij [E,3,3] = rows (d, c, d x c), d=(x_r-x_c)/(|.|+1), c=(x_r x x_c)/(|.|+1).

    components/__init__.py:123-171 with norm_x_diff=True; `ei` already holds only unmasked pairs so
    the reference's edge_mask branch is the identity.
    """
    xr, xcn = xc[ei[0]], xc[ei[1]]
    d = xr - xcn
    c = torch.linalg.cross(xr, xcn, dim=1)
    d = d / (torch.sqrt((d * d).sum(1, keepdim=True)) + 1)
    c = c / (torch.sqrt((c * c).sum(1, keepdim=True)) + 1)
    v = torch.linalg.cross(d, c, dim=1)
    return torch.stack((d, c, v), dim=1)


def safe_norm(x: torch.Tensor, dim: int) -> torch.Tensor:
    """sqrt(sum x^2 + 1e-8) + 1e-8   (components/__init__.py:276-286)."""
    return torch.sqrt((x * x).sum(dim=dim) + 1e-8) + 1e-8


def scalarize(vdf: torch.Tensor, ei: torch.Tensor, frames: torch.Tensor, node_inputs: bool,
              num_entities: int) -> torch.Tensor:
    """q[ch*3 + a] = sum_xyz frames[a, xyz] * vdf[ch, xyz]; node inputs: mean over the row's edges.

    components/__init__.py:175-219.  `vdf` is [entities, 3 channels, 3 xyz].
    """
    src = vdf[ei[0]] if node_inputs else vdf
    q = torch.einsum("eax,ecx->eca", frames, src).reshape(src.shape[0], 9)
    if not node_inputs:
        return q
    tot = torch.zeros((num_entities, 9), dtype=q.dtype).index_add_(0, ei[0], q)
    cnt = torch.zeros(num_entities, dtype=q.dtype).index_add_(0, ei[0], torch.ones(ei.shape[1], dtype=q.dtype))
    return tot / cnt.clamp(min=1).unsqueeze(-1)


# ----------------------------------------------------------------------------------------------
# GCP2 and the layers built from it
# ----------------------------------------------------------------------------------------------
def _act(name: Optional[str], x: torch.Tensor) -> torch.Tensor:
    return F.silu(x) if name == "silu" else x


def gcp2(sd: Dict[str, torch.Tensor], p: str, s: torch.Tensor, v: Optional[torch.Tensor],
         ei: torch.Tensor, frames: torch.Tensor, node_inputs: bool,
         nonlin: Tuple[Optional[str], Optional[str]], feedforward_out: bool = False,
         vector_out: bool = True) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """One geometry-complete perceptron (gcpnet.py:418-491 with :378-415, vector_gate branch).

    s [M, S_in]; v [M, V_in, 3].  Returns (s' [M, S_out], v' [M, V_out, 3] or None).
    """
    W = lambda k: sd[p + k]
    vt = v.transpose(-1, -2)                                   # [M, 3, V_in]
    hid = vt @ W("vector_down.weight").t()                     # [M, 3, hid]      (:444)
    vnorm = safe_norm(hid, dim=-2)                             # [M, hid]         (:445)
    vdf = (vt @ W("vector_down_frames.weight").t()).transpose(-1, -2)   # [M, 3ch, 3xyz] (:450-452)
    q = scalarize(vdf, ei, frames, node_inputs, s.shape[0])    # [M, 9]           (:451-458)
    merged = torch.cat((s, vnorm, q), dim=-1)                  # (:446,459)
    if feedforward_out:                                        # (:321-325)
        z = F.linear(merged, W("scalar_out.0.weight"), W("scalar_out.0.bias"))
        z = F.linear(F.silu(z), W("scalar_out.2.weight"), W("scalar_out.2.bias"))
    else:
        z = F.linear(merged, W("scalar_out.weight"), W("scalar_out.bias"))
    if not vector_out:
        return _act(nonlin[0], z), None                        # (:466-469)
    up = (hid @ W("vector_up.weight").t()).transpose(-1, -2)   # [M, V_out, 3]    (:388-391)
    gate = F.linear(_act(nonlin[1], z), W("vector_out_scale.weight"), W("vector_out_scale.bias"))
    vout = up * torch.sigmoid(gate).unsqueeze(-1)              # (:409-411)
    return _act(nonlin[0], z), vout                            # (:488-491)


def message_passing(sd, p: str, cfg: OracleConfig, h, chi, e, xi, ei, frames, taps=None):
    """GCPMessagePassing.forward (gcpnet.py:676-737): gather, 4 residual GCP2s, gate, row-sum."""
    r, c = ei[0], ei[1]
    ms = torch.cat((h[r], e, h[c]), dim=-1)                    # (:694) scalars [s_r | e | s_c]
    mv = torch.cat((chi[r], xi, chi[c]), dim=1)                # vectors [v_r | xi | v_c]
    act = ("silu", "silu")
    s, v = gcp2(sd, p + "message_fusion.0.", ms, mv, ei, frames, False, act)          # (:697)
    for k in range(1, cfg.num_message_layers):                 # (:698-701)
        ds, dv = gcp2(sd, p + f"message_fusion.{k}.", s, v, ei, frames, False, act)
        s, v = s + ds, v + dv
    attn = torch.sigmoid(F.linear(s, sd[p + "scalar_message_attention.0.weight"],
                                  sd[p + "scalar_message_attention.0.bias"]))        # (:709-711)
    s = s * attn
    if taps is not None:
        taps["msg_s"], taps["msg_v"] = s, v
    flat = torch.cat((s, v.flatten(1)), dim=-1)                # ScalarVector.flatten (:713)
    agg = torch.zeros((h.shape[0], flat.shape[1]), dtype=flat.dtype).index_add_(0, r, flat)   # (:723)
    vd = cfg.chi_hidden
    return agg[:, :-3 * vd], agg[:, -3 * vd:].reshape(-1, vd, 3)


def interaction_layer(sd, p: str, cfg: OracleConfig, h, chi, e, xi, ei, frames, mask_f, x, taps=None):
    """GCPInteractions.forward (gcpnet.py:860-930), post-norm identity, dropout identity."""
    a_s, a_v = message_passing(sd, p + "interaction.", cfg, h, chi, e, xi, ei, frames, taps)
    if taps is not None:
        taps["agg_s"], taps["agg_v"] = a_s, a_v
    fs = torch.cat((a_s, h), dim=-1)                           # (:894)
    fv = torch.cat((a_v, chi), dim=1)
    r_s, r_v = gcp2(sd, p + "feedforward_network.0.", fs, fv, ei, frames, True, (None, None),
                    feedforward_out=True)                      # (:897-904)
    h = (h + r_s) * mask_f[:, None]                            # (:907,914-915)
    chi = (chi + r_v) * mask_f[:, None, None]
    _, pv = gcp2(sd, p + "node_position_update_gcp.", h, chi, ei, frames, True, ("silu", "silu"))
    x = (x + pv[:, 0, :]) * mask_f[:, None]                    # (:852,922-928)
    return h, chi, x


def denoiser_forward(sd: Dict[str, torch.Tensor], cfg: OracleConfig, batch_index: torch.Tensor,
                     mask: torch.Tensor, xh: torch.Tensor, t: torch.Tensor,
                     context: Optional[torch.Tensor] = None, taps: Optional[dict] = None,
                     dtype=torch.float32, guard_empty: bool = False) -> torch.Tensor:
    """GCPNetDynamics.atom_types_and_coords_forward (gcpnet.py:1069-1232) -> net_out [N, 3+F].

    guard_empty: see `centralize`.  Without it, a molecule with no active atoms gets NaN coordinate rows, and the NaN guard
    below then zeroes the velocity of every molecule in the batch (the reference's behaviour)."""
    sd = {k: v.to(dtype) for k, v in sd.items()}
    mask_f = mask.to(dtype)
    xh = xh.to(dtype) * mask_f[:, None]                        # (:1081)
    x_init, h_in = xh[:, :3], xh[:, 3:]
    ei = fully_connected_edge_index(batch_index, mask)         # (:1096-1099)
    chi_in = orientations(x_init)                              # (:1105)
    e_in, xi_in = edge_features(x_init, ei)                    # (:1109) un-centred x
    h_in = torch.cat((h_in, t.to(dtype).reshape(-1, 1)), dim=-1)        # (:1142-1150)
    if cfg.num_context:
        h_in = torch.cat((h_in, context.to(dtype).reshape(xh.shape[0], cfg.num_context)), dim=-1)
    nmol = int(batch_index.max().item()) + 1
    _, x = centralize(x_init, batch_index, mask, nmol, guard_empty)     # (:1160-1166)
    frames = localize(x, ei)                                   # (:1169-1174) frozen across layers
    # embedding (gcpnet.py:551-603): edge GCP2 silu/silu, node GCP2 no activation
    e, xi = gcp2(sd, "gcp_embedding.edge_embedding.", e_in, xi_in, ei, frames, False, ("silu", "silu"))
    h, chi = gcp2(sd, "gcp_embedding.node_embedding.", h_in, chi_in, ei, frames, True, (None, None))
    if taps is not None:
        taps.update(edge_index=ei, chi_in=chi_in, e_in=e_in, xi_in=xi_in, x_centered=x, f_ij=frames,
                    e=e, xi=xi, h0=h, chi0=chi, layers=[])
    for l in range(cfg.num_layers):                            # (:1180-1188)
        lt = {} if taps is not None else None
        h, chi, x = interaction_layer(sd, f"interaction_layers.{l}.", cfg, h, chi, e, xi, ei, frames,
                                      mask_f, x, lt)
        if taps is not None:
            lt.update(h=h, chi=chi, x=x)
            taps["layers"].append(lt)
    hp, _ = gcp2(sd, "scalar_node_projection_gcp.", h, chi, ei, frames, True, (None, None),
                 vector_out=False)                             # (:1191-1197)
    vel = (x - x_init) * mask_f[:, None]                       # (:1204)
    h_final = hp[:, :cfg.num_h]                                # (:1208-1211) strip ctx + time
    if torch.isnan(vel).any():                                 # (:1214-1216)
        vel = torch.zeros_like(vel)
    _, vel = centralize(vel, batch_index, mask, nmol, guard_empty)      # (:1219-1227)
    return torch.cat((vel, h_final), dim=-1)                   # (:1230)


# ----------------------------------------------------------------------------------------------
# diffusion schedule and the reverse step
# ----------------------------------------------------------------------------------------------
def gamma_table(num_timesteps: int = 1000, precision: float = 1e-5, power: float = 2.0) -> torch.Tensor:
    """gamma[0..T] as float32, built in float64 numpy like the reference.

    variational_diffusion.py:88-107 (polynomial_schedule), :68-84 (clip_noise_schedule),
    :206-250 (PredefinedNoiseSchedule).
    """
    steps = num_timesteps + 1
    x = np.linspace(0, steps, steps)
    a2 = (1 - np.power(x / steps, power)) ** 2
    a2 = np.concatenate([np.ones(1), a2])
    ratio = np.clip(a2[1:] / a2[:-1], 0.001, 1.0)
    a2 = np.cumprod(ratio)
    a2 = (1 - 2 * precision) * a2 + precision
    g = -(np.log(a2) - np.log(1 - a2))
    return torch.tensor(g).float()


def step_coefficients(gamma_s: torch.Tensor, gamma_t: torch.Tensor):
    """(1/alpha_ts, sigma2_ts/alpha_ts/sigma_t, sigma_ts*sigma_s/sigma_t) for p(z_s | z_t).

    variational_diffusion.py:342-367 (sigma_and_alpha_t_given_s), :318-332, :1247-1253.
    """
    sigma2_ts = -torch.expm1(F.softplus(gamma_s) - F.softplus(gamma_t))
    alpha_ts = torch.exp(0.5 * (F.logsigmoid(-gamma_t) - F.logsigmoid(-gamma_s)))
    sigma_ts = torch.sqrt(sigma2_ts)
    sigma_s = torch.sqrt(torch.sigmoid(gamma_s))
    sigma_t = torch.sqrt(torch.sigmoid(gamma_t))
    return alpha_ts, sigma2_ts / alpha_ts / sigma_t, sigma_ts * sigma_s / sigma_t


NoiseFn = Callable[[Tuple[int, int]], torch.Tensor]


def combined_noise(randn: NoiseFn, cfg: OracleConfig, batch_index, mask, nmol) -> torch.Tensor:
    """randn(N,3) -> mask -> centre ; randn(N,F) -> mask   (variational_diffusion.py:795-819,400-440).

    The two draws happen in exactly this order; `randn` is the injected generator.
    """
    n = batch_index.shape[0]
    mf = mask.float()
    zx = randn((n, 3)) * mf[:, None]
    _, zx = centralize(zx, batch_index, mask, nmol)
    zh = randn((n, cfg.num_h)) * mf[:, None]
    return torch.cat((zx, zh), dim=-1)


def reverse_step(sd, cfg: OracleConfig, gamma: torch.Tensor, s_int: int, t_int: int, z: torch.Tensor,
                 batch_index, mask, context, randn: NoiseFn, num_timesteps: int, nmol: int) -> torch.Tensor:
    """sample_p_zs_given_zt (variational_diffusion.py:1204-1278)."""
    s = torch.tensor(s_int / num_timesteps, dtype=torch.float32)
    t = torch.tensor(t_int / num_timesteps, dtype=torch.float32)
    g_s = gamma[torch.round(s * cfg.num_timesteps).long()]      # PredefinedNoiseSchedule.forward :252-255
    g_t = gamma[torch.round(t * cfg.num_timesteps).long()]
    a_ts, c_eps, sig = step_coefficients(g_s, g_t)
    t_nodes = t.expand(z.shape[0], 1)
    eps_hat = denoiser_forward(sd, cfg, batch_index, mask, z, t_nodes, context)
    mu = z / a_ts - c_eps * eps_hat                             # (:1247-1250)
    zs = mu + sig * combined_noise(randn, cfg, batch_index, mask, nmol)   # (:1256-1263, :822-837)
    _, zx = centralize(zs[:, :3], batch_index, mask, nmol)      # (:1266-1272)
    return torch.cat((zx, zs[:, 3:]), dim=-1)


def decode_z0(sd, cfg: OracleConfig, gamma, z0, batch_index, mask, context, randn: NoiseFn, nmol: int):
    """sample_p_xh_given_z0 (variational_diffusion.py:840-907) + unnormalize (:735-760).

    Returns (x [N,3] float, h_cat one-hot int64 [N,A], h_int int64 [N,1 or 0]).
    """
    g0 = gamma[0]
    sigma_x = torch.exp(0.5 * g0)                               # SNR(-0.5*gamma_0) (:864)
    t0 = torch.zeros((z0.shape[0], 1))
    eps_hat = denoiser_forward(sd, cfg, batch_index, mask, z0, t0, context)
    sigma_0 = torch.sqrt(torch.sigmoid(g0))
    alpha_0 = torch.sqrt(torch.sigmoid(-g0))
    mu = 1.0 / alpha_0 * (z0 - sigma_0 * eps_hat)              # compute_x_pred (:559-577)
    xh = mu + sigma_x * combined_noise(randn, cfg, batch_index, mask, nmol)
    mf = mask.float()
    x = xh[:, :3] * cfg.norm_values[0]
    a = cfg.num_atom_types
    h_cat = (xh[:, 3:3 + a] * cfg.norm_values[1] + cfg.norm_biases[1]) * mf[:, None]
    h_cat = F.one_hot(torch.argmax(h_cat, dim=-1), a) * mask.long()[:, None]
    if cfg.include_charges:
        h_int = (xh[:, 3 + a:] * cfg.norm_values[2] + cfg.norm_biases[2]) * mf[:, None]
        h_int = torch.round(h_int).long() * mask.long()[:, None]
    else:
        h_int = torch.zeros((xh.shape[0], 0), dtype=torch.int64)
    return x, h_cat, h_int


def sample_chain(sd, cfg: OracleConfig, num_nodes: torch.Tensor, randn: NoiseFn,
                 num_timesteps: Optional[int] = None, context: Optional[torch.Tensor] = None,
                 mask: Optional[torch.Tensor] = None, return_z0: bool = False, z_init: Optional[torch.Tensor] = None):
    """mol_gen_sample (variational_diffusion.py:1280-1412), return_frames=1, no self-conditioning.

    With `z_init` (normalised [x | one-hot], see `normalize_samples`) this is mol_gen_optimize (:1414-1546,
    norm_with_original_timesteps=False): the same loop started from existing samples instead of z_T ~ N(0, I) — no
    initial noise draw, everything else (time grid s/num_timesteps, per-step noise order, final decode, CoG fix) equal.
    Returns (out [N, 3+A(+1)], batch_index, mask)  (and z_0 when asked).
    """
    T = cfg.num_timesteps if num_timesteps is None else num_timesteps
    nmol = int(num_nodes.shape[0])
    batch_index = torch.repeat_interleave(torch.arange(nmol), num_nodes)
    mask = torch.ones_like(batch_index, dtype=torch.bool) if mask is None else mask
    ctx = None
    if context is not None:                                      # (:1316-1320)
        ctx = context[batch_index] * mask.float()[:, None]
    gamma = gamma_table(cfg.num_timesteps, cfg.noise_precision, cfg.schedule_power)
    z = combined_noise(randn, cfg, batch_index, mask, nmol) if z_init is None else z_init.clone()      # p(z_T) / samples
    for s in reversed(range(T)):                                 # (:1335-1351)
        z = reverse_step(sd, cfg, gamma, s, s + 1, z, batch_index, mask, ctx, randn, T, nmol)
    x, h_cat, h_int = decode_z0(sd, cfg, gamma, z, batch_index, mask, ctx, randn, nmol)
    tot = torch.zeros((nmol, 3)).index_add_(0, batch_index, x)   # CoG drift fix (:1391-1402)
    if tot.abs().max().item() > 5e-2:
        _, x = centralize(x, batch_index, mask, nmol)
    parts = [x, h_cat.float()] + ([h_int.float()] if cfg.include_charges else [])
    out = torch.cat(parts, dim=-1)
    return (out, batch_index, mask, z) if return_z0 else (out, batch_index, mask)


def normalize_samples(cfg: OracleConfig, x: torch.Tensor, one_hot: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """The input side of mol_gen_optimize (:1456-1464): normalize (:702-732) x and the categorical features, stack."""
    mf = mask.float()[:, None]
    return torch.cat((x / cfg.norm_values[0] * mf, (one_hot.float() - cfg.norm_biases[1]) / cfg.norm_values[1] * mf), dim=-1)


# ----------------------------------------------------------------------------------------------
# helpers shared by tests / bench
# ----------------------------------------------------------------------------------------------
def param_shapes(cfg: OracleConfig) -> Dict[str, Tuple[int, ...]]:
    """Reference parameter names -> shapes (== GCPNetDynamics.named_parameters(), gcpnet.py:933-1039)."""
    sh: Dict[str, Tuple[int, ...]] = {}

    def gcp(p, s_in, v_in, s_out, v_out, bott, ff=False):
        hid = v_in // bott if bott > 1 else max(v_in, v_out)
        sh[p + "vector_down.weight"] = (hid, v_in)
        fan = hid + s_in + 9
        if ff:
            sh[p + "scalar_out.0.weight"] = (s_out, fan); sh[p + "scalar_out.0.bias"] = (s_out,)
            sh[p + "scalar_out.2.weight"] = (s_out, s_out); sh[p + "scalar_out.2.bias"] = (s_out,)
        else:
            sh[p + "scalar_out.weight"] = (s_out, fan); sh[p + "scalar_out.bias"] = (s_out,)
        sh[p + "vector_down_frames.weight"] = (3, v_in)
        if v_out:
            sh[p + "vector_up.weight"] = (v_out, hid)
            sh[p + "vector_out_scale.weight"] = (v_out, s_out); sh[p + "vector_out_scale.bias"] = (v_out,)

    H, C, E, X, b = cfg.h_hidden, cfg.chi_hidden, cfg.e_hidden, cfg.xi_hidden, cfg.bottleneck
    gcp("gcp_embedding.edge_embedding.", 1, 1, E, X, 1)
    gcp("gcp_embedding.node_embedding.", cfg.h_in, 2, H, C, 1)
    for l in range(cfg.num_layers):
        p = f"interaction_layers.{l}."
        gcp(p + "interaction.message_fusion.0.", 2 * H + E, 2 * C + X, H, C, b)
        for k in range(1, cfg.num_message_layers):
            gcp(p + f"interaction.message_fusion.{k}.", H, C, H, C, b)
        sh[p + "interaction.scalar_message_attention.0.weight"] = (1, H)
        sh[p + "interaction.scalar_message_attention.0.bias"] = (1,)
        gcp(p + "feedforward_network.0.", 2 * H, 2 * C, H, C, b, ff=True)
        gcp(p + "node_position_update_gcp.", H, C, H, 1, b)
    gcp("scalar_node_projection_gcp.", H, C, cfg.h_in, 0, 1)
    return sh


def random_state_dict(cfg: OracleConfig, seed: int = 0, scale: float = 1.0) -> Dict[str, torch.Tensor]:
    """Seeded weights with nn.Linear-style U(-1/sqrt(fan_in), 1/sqrt(fan_in)) ranges.

    NOT bit-identical to the reference's default init (different draw order); used where only the
    shapes and magnitudes matter (bench, smoke, full-size property tests).
    """
    g = torch.Generator().manual_seed(seed)
    sd = {}
    shapes = param_shapes(cfg)
    for name, shape in shapes.items():
        fan_in = shape[1] if len(shape) == 2 else None
        if fan_in is None:      # bias: bound by the matching weight's fan-in
            wname = name[:-4] + "weight"
            fan_in = shapes[wname][1]
        bound = scale / math.sqrt(fan_in)
        sd[name] = (torch.rand(shape, generator=g) * 2 - 1) * bound
    return sd


class SeededNoise:
    """randn provider drawing from one torch.Generator in call order (CPU)."""

    def __init__(self, seed: int):
        self.g = torch.Generator().manual_seed(seed)

    def __call__(self, shape):
        return torch.randn(shape, generator=self.g)


class RecordedNoise:
    """randn provider replaying a recorded list of tensors (so CPU oracle and GPU path share noise)."""

    def __init__(self, tensors: List[torch.Tensor]):
        self.tensors = list(tensors)
        self.i = 0

    def __call__(self, shape):
        t = self.tensors[self.i]
        self.i += 1
        assert tuple(t.shape) == tuple(shape), (t.shape, shape)
        return t


# ----------------------------------------------------------------------------------------------
# evaluation NLL (forward only): the loss terms of EquivariantVariationalDiffusion in eval mode
# ----------------------------------------------------------------------------------------------
def _cdf_std_gaussian(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2)))            # variational_diffusion.py:395-396


def eval_nll(sd, cfg: OracleConfig, batch_index: torch.Tensor, mask: torch.Tensor, x: torch.Tensor,
             one_hot: torch.Tensor, charges: torch.Tensor, context: Optional[torch.Tensor],
             n_nodes_hist: Dict[int, int], randn: NoiseFn, t_int: Optional[torch.Tensor] = None,
             denoise: Optional[Callable] = None, training: bool = False, norm_training_by_max_nodes: bool = False):
    """NLL per molecule in evaluation mode (two denoiser calls) + its terms; with `training=True` the training-mode
    L2 objective instead (ONE denoiser call; variational_diffusion.py:979-980,985,1054-1055,1068-1069,1083-1103 and the
    training branch of the Lightning assembly, qm9_mol_gen_ddpm.py:232-245; loss_type "l2" as shipped): t_int ~
    randint(0, T+1), delta_log_px = 0, SNR weight 1, no constants, L0 from (z_t, eps_t, net_out, gamma_t) masked by
    t == 0, error_t masked by t != 0, both normalised by (3 + F) * n.

    Restates EquivariantVariationalDiffusion.atom_types_and_coords_forward with self.training == False
    (variational_diffusion.py:955-1160: normalize :702-732, compute_noised_representation :910-931,
    compute_kl_prior :501-556, log_pxh_given_z0_without_constants :598-699, log_constants_p_x_given_z0 :579-595,
    delta_log_px :950-952, log_pN :932-940) and the evaluation branch of the Lightning module's assembly
    (qm9_mol_gen_ddpm.py:184-262).  `x` must already be CoG-free (the module centralises first, :196-202).
    RNG order: t_int ~ randint(1, T+1) [unless given], then randn(N,3), randn(N,F) for z_t, then again for z_0.
    `denoise(batch_index, mask, z, t_nodes, context)` defaults to the oracle denoiser.
    """
    T = cfg.num_timesteps
    nmol = int(batch_index.max().item()) + 1
    mf = mask.float()
    gamma = gamma_table(T, cfg.noise_precision, cfg.schedule_power)
    if denoise is None:
        denoise = lambda bi, mk, z, tn, ctx: denoiser_forward(sd, cfg, bi, mk, z, tn, ctx)
    # normalize (:702-732)
    xn = x / cfg.norm_values[0]
    h_cat = (one_hot.float() - cfg.norm_biases[1]) / cfg.norm_values[1] * mf[:, None]
    h_int = (charges.float() - cfg.norm_biases[2]) / cfg.norm_values[2]
    if cfg.include_charges:
        h_int = h_int * mf.reshape(h_int.shape[0], *([1] * (h_int.dim() - 1)))
    num_nodes = torch.zeros(nmol, dtype=torch.long).index_add_(0, batch_index, mask.long())
    sub_d = ((num_nodes - 1) * 3).float()                                       # subspace_dimensionality :492-498
    delta_log_px = -sub_d * math.log(cfg.norm_values[0])                        # :950-952
    if training:
        delta_log_px = torch.zeros_like(delta_log_px)                           # :979-980
    if t_int is None:
        t_int = torch.randint(0 if training else 1, T + 1, size=(nmol, 1))      # lowest_t (:985-991)
    s_int = t_int - 1
    s, t = s_int / T, t_int / T
    g_s = gamma[torch.round(s * T).long()]                                      # [B,1]
    g_t = gamma[torch.round(t * T).long()]
    xh = torch.cat([xn, h_cat] + ([h_int.reshape(-1, 1)] if cfg.include_charges else []), dim=-1)
    alpha = lambda g: torch.sqrt(torch.sigmoid(-g))
    sigma = lambda g: torch.sqrt(torch.sigmoid(g))
    eps_t = combined_noise(randn, cfg, batch_index, mask, nmol)
    z_t = alpha(g_t)[batch_index] * xh + sigma(g_t)[batch_index] * eps_t        # :910-931
    ctx = context
    net_out = denoise(batch_index, mask, z_t, t[batch_index], ctx)
    sum_mol = lambda v: torch.zeros(nmol).index_add_(0, batch_index, v.sum(-1))  # sum_node_features_except_batch
    error_t = sum_mol((eps_t - net_out) ** 2)                                   # :1052
    snr_weight = (torch.exp(-(g_s - g_t)) - 1).squeeze(-1)                      # :1057-1058
    g0 = gamma[0]
    neg_log_constants = -(sub_d * (-(0.5 * g0) - 0.5 * math.log(2 * math.pi)))  # :579-595,1062-1066
    if training:
        snr_weight = torch.ones_like(error_t)                                   # :1054-1055
        neg_log_constants = torch.zeros_like(neg_log_constants)                 # :1068-1069
    # KL prior (:501-556)
    g_T = gamma[T]
    mu_T = alpha(g_T) * xh
    sig_T = sigma(g_T)
    kl = lambda mu2, qs, d: d * torch.log(1.0 / qs) + 0.5 * (d * qs ** 2 + mu2) - 0.5 * d     # gaussian_KL, p_sigma = 1
    kl_x = kl(sum_mol(mu_T[:, :3] ** 2), sig_T, sub_d)
    kl_h = kl(sum_mol((mu_T[:, 3:] ** 2) * mf[:, None]), sig_T, 1)
    kl_prior = kl_x + kl_h
    if training:
        # L0 from the SAME noised sample, as if gamma_t were gamma_0; selected by the t == 0 mask below (:1083-1103)
        eps_0, z_0, net_0 = eps_t, z_t, net_out
        sig0 = sigma(g_t)[batch_index]
    else:
        # L0 at t = 0 with fresh noise (:1104-1132)
        eps_0 = combined_noise(randn, cfg, batch_index, mask, nmol)
        z_0 = alpha(g0) * xh + sigma(g0) * eps_0
        net_0 = denoise(batch_index, mask, z_0, torch.zeros((xh.shape[0], 1)), ctx)
        sig0 = sigma(g0)
    loss_0_x = 0.5 * sum_mol((eps_0[:, :3] - net_0[:, :3]) ** 2)                # -log p(x|z0) w/o constants (:611-622)
    a = cfg.num_atom_types
    est_cat = z_0[:, 3:3 + a] * cfg.norm_values[1] + cfg.norm_biases[1]
    onehot_u = h_cat * cfg.norm_values[1] + cfg.norm_biases[1]
    cen = est_cat - 1
    log_prop = torch.log(_cdf_std_gaussian((cen + 0.5) / (sig0 * cfg.norm_values[1]))
                         - _cdf_std_gaussian((cen - 0.5) / (sig0 * cfg.norm_values[1])) + 1e-10)
    log_prob = log_prop - torch.logsumexp(log_prop, dim=-1, keepdim=True)
    log_ph_cat = sum_mol(log_prob * onehot_u * mf[:, None])
    if cfg.include_charges:
        h_integer = torch.round(h_int.reshape(-1, 1) * cfg.norm_values[2] + cfg.norm_biases[2]).long()
        est_int = z_0[:, 3 + a:] * cfg.norm_values[2] + cfg.norm_biases[2]
        d_int = h_integer - est_int
        log_ph_int = torch.log(_cdf_std_gaussian((d_int + 0.5) / (sig0 * cfg.norm_values[2]))
                               - _cdf_std_gaussian((d_int - 0.5) / (sig0 * cfg.norm_values[2])) + 1e-10)
        log_ph_int = sum_mol(log_ph_int * mf[:, None])
    else:
        log_ph_int = torch.zeros(nmol)                                          # sum over an empty feature axis
    loss_0_h = -(log_ph_int + log_ph_cat)
    # log p(N) (models/__init__.py:264-308)
    keys = list(n_nodes_hist.keys())
    prob = torch.tensor([float(n_nodes_hist[k]) for k in keys])
    prob = prob / prob.sum()
    log_pn = torch.log(prob + 1e-30)[torch.tensor([keys.index(int(n)) for n in num_nodes.tolist()])]
    if training:
        t0 = (t_int == 0).float().squeeze(-1)
        loss_0_x, loss_0_h, error_t = loss_0_x * t0, loss_0_h * t0, error_t * (1 - t0)       # :1095-1103
        # assembly, training branch with loss_type "l2" (qm9_mol_gen_ddpm.py:232-245)
        eff = (num_nodes.max() if norm_training_by_max_nodes else num_nodes).float()
        denom = (3 + cfg.num_h) * eff
        loss_t = 0.5 * (error_t / denom)
        nll = loss_t + (loss_0_x / denom + loss_0_h) + kl_prior - delta_log_px - log_pn
    else:
        # assembly, evaluation branch (qm9_mol_gen_ddpm.py:247-262)
        loss_t = T * 0.5 * snr_weight * error_t
        nll = loss_t + (loss_0_x + loss_0_h + neg_log_constants) + kl_prior - delta_log_px - log_pn
    terms = dict(delta_log_px=delta_log_px, error_t=error_t, SNR_weight=snr_weight, loss_0_x=loss_0_x,
                 loss_0_h=loss_0_h, neg_log_constants=neg_log_constants, kl_prior=kl_prior, log_pN=log_pn,
                 t_int=t_int.squeeze(-1))
    return nll, terms

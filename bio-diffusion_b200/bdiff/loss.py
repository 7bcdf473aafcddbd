"""GCDMEvalNLL / GCDMTrainLoss — the GCDM objective with the CUDA denoiser (forward only).

Replaces EquivariantVariationalDiffusion.forward in eval mode (reference
src/models/components/variational_diffusion.py:955-1160 with :501-556, :598-699, :702-732, :910-931) and the
evaluation branch of the Lightning module's assembly (src/models/qm9_mol_gen_ddpm.py:184-262): two denoiser calls
(t ~ U{1..T} and t = 0) through libbdiff_sm90, the scalar bookkeeping in torch on the same device.
`GCDMTrainLoss` is the training-mode L2 objective of the same function (one denoiser call, t ~ U{0..T}, L0 selected
by the t == 0 mask; :979-980,985,1054-1055,1068-1069,1083-1103 and qm9_mol_gen_ddpm.py:232-245).  Called with autograd
enabled and trainable parameters it runs the library's training pass, so `loss.mean().backward()` fills `p.grad` of
every denoiser parameter (SURVEY.md §8 a20); under no_grad / inference_mode it is the value only.
"""
from __future__ import annotations

import math
from typing import Callable, Dict, Optional, Tuple

import torch

from . import _lib
from .dynamics import GCPNetDynamicsB200
from .schedule import gamma_table

NoiseFn = Callable[[Tuple[int, int]], torch.Tensor]


def _cdf(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2)))


class GCDMEvalNLL:
    def __init__(self, dynamics: GCPNetDynamicsB200, n_nodes_histogram: Dict[int, int]):
        self.net = dynamics
        self.cfg = dynamics.cfg
        self.gamma = gamma_table(self.cfg.num_timesteps, self.cfg.noise_precision, self.cfg.noise_schedule)
        self.keys = [int(k) for k in n_nodes_histogram.keys()]
        prob = torch.tensor([float(n_nodes_histogram[k]) for k in n_nodes_histogram.keys()])
        self.log_pn = torch.log(prob / prob.sum() + 1e-30)           # NumNodesDistribution (models/__init__.py:264-308)

    def __call__(self, *args, **kwargs):
        with torch.inference_mode():
            return self._impl(*args, **kwargs)

    def _impl(self, batch_index: torch.Tensor, mask: torch.Tensor, x: torch.Tensor, one_hot: torch.Tensor,
                 charges: torch.Tensor, context: Optional[torch.Tensor] = None, t_int: Optional[torch.Tensor] = None,
                 noise: Optional[NoiseFn] = None, training: bool = False, norm_training_by_max_nodes: bool = False):
        """x [N,3] (CoG-free), one_hot [N,A], charges [N] (or [N,0] without charges), context [N,C] or None.
        Returns (nll [B], terms dict).  RNG order matches the reference: t_int, then randn(N,3), randn(N,F) twice."""
        cfg = self.cfg
        dev = x.device
        if dev.type != "cuda":
            raise _lib.BdiffError("GCDMEvalNLL runs on CUDA tensors only (no CPU fallback)")
        T = cfg.num_timesteps
        nmol = int(batch_index[-1].item()) + 1
        n = batch_index.shape[0]
        mf = mask.float()
        gamma = self.gamma.to(dev)
        randn = (lambda shape: torch.randn(shape, device=dev)) if noise is None else (lambda shape: noise(shape).to(dev))

        def seg_sum(v):            # sum_node_features_except_batch (:449-453)
            return torch.zeros(nmol, device=dev).index_add_(0, batch_index, v.sum(-1))

        def centered_noise():      # sample_combined_position_feature_noise (:795-819)
            zx = randn((n, 3)) * mf[:, None]
            tot = torch.zeros((nmol, 3), device=dev).index_add_(0, batch_index, zx)
            cnt = torch.zeros(nmol, device=dev).index_add_(0, batch_index, mf)
            zx = zx - (tot / cnt[:, None])[batch_index] * mf[:, None]
            zh = randn((n, cfg.num_h)) * mf[:, None]
            return torch.cat((zx, zh), dim=-1)

        xn = x / cfg.norm_values[0]
        h_cat = (one_hot.float() - cfg.norm_biases[1]) / cfg.norm_values[1] * mf[:, None]
        h_int = (charges.float() - cfg.norm_biases[2]) / cfg.norm_values[2]
        if cfg.include_charges:
            h_int = h_int.reshape(n) * mf
        num_nodes = torch.zeros(nmol, dtype=torch.long, device=dev).index_add_(0, batch_index, mask.long())
        sub_d = ((num_nodes - 1) * 3).float()
        delta_log_px = -sub_d * math.log(cfg.norm_values[0])
        if training:
            delta_log_px = torch.zeros_like(delta_log_px)
        if t_int is None:
            t_int = torch.randint(0 if training else 1, T + 1, size=(nmol, 1), device=dev)
        t_int = t_int.to(dev)
        s = (t_int - 1) / T
        t = t_int / T
        g_s = gamma[torch.round(s * T).long()]
        g_t = gamma[torch.round(t * T).long()]
        xh = torch.cat([xn, h_cat] + ([h_int.reshape(-1, 1)] if cfg.include_charges else []), dim=-1)
        alpha = lambda g: torch.sqrt(torch.sigmoid(-g))
        sigma = lambda g: torch.sqrt(torch.sigmoid(g))
        eps_t = centered_noise()
        z_t = alpha(g_t)[batch_index] * xh + sigma(g_t)[batch_index] * eps_t
        denoise = self.net.denoise_train if self.net.wants_grad() else self.net.denoise
        net_out = denoise(batch_index, mask, z_t, t[batch_index], context, nmol)
        error_t = seg_sum((eps_t - net_out) ** 2)
        snr_weight = (torch.exp(-(g_s - g_t)) - 1).squeeze(-1)
        g0, g_T = gamma[0], gamma[T]
        neg_log_constants = -(sub_d * (-(0.5 * g0) - 0.5 * math.log(2 * math.pi)))
        if training:
            snr_weight = torch.ones_like(error_t)
            neg_log_constants = torch.zeros_like(neg_log_constants)
        mu_T = alpha(g_T) * xh
        sig_T = sigma(g_T)
        kl = lambda mu2, qs, d: d * torch.log(1.0 / qs) + 0.5 * (d * qs ** 2 + mu2) - 0.5 * d
        kl_prior = kl(seg_sum(mu_T[:, :3] ** 2), sig_T, sub_d) + kl(seg_sum((mu_T[:, 3:] ** 2) * mf[:, None]), sig_T, 1)
        if training:      # L0 from the same noised sample, selected by the t == 0 mask below
            eps_0, z_0, net_0 = eps_t, z_t, net_out
            sig0 = sigma(g_t)[batch_index]
        else:
            eps_0 = centered_noise()
            z_0 = alpha(g0) * xh + sigma(g0) * eps_0
            net_0 = self.net.denoise(batch_index, mask, z_0, torch.zeros((n, 1), device=dev), context, nmol)
            sig0 = sigma(g0)
        loss_0_x = 0.5 * seg_sum((eps_0[:, :3] - net_0[:, :3]) ** 2)
        a = cfg.num_atom_types
        cen = z_0[:, 3:3 + a] * cfg.norm_values[1] + cfg.norm_biases[1] - 1
        onehot_u = h_cat * cfg.norm_values[1] + cfg.norm_biases[1]
        log_prop = torch.log(_cdf((cen + 0.5) / (sig0 * cfg.norm_values[1])) - _cdf((cen - 0.5) / (sig0 * cfg.norm_values[1]))
                             + 1e-10)
        log_prob = log_prop - torch.logsumexp(log_prop, dim=-1, keepdim=True)
        log_ph = seg_sum(log_prob * onehot_u * mf[:, None])
        if cfg.include_charges:
            h_integer = torch.round(h_int.reshape(-1, 1) * cfg.norm_values[2] + cfg.norm_biases[2]).long()
            d_int = h_integer - (z_0[:, 3 + a:] * cfg.norm_values[2] + cfg.norm_biases[2])
            lpi = torch.log(_cdf((d_int + 0.5) / (sig0 * cfg.norm_values[2])) - _cdf((d_int - 0.5) / (sig0 * cfg.norm_values[2]))
                            + 1e-10)
            log_ph = log_ph + seg_sum(lpi * mf[:, None])
        loss_0_h = -log_ph
        idx = torch.tensor([self.keys.index(int(v)) for v in num_nodes.tolist()], device=dev)
        log_pn = self.log_pn.to(dev)[idx]
        if training:
            t0 = (t_int == 0).float().squeeze(-1)
            loss_0_x, loss_0_h, error_t = loss_0_x * t0, loss_0_h * t0, error_t * (1 - t0)
            eff = (num_nodes.max() if norm_training_by_max_nodes else num_nodes).float()
            denom = (3 + cfg.num_h) * eff
            nll = 0.5 * (error_t / denom) + (loss_0_x / denom + loss_0_h) + kl_prior - delta_log_px - log_pn
        else:
            nll = T * 0.5 * snr_weight * error_t + (loss_0_x + loss_0_h + neg_log_constants) + kl_prior - delta_log_px - log_pn
        terms = dict(delta_log_px=delta_log_px, error_t=error_t, SNR_weight=snr_weight, loss_0_x=loss_0_x, loss_0_h=loss_0_h,
                     neg_log_constants=neg_log_constants, kl_prior=kl_prior, log_pN=log_pn, t_int=t_int.squeeze(-1))
        return nll, terms


class GCDMTrainLoss(GCDMEvalNLL):
    """Training-mode objective (loss_type "l2"): `loss, terms = GCDMTrainLoss(net, histogram)(batch_index, mask, x, ...)`;
    `loss.mean().backward()` is the reference's training_step (qm9_mol_gen_ddpm.py:340-362).  With autograd disabled (or
    no trainable parameter) the value is computed by the sampler kernels in inference mode."""

    def __call__(self, *args, **kwargs):
        kwargs.setdefault("training", True)
        if self.net.wants_grad():
            return self._impl(*args, **kwargs)
        return super().__call__(*args, **kwargs)

"""GCDMSampler — the T-step ancestral sampler of GCDM with the CUDA denoiser in its inner loop.

Replaces the inner loop of EquivariantVariationalDiffusion.mol_gen_sample / sample_p_zs_given_zt /
sample_p_xh_given_z0 (reference src/models/components/variational_diffusion.py:1280-1412, 1204-1278, 840-907):
one reverse step = two torch.randn draws (same order as the reference: randn(N,3) then randn(N,F)) + one
C-ABI call (bdiff_reverse_step: 4+2L+2 kernels) + a device counter bump, captured ONCE in a CUDA graph and
replayed T times — no host synchronisation inside the chain.

inpaint (variational_diffusion.py:1580-1789, RePaint) replays two such graphs in the order of the RePaint schedule: the
denoise op (4 draws, the reverse step, bdiff_repaint_combine, frame write, op counter bump) and the jump back (2 draws,
bdiff_renoise, jump counter bump).  Every per-op coefficient is read on the device at the counters.
"""
from __future__ import annotations

import ctypes as C
from typing import Callable, Optional, Tuple

import torch
import torch.nn.functional as F

from . import _lib
from .dynamics import GCPNetDynamicsB200
from .schedule import (chain_frame_slots, check_frames, check_repaint, decode_coefficients, gamma_table,
                       repaint_program, step_coefficient_table)

NoiseFn = Callable[[Tuple[int, int]], torch.Tensor]


class GCDMSampler:
    def __init__(self, dynamics: GCPNetDynamicsB200, use_cuda_graph: bool = True):
        self.net = dynamics
        self.cfg = dynamics.cfg
        self.use_cuda_graph = use_cuda_graph
        self.gamma = gamma_table(self.cfg.num_timesteps, self.cfg.noise_precision, self.cfg.noise_schedule)
        self._graph_key = None
        self._graph = None
        self._static = None
        self._ip = None              # inpaint: statics, and the op / jump graphs with their key
        self._ip_graphs = None
        self._ip_graph_key = None
        self.kernel_launches = 0     # libbdiff kernels launched (or replayed from the graph) by sample() / inpaint()
        self.last_moments = None     # [T, 4] per-step (mean|x|, max|x|, mean h, mean|h|) of z when sample(record_moments=True)

    # -------------------------------------------------------------------------------------------- helpers
    def _device(self) -> torch.device:
        return next(self.net.parameters()).device

    def _statics(self, n: int, steps: int, dev: torch.device):
        key = (n, steps, dev)
        if self._static is not None and self._static["key"] == key:
            return self._static
        f = self.cfg.num_h
        st = dict(key=key,
                  z=torch.zeros((n, 3 + f), device=dev), nx=torch.zeros((n, 3), device=dev),
                  nh=torch.zeros((n, f), device=dev), step=torch.zeros((), dtype=torch.int32, device=dev),
                  coef=step_coefficient_table(self.gamma, steps).to(dev),
                  dec=decode_coefficients(self.gamma).to(dev), xh=torch.zeros((n, 3 + f), device=dev))
        self._static = st
        self._graph = None
        self._graph_key = None
        return st

    def _reverse_step(self, st, ctx_ptr):
        lib = _lib.load()
        h = self.net._handle
        _lib.check(h, lib.bdiff_reverse_step(h, self.net._stream(), C.c_void_p(st["z"].data_ptr()), ctx_ptr,
                                             C.c_void_p(st["nx"].data_ptr()), C.c_void_p(st["nh"].data_ptr()),
                                             C.c_void_p(st["coef"].data_ptr()), C.c_void_p(st["step"].data_ptr())),
                   "bdiff_reverse_step")

    def _write_frame(self, frames: torch.Tensor, slots: torch.Tensor, counter: torch.Tensor, z: torch.Tensor,
                     mf: torch.Tensor) -> None:
        """frames[slots[counter]] = unnormalize_z(z) (variational_diffusion.py:762-792, 1353-1360), all on the device
        so that it can sit in a captured graph; slot `return_frames` is the dummy row of ops that write no frame."""
        cfg = self.cfg
        a = cfg.num_atom_types
        parts = [z[:, :3] * cfg.norm_values[0], (z[:, 3:3 + a] * cfg.norm_values[1] + cfg.norm_biases[1]) * mf]
        if cfg.include_charges:
            parts.append((z[:, 3 + a:] * cfg.norm_values[2] + cfg.norm_biases[2]) * mf)
        frames.index_copy_(0, slots.index_select(0, counter.long().view(1)), torch.cat(parts, dim=-1).unsqueeze(0))

    def _finish(self, xh: torch.Tensor, batch_index: torch.Tensor, mask: torch.Tensor, b: int, cog_fix: bool):
        """Unnormalise and discretise p(x, h | z_0) (variational_diffusion.py:892-907), check the chain, CoG fix."""
        cfg = self.cfg
        h = self.net._handle
        lib = _lib.load()
        dev = xh.device
        mf = mask.float().unsqueeze(-1)
        a = cfg.num_atom_types
        x = xh[:, :3] * cfg.norm_values[0]
        h_cat = (xh[:, 3:3 + a] * cfg.norm_values[1] + cfg.norm_biases[1]) * mf
        h_cat = F.one_hot(torch.argmax(h_cat, dim=-1), a) * mask.long().unsqueeze(-1)
        parts = [None, h_cat.float()]
        if cfg.include_charges:
            h_int = (xh[:, 3 + a:] * cfg.norm_values[2] + cfg.norm_biases[2]) * mf
            parts.append((torch.round(h_int).long() * mask.long().unsqueeze(-1)).float())
        # deferred device-side conditions of the chain (synchronises; see bdiff_check in include/bdiff.h)
        _lib.check(h, lib.bdiff_check(h, self.net._stream()), "bdiff_check")
        # CoG drift correction (variational_diffusion.py:1391-1402) — the single host sync of the chain; the reference
        # skips it when intermediate frames are returned
        if cog_fix:
            tot = torch.zeros((b, 3), device=dev).index_add_(0, batch_index, x)
            if tot.abs().max().item() > 5e-2:
                cnt = torch.zeros(b, device=dev).index_add_(0, batch_index, mask.float())
                x = x - (tot / cnt.unsqueeze(-1))[batch_index] * mf
        parts[0] = x
        return torch.cat(parts, dim=-1)

    # -------------------------------------------------------------------------------------------- sampling
    @torch.inference_mode()
    def sample(self, num_nodes: torch.Tensor, context: Optional[torch.Tensor] = None,
               num_timesteps: Optional[int] = None, node_mask: Optional[torch.Tensor] = None,
               noise: Optional[NoiseFn] = None, return_z0: bool = False, z_init: Optional[torch.Tensor] = None,
               record_moments: bool = False, return_frames: int = 1):
        """mol_gen_sample (variational_diffusion.py:1280-1412).

        num_nodes int64[B]; context [B,C] or None; `noise(shape)` optionally injects the randn draws (tests).
        `z_init` [N, 3+F] (normalised, CoG-free) starts the chain from given states instead of z_T ~ N(0, I) — no
        initial noise draw (this is what `optimize` / the reference's mol_gen_optimize does).
        Returns (out [N, 3+A(+1)], batch_index [N], node_mask [N]) like the reference (+ z_0 when asked).  With
        return_frames = F > 1, out is [F, N, 3+A(+1)]: frame k is the unnormalised latent after the step that lands on
        s = k*T/F, frame 0 the decoded molecules (no CoG drift correction, as in the reference).
        """
        cfg = self.cfg
        steps = cfg.num_timesteps if num_timesteps is None else int(num_timesteps)
        check_frames(steps, return_frames)
        dev = self._device()
        if dev.type != "cuda":
            raise _lib.BdiffError("GCDMSampler needs the denoiser on a CUDA device (no CPU fallback)")
        num_nodes = num_nodes.to(dev, non_blocking=True)
        b = int(num_nodes.shape[0])
        batch_index = torch.repeat_interleave(torch.arange(b, device=dev), num_nodes)
        n = int(batch_index.shape[0])
        mask = torch.ones(n, dtype=torch.bool, device=dev) if node_mask is None else node_mask.to(dev)
        ctx = None
        ctx_ptr = None
        if cfg.num_context:
            if context is None:
                raise ValueError("property-conditional configuration: `context` [B,C] is required")
            ctx = (context.to(dev, torch.float32)[batch_index] * mask.float().unsqueeze(-1)).contiguous()
            ctx_ptr = C.c_void_p(ctx.data_ptr())
        self.net.sync_weights()
        # the plan is keyed on tensor identity: reuse the tensors of the previous call when the topology repeats
        if self._static is not None and self._static.get("topo") is not None:
            pbi, pmask = self._static["topo"]
            if pbi.shape == batch_index.shape and torch.equal(pbi, batch_index) and torch.equal(pmask, mask):
                batch_index, mask = pbi, pmask
        self.net.plan(batch_index, mask, b)
        st = self._statics(n, steps, dev)
        st["topo"] = (batch_index, mask)
        lib = _lib.load()
        h = self.net._handle
        f = cfg.num_h

        def draw(buf_x, buf_h):
            if noise is None:
                torch.randn((n, 3), device=dev, out=buf_x)
                torch.randn((n, f), device=dev, out=buf_h)
            else:
                buf_x.copy_(noise((n, 3)))
                buf_h.copy_(noise((n, f)))

        if z_init is None:
            # z_T ~ N(0, I) on the zero-CoG subspace (variational_diffusion.py:1322-1328)
            draw(st["nx"], st["nh"])
            _lib.check(h, lib.bdiff_center_noise(h, self.net._stream(), C.c_void_p(st["nx"].data_ptr()),
                                                 C.c_void_p(st["nh"].data_ptr()), C.c_void_p(st["z"].data_ptr())),
                       "bdiff_center_noise")
        else:
            if tuple(z_init.shape) != (n, 3 + f):
                raise ValueError(f"z_init must be [{n}, {3 + f}]")
            st["z"].copy_(z_init.to(dev, torch.float32))
        st["step"].zero_()

        moments = torch.zeros((steps, 4), device=dev) if record_moments else None

        def record():
            # diagnostics only (tests): moments of the latent after this step, written at row `step` on the device
            zx, zh = st["z"][:, :3], st["z"][:, 3:]
            m = torch.stack((zx.abs().mean(), zx.abs().max(), zh.mean(), zh.abs().mean())).view(1, 4)
            moments.index_copy_(0, st["step"].long().view(1), m)

        frames = None
        if return_frames > 1:
            fkey = ("frames", return_frames)
            if fkey not in st:
                st[fkey] = (torch.zeros((return_frames + 1, n, 3 + f), device=dev),
                            chain_frame_slots(steps, return_frames).to(dev), torch.zeros((n, 1), device=dev))
            frames, slots, mf_frames = st[fkey]
            frames.zero_()
            mf_frames.copy_(mask.float().unsqueeze(-1))

        graph_ok = self.use_cuda_graph and noise is None
        if graph_ok:
            # the captured graph bakes in raw pointers of the library's plan / workspace buffers, which move when a larger
            # topology was planned in between: the plan epoch (bumped by every bdiff_plan_topology) is part of the key
            gkey = (st["key"], self.net._plan_key, self.net._plan_epoch, self.net._weights_key,
                    ctx.data_ptr() if ctx is not None else 0, moments.data_ptr() if record_moments else 0)
            if return_frames > 1:
                gkey = gkey + (frames.data_ptr(),)
            if self._graph is None or self._graph_key != gkey:
                torch.cuda.current_stream().synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    draw(st["nx"], st["nh"])
                    self._reverse_step(st, ctx_ptr)
                    if record_moments:
                        record()
                    if return_frames > 1:
                        self._write_frame(frames, slots, st["step"], st["z"], mf_frames)
                    st["step"].add_(1)
                self._graph, self._graph_key = g, gkey
                self._ctx_keep = ctx
            for _ in range(steps):
                self._graph.replay()
        else:
            for _ in range(steps):
                draw(st["nx"], st["nh"])
                self._reverse_step(st, ctx_ptr)
                if record_moments:
                    record()
                if return_frames > 1:
                    self._write_frame(frames, slots, st["step"], st["z"], mf_frames)
                st["step"].add_(1)
        self.last_moments = moments

        # one forward = prep, node_frames, edge_embed, node_embed, L x (edge_message, node_update), finalize
        per_forward = self.net.kernels_per_forward
        self.kernel_launches += 1 + steps * (per_forward + 1) + (per_forward + 1)
        # p(x, h | z_0)  (variational_diffusion.py:1378-1387, 840-907)
        z0 = st["z"].clone() if return_z0 else None
        draw(st["nx"], st["nh"])
        _lib.check(h, lib.bdiff_decode_z0(h, self.net._stream(), C.c_void_p(st["z"].data_ptr()), ctx_ptr,
                                          C.c_void_p(st["nx"].data_ptr()), C.c_void_p(st["nh"].data_ptr()),
                                          C.c_void_p(st["dec"].data_ptr()), C.c_void_p(st["xh"].data_ptr())),
                   "bdiff_decode_z0")
        out = self._finish(st["xh"], batch_index, mask, b, cog_fix=return_frames == 1)
        if return_frames > 1:
            out = torch.cat((out.unsqueeze(0), frames[1:return_frames]), dim=0)    # out[0] <- the molecules (:1404-1410)
        return (out, batch_index, mask, z0) if return_z0 else (out, batch_index, mask)

    def nan_guard_count(self, reset: bool = False) -> int:
        """Denoiser forwards in which the NaN guard of gcpnet.py:1214-1216 fired since the workspace was (re)planned."""
        lib = _lib.load()
        v = C.c_int64(0)
        _lib.check(self.net._handle, lib.bdiff_nan_guard_count(self.net._handle, self.net._stream(), C.byref(v),
                                                              1 if reset else 0), "bdiff_nan_guard_count")
        return int(v.value)

    @torch.inference_mode()
    def reverse_step_once(self, z: torch.Tensor, row: int, steps: int, batch_index: torch.Tensor,
                          mask: torch.Tensor, noise_x: torch.Tensor, noise_h: torch.Tensor,
                          context: Optional[torch.Tensor] = None, num_mols: Optional[int] = None) -> torch.Tensor:
        """One p(z_s | z_t) step from a given z (row `row` of the coefficient table for a `steps`-step chain):
        sample_p_zs_given_zt, variational_diffusion.py:1204-1278.  Used by teacher-forced parity tests."""
        dev = z.device
        self.net.sync_weights()
        self.net.plan(batch_index, mask, num_mols)
        lib = _lib.load()
        h = self.net._handle
        coef = step_coefficient_table(self.gamma, steps).to(dev)
        idx = torch.tensor(row, dtype=torch.int32, device=dev)
        zz = z.detach().to(torch.float32).clone().contiguous()
        nx = noise_x.to(torch.float32).contiguous()
        nh = noise_h.to(torch.float32).contiguous()
        ctx_ptr = None
        if self.cfg.num_context:
            ctx = context.to(torch.float32).contiguous()
            ctx_ptr = C.c_void_p(ctx.data_ptr())
        _lib.check(h, lib.bdiff_reverse_step(h, self.net._stream(), C.c_void_p(zz.data_ptr()), ctx_ptr,
                                             C.c_void_p(nx.data_ptr()), C.c_void_p(nh.data_ptr()),
                                             C.c_void_p(coef.data_ptr()), C.c_void_p(idx.data_ptr())),
                   "bdiff_reverse_step")
        torch.cuda.current_stream().synchronize()
        return zz

    @torch.inference_mode()
    @torch.inference_mode()
    def optimize(self, samples, num_nodes: torch.Tensor, context: Optional[torch.Tensor] = None,
                 num_timesteps: Optional[int] = None, node_mask: Optional[torch.Tensor] = None,
                 noise: Optional[NoiseFn] = None, return_frames: int = 1):
        """mol_gen_optimize (variational_diffusion.py:1414-1546, norm_with_original_timesteps=False):
        run `num_timesteps` reverse steps starting from existing molecules.  `samples` = list of (x [n_k,3] CoG-free,
        one_hot [n_k,A]) per molecule as in the reference.  Only configurations without integer features
        (include_charges=False) — the reference stacks positions and categorical features only.  return_frames as in
        `sample` (:1471-1498)."""
        cfg = self.cfg
        if cfg.include_charges:
            raise NotImplementedError("mol_gen_optimize stacks [x | one-hot] only: needs include_charges=False")
        check_frames(cfg.num_timesteps if num_timesteps is None else int(num_timesteps), return_frames)
        dev = self._device()
        x = torch.vstack([s[0] for s in samples]).to(dev, torch.float32)
        hc = torch.vstack([s[1] for s in samples]).to(dev, torch.float32)
        n = x.shape[0]
        mask = torch.ones(n, dtype=torch.bool, device=dev) if node_mask is None else node_mask.to(dev)
        mf = mask.float().unsqueeze(-1)
        bi = torch.repeat_interleave(torch.arange(len(samples), device=dev), num_nodes.to(dev))
        if bi.shape[0] != n:
            raise ValueError("num_nodes does not match the samples")
        z = torch.cat((x / cfg.norm_values[0] * mf, (hc - cfg.norm_biases[1]) / cfg.norm_values[1] * mf), dim=-1)   # normalize (:702-732)
        largest = z[:, :3].abs().max().item()                                 # assert_mean_zero_with_mask (:465-474):
        err = z[:, :3].sum(dim=0).abs().max().item()                          # the reference sums over the WHOLE batch
        if err / (largest + 1e-10) >= 1e-2:
            raise AssertionError(f"Mean is not zero, as relative_error {err / (largest + 1e-10)}")
        return self.sample(num_nodes, context, num_timesteps, node_mask, noise, z_init=z, return_frames=return_frames)

    @staticmethod
    def _inpaint_inputs(cfg, molecule, node_mask_fixed, context):
        """Validates the arguments of `inpaint` on the host; returns (num_nodes, batch_index, xh0_parts, fixed, context)."""
        for key in ("x", "one_hot", "num_nodes", "batch_index"):
            if key not in molecule:
                raise ValueError(f"molecule['{key}'] is required")
        x, one_hot = molecule["x"], molecule["one_hot"]
        num_nodes = torch.as_tensor(molecule["num_nodes"]).reshape(-1).cpu().long()
        n = int(x.shape[0]) if x.dim() == 2 else -1
        if x.dim() != 2 or x.shape[1] != 3:
            raise ValueError(f"molecule['x'] must be [N, 3], got {tuple(x.shape)}")
        if tuple(one_hot.shape) != (n, cfg.num_atom_types):
            raise ValueError(f"molecule['one_hot'] must be [{n}, {cfg.num_atom_types}], got {tuple(one_hot.shape)}")
        parts = [x, one_hot]
        if cfg.include_charges:
            if "charges" not in molecule:
                raise ValueError("molecule['charges'] is required by a configuration with include_charges")
            ch = molecule["charges"]
            if tuple(ch.shape) not in ((n, 1), (n,)):
                raise ValueError(f"molecule['charges'] must be [{n}, 1], got {tuple(ch.shape)}")
            parts.append(ch.reshape(n, 1))
        if tuple(node_mask_fixed.shape) != (n,):
            raise ValueError(f"node_mask_fixed must be [{n}], got {tuple(node_mask_fixed.shape)}")
        if int(num_nodes.sum()) != n or bool((num_nodes < 1).any()):
            raise ValueError("molecule['num_nodes'] must be positive and sum to the number of atoms")
        b = int(num_nodes.shape[0])
        batch_index = torch.repeat_interleave(torch.arange(b), num_nodes)
        bi_in = molecule["batch_index"]
        if tuple(bi_in.shape) != (n,) or not torch.equal(bi_in.cpu().long(), batch_index):
            raise ValueError("molecule['batch_index'] must be the sorted molecule index implied by num_nodes")
        if cfg.num_context:
            if context is None or tuple(context.shape) != (b, cfg.num_context):
                raise ValueError(f"property-conditional configuration: `context` [{b}, {cfg.num_context}] is required")
        elif context is not None:
            raise ValueError("`context` given to a configuration without conditioning")
        return num_nodes, batch_index, parts, node_mask_fixed.bool(), context

    def _inpaint_statics(self, n: int, steps: int, r: int, j: int, frames: int, dev: torch.device):
        key = (n, steps, r, j, frames, dev)
        if self._ip is not None and self._ip["key"] == key:
            return self._ip
        f = self.cfg.num_h
        prog = repaint_program(self.gamma, r, j, steps, frames)
        st = dict(key=key, prog=prog,
                  z=torch.zeros((n, 3 + f), device=dev), xh=torch.zeros((n, 3 + f), device=dev),
                  nx=torch.zeros((n, 3), device=dev), nh=torch.zeros((n, f), device=dev),
                  kx=torch.zeros((n, 3), device=dev), kh=torch.zeros((n, f), device=dev),
                  step=torch.zeros((), dtype=torch.int32, device=dev), jstep=torch.zeros((), dtype=torch.int32, device=dev),
                  coef=prog["rev"].to(dev), known=prog["known"].to(dev), jump=prog["jump"].to(dev),
                  slot=prog["slot"].to(dev), dec=decode_coefficients(self.gamma).to(dev),
                  xh0=torch.zeros((n, 3 + f), device=dev), fixed=torch.zeros(n, dtype=torch.uint8, device=dev),
                  mf=torch.ones((n, 1), device=dev), topo=None,
                  frames=torch.zeros((frames + 1, n, 3 + f), device=dev) if frames > 1 else None)
        self._ip = st
        self._ip_graphs = None
        self._ip_graph_key = None
        return st

    @torch.inference_mode()
    def inpaint(self, molecule: dict, node_mask_fixed: torch.Tensor, num_resamplings: int = 1, jump_length: int = 1,
                return_frames: int = 1, num_timesteps: Optional[int] = None, context: Optional[torch.Tensor] = None,
                noise: Optional[NoiseFn] = None) -> torch.Tensor:
        """EquivariantVariationalDiffusion.inpaint (variational_diffusion.py:1580-1789): generate the rest of each molecule
        around the atoms with node_mask_fixed = True, which keep their type and 3-D position (RePaint).

        molecule: dict with x [N,3], one_hot [N,A], charges [N,1] (configurations with include_charges), num_nodes [B] and
        batch_index [N] (sorted).  Defined as the reference with two repairs: the dead self-conditioning line that raises
        UnboundLocalError (:1650) is dropped, and the jump back takes alpha_t|s per molecule (:1177 indexes it by the node
        mask).  xh0 = [x | one_hot | charges] enters the latent space unnormalised, as in the reference.  A molecule
        without fixed atoms is sampled freely.  `noise(shape)` optionally injects the randn draws in the reference's
        order: z_T, then per denoise op the known part and the unknown part, per jump one pair, the final decode.
        Returns out [N, 3+A(+1)], or [F, N, 3+A(+1)] for return_frames = F > 1 (frame 0 = the molecules).
        """
        cfg = self.cfg
        steps = cfg.num_timesteps if num_timesteps is None else int(num_timesteps)
        r, j, nfr = int(num_resamplings), int(jump_length), int(return_frames)
        check_repaint(r, j, steps, nfr)
        num_nodes, batch_index, parts, fixed, context = self._inpaint_inputs(cfg, molecule, node_mask_fixed, context)
        dev = self._device()
        if dev.type != "cuda":
            raise _lib.BdiffError("GCDMSampler needs the denoiser on a CUDA device (no CPU fallback)")
        b = int(num_nodes.shape[0])
        n = int(batch_index.shape[0])
        f = cfg.num_h
        batch_index = batch_index.to(dev)
        mask = torch.ones(n, dtype=torch.bool, device=dev)          # inpaint has no padding mask (:1638)
        ctx, ctx_ptr = None, None
        if cfg.num_context:
            ctx = context.to(dev, torch.float32)[batch_index].contiguous()     # (:1614-1615)
            ctx_ptr = C.c_void_p(ctx.data_ptr())
        self.net.sync_weights()
        st = self._inpaint_statics(n, steps, r, j, nfr, dev)
        if st["topo"] is not None and torch.equal(st["topo"][0], batch_index):
            batch_index, mask = st["topo"]
        self.net.plan(batch_index, mask, b)
        st["topo"] = (batch_index, mask)
        prog = st["prog"]
        lib = _lib.load()
        h = self.net._handle

        # xh0 with x centred on the fixed atoms of its molecule (:1617-1633); a molecule without fixed atoms is not moved.
        # A one-off step on the host: sequential float32 sums like the reference, and run-to-run reproducible (the
        # device's index_add_ sums in atomic order)
        xh0 = torch.cat([p.detach().to("cpu", torch.float32).reshape(n, -1) for p in parts], dim=-1)
        bi_h = batch_index.cpu()
        ff = fixed.cpu().float()
        tot = torch.zeros((b, 3)).index_add_(0, bi_h, xh0[:, :3] * ff.unsqueeze(-1))
        cnt = torch.zeros(b).index_add_(0, bi_h, ff)
        xh0[:, :3] -= (tot / cnt.clamp(min=1.0).unsqueeze(-1))[bi_h]
        st["xh0"].copy_(xh0)
        st["fixed"].copy_(fixed.cpu().to(torch.uint8))

        def draw(buf_x, buf_h):
            if noise is None:
                torch.randn((n, 3), device=dev, out=buf_x)
                torch.randn((n, f), device=dev, out=buf_h)
            else:
                buf_x.copy_(noise((n, 3)))
                buf_h.copy_(noise((n, f)))

        def ptr(t):
            return C.c_void_p(t.data_ptr())

        def denoise_op():
            draw(st["kx"], st["kh"])                                  # z_known's noise (:1661-1667)
            draw(st["nx"], st["nh"])                                  # z_unknown = p(z_s | z_t) (:1670-1679)
            self._reverse_step(st, ctx_ptr)
            _lib.check(h, lib.bdiff_repaint_combine(h, self.net._stream(), ptr(st["z"]), ptr(st["xh0"]), ptr(st["fixed"]),
                                                    ptr(st["kx"]), ptr(st["kh"]), ptr(st["known"]), ptr(st["step"])),
                       "bdiff_repaint_combine")
            if nfr > 1:
                self._write_frame(st["frames"], st["slot"], st["step"], st["z"], st["mf"])
            st["step"].add_(1)

        def jump_back():
            draw(st["nx"], st["nh"])
            _lib.check(h, lib.bdiff_renoise(h, self.net._stream(), ptr(st["z"]), ptr(st["nx"]), ptr(st["nh"]), ptr(st["jump"]),
                                            ptr(st["jstep"])), "bdiff_renoise")
            st["jstep"].add_(1)

        # z_T ~ N(0, I) on the zero-CoG subspace (:1635-1640)
        draw(st["nx"], st["nh"])
        _lib.check(h, lib.bdiff_center_noise(h, self.net._stream(), ptr(st["nx"]), ptr(st["nh"]), ptr(st["z"])), "bdiff_center_noise")
        st["step"].zero_()
        st["jstep"].zero_()
        if nfr > 1:
            st["frames"].zero_()

        if self.use_cuda_graph and noise is None:
            gkey = (st["key"], self.net._plan_key, self.net._plan_epoch, self.net._weights_key,
                    ctx.data_ptr() if ctx is not None else 0)
            if self._ip_graphs is None or self._ip_graph_key != gkey:
                torch.cuda.current_stream().synchronize()
                g_op = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g_op):
                    denoise_op()
                g_jump = None
                if prog["num_jumps"]:
                    g_jump = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g_jump):
                        jump_back()
                self._ip_graphs, self._ip_graph_key = (g_op, g_jump), gkey
                self._ip_ctx_keep = ctx
            g_op, g_jump = self._ip_graphs
            for jump in prog["jump_after"]:
                g_op.replay()
                if jump:
                    g_jump.replay()
        else:
            for jump in prog["jump_after"]:
                denoise_op()
                if jump:
                    jump_back()

        ops = len(prog["jump_after"])
        per_forward = self.net.kernels_per_forward
        self.kernel_launches += 1 + ops * (per_forward + 2) + prog["num_jumps"] + (per_forward + 1)
        # p(x, h | z_0) (:1753-1762), then the CoG fix when no frames are returned (:1768-1778)
        draw(st["nx"], st["nh"])
        _lib.check(h, lib.bdiff_decode_z0(h, self.net._stream(), ptr(st["z"]), ctx_ptr, ptr(st["nx"]), ptr(st["nh"]), ptr(st["dec"]),
                                          ptr(st["xh"])), "bdiff_decode_z0")
        out = self._finish(st["xh"], batch_index, mask, b, cog_fix=nfr == 1)
        if nfr > 1:
            out = torch.cat((out.unsqueeze(0), st["frames"][1:nfr]), dim=0)          # out[0] <- the molecules (:1780-1786)
        return out

    def sample_from_host(self, num_nodes_host: torch.Tensor, context_host: Optional[torch.Tensor] = None,
                         num_timesteps: Optional[int] = None, out_host: Optional[torch.Tensor] = None):
        """End-to-end entry used by bench.py: pinned host inputs -> device -> chain -> pinned host result."""
        dev = self._device()
        nn_dev = num_nodes_host.to(dev, non_blocking=True)
        ctx_dev = context_host.to(dev, non_blocking=True) if context_host is not None else None
        out, batch_index, mask = self.sample(nn_dev, ctx_dev, num_timesteps)
        if out_host is None:
            out_host = torch.empty(out.shape, dtype=out.dtype, pin_memory=True)
        out_host.copy_(out, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return out_host

"""GCDMSampler — the T-step ancestral sampler of GCDM with the CUDA denoiser in its inner loop.

Replaces the inner loop of EquivariantVariationalDiffusion.mol_gen_sample / sample_p_zs_given_zt /
sample_p_xh_given_z0 (reference src/models/components/variational_diffusion.py:1280-1412, 1204-1278, 840-907):
one reverse step = two torch.randn draws (same order as the reference: randn(N,3) then randn(N,F)) + one
C-ABI call (bdiff_reverse_step: 4+2L+2 kernels) + a device counter bump, captured ONCE in a CUDA graph and
replayed T times — no host synchronisation inside the chain.

inpaint (variational_diffusion.py:1580-1789, RePaint) runs the same chain with two bodies replayed in the order of the
RePaint schedule: the denoise op (4 draws, the reverse step, bdiff_repaint_combine, frame write, op counter bump) and the
jump back (2 draws, bdiff_renoise, jump counter bump).  Every per-op coefficient is read on the device at the counters.
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


def _ptr(t: Optional[torch.Tensor]) -> Optional[C.c_void_p]:
    return None if t is None else C.c_void_p(t.data_ptr())


class GCDMSampler:
    def __init__(self, dynamics: GCPNetDynamicsB200, use_cuda_graph: bool = True):
        self.net = dynamics
        self.cfg = dynamics.cfg
        self.use_cuda_graph = use_cuda_graph
        self.gamma = gamma_table(self.cfg.num_timesteps, self.cfg.noise_precision, self.cfg.noise_schedule)
        self._static = None          # every device buffer the chain's graphs read or write (see _statics)
        self._graphs = None          # the captured bodies of the chain on these statics, and their key
        self._graph_key = None
        self._topo = None            # (batch_index, mask) of the last plan
        self.kernel_launches = 0     # libbdiff kernels launched (or replayed from the graph) by sample() / inpaint()
        self.last_moments = None     # [T, 4] per-step (mean|x|, max|x|, mean h, mean|h|) of z when sample(record_moments=True)

    # -------------------------------------------------------------------------------------------- helpers
    def _device(self) -> torch.device:
        return next(self.net.parameters()).device

    def _statics(self, n: int, steps: int, repaint: Optional[Tuple[int, int]], frames: int, moments: bool,
                 dev: torch.device):
        """The chain's device buffers and tables, cached by shape and chain kind (plain, or RePaint with (r, j)).
        Building new statics drops the graphs captured on the old ones."""
        key = (n, steps, repaint, frames, moments, dev)
        if self._static is not None and self._static["key"] == key:
            return self._static
        f, c = self.cfg.num_h, self.cfg.num_context

        def zeros(*shape, dtype=torch.float32):
            return torch.zeros(shape, dtype=dtype, device=dev)

        if repaint is None:
            prog = dict(rev=step_coefficient_table(self.gamma, steps), slot=chain_frame_slots(steps, frames),
                        jump_after=[False] * steps, num_jumps=0)
        else:
            prog = repaint_program(self.gamma, *repaint, steps, frames)
        st = dict(key=key, repaint=repaint, schedule=prog["jump_after"], num_jumps=prog["num_jumps"],
                  z=zeros(n, 3 + f), xh=zeros(n, 3 + f), nx=zeros(n, 3), nh=zeros(n, f),
                  step=zeros(dtype=torch.int32), coef=prog["rev"].to(dev), dec=decode_coefficients(self.gamma).to(dev),
                  ctx=zeros(n, c) if c else None, mf=zeros(n, 1), slot=prog["slot"].to(dev),
                  frames=zeros(frames + 1, n, 3 + f) if frames > 1 else None,
                  moments=zeros(steps, 4) if moments else None)
        if repaint is not None:
            st.update(kx=zeros(n, 3), kh=zeros(n, f), jstep=zeros(dtype=torch.int32), known=prog["known"].to(dev),
                      jump=prog["jump"].to(dev), xh0=zeros(n, 3 + f), fixed=zeros(n, dtype=torch.uint8))
        self._static = st
        self._graphs = None
        self._graph_key = None
        return st

    def _prepare(self, batch_index: torch.Tensor, mask: torch.Tensor, b: int, context: Optional[torch.Tensor],
                 steps: int, repaint: Optional[Tuple[int, int]] = None, frames: int = 1, moments: bool = False):
        """What every chain does before its first draw: weights, plan and statics for (batch_index, mask) on the
        denoiser's device, and the per-atom context written into the statics.  Returns (statics, batch_index, mask)."""
        dev = batch_index.device
        if dev.type != "cuda":
            raise _lib.BdiffError("GCDMSampler needs the denoiser on a CUDA device (no CPU fallback)")
        if self.cfg.num_context and context is None:
            raise ValueError("property-conditional configuration: `context` [B,C] is required")
        self.net.sync_weights()
        # the plan is keyed on tensor identity: reuse the tensors of the previous call when the topology repeats
        if self._topo is not None:
            pbi, pmask = self._topo
            if pbi.shape == batch_index.shape and torch.equal(pbi, batch_index) and torch.equal(pmask, mask):
                batch_index, mask = pbi, pmask
        self.net.plan(batch_index, mask, b)
        self._topo = (batch_index, mask)
        st = self._statics(int(batch_index.shape[0]), steps, repaint, frames, moments, dev)
        st["mf"].copy_(mask.float().unsqueeze(-1))
        if st["ctx"] is not None:
            st["ctx"].copy_(context.to(dev, torch.float32)[batch_index] * st["mf"])
        return st, batch_index, mask

    @staticmethod
    def _draw(noise: Optional[NoiseFn], *bufs: torch.Tensor) -> None:
        """Fills each buffer in turn with N(0, I) draws: the device generator's, or `noise(shape)`'s when injected."""
        for buf in bufs:
            if noise is None:
                torch.randn(buf.shape, device=buf.device, out=buf)
            else:
                buf.copy_(noise(tuple(buf.shape)))

    def _reverse_step(self, z, ctx, nx, nh, coef, step) -> None:
        h = self.net._handle
        _lib.check(h, _lib.load().bdiff_reverse_step(h, self.net._stream(), _ptr(z), _ptr(ctx), _ptr(nx), _ptr(nh),
                                                     _ptr(coef), _ptr(step)), "bdiff_reverse_step")

    def _write_frame(self, st) -> None:
        """frames[slot[step]] = unnormalize_z(z) (variational_diffusion.py:762-792, 1353-1360), all on the device
        so that it can sit in a captured graph; slot `return_frames` is the dummy row of ops that write no frame."""
        cfg = self.cfg
        a = cfg.num_atom_types
        z, mf = st["z"], st["mf"]
        parts = [z[:, :3] * cfg.norm_values[0], (z[:, 3:3 + a] * cfg.norm_values[1] + cfg.norm_biases[1]) * mf]
        if cfg.include_charges:
            parts.append((z[:, 3 + a:] * cfg.norm_values[2] + cfg.norm_biases[2]) * mf)
        st["frames"].index_copy_(0, st["slot"].index_select(0, st["step"].long().view(1)),
                                 torch.cat(parts, dim=-1).unsqueeze(0))

    def _op(self, st, noise: Optional[NoiseFn]) -> None:
        """One reverse step of the chain at the device counter: a `sample` step, or RePaint's denoise op, which draws the
        known part's noise first (:1661-1667) and then combines the step's z_unknown (:1670-1679) with it."""
        h = self.net._handle
        if st["repaint"]:
            self._draw(noise, st["kx"], st["kh"])
        self._draw(noise, st["nx"], st["nh"])
        self._reverse_step(st["z"], st["ctx"], st["nx"], st["nh"], st["coef"], st["step"])
        if st["repaint"]:
            _lib.check(h, _lib.load().bdiff_repaint_combine(h, self.net._stream(), _ptr(st["z"]), _ptr(st["xh0"]),
                                                            _ptr(st["fixed"]), _ptr(st["kx"]), _ptr(st["kh"]),
                                                            _ptr(st["known"]), _ptr(st["step"])), "bdiff_repaint_combine")
        if st["moments"] is not None:
            # diagnostics only (tests): moments of the latent after this step, written at row `step` on the device
            zx, zh = st["z"][:, :3], st["z"][:, 3:]
            m = torch.stack((zx.abs().mean(), zx.abs().max(), zh.mean(), zh.abs().mean())).view(1, 4)
            st["moments"].index_copy_(0, st["step"].long().view(1), m)
        if st["frames"] is not None:
            self._write_frame(st)
        st["step"].add_(1)

    def _jump(self, st, noise: Optional[NoiseFn]) -> None:
        """RePaint's jump back from s to t = s + jump_length (:1730-1749) at the jump counter."""
        h = self.net._handle
        self._draw(noise, st["nx"], st["nh"])
        _lib.check(h, _lib.load().bdiff_renoise(h, self.net._stream(), _ptr(st["z"]), _ptr(st["nx"]), _ptr(st["nh"]),
                                                _ptr(st["jump"]), _ptr(st["jstep"])), "bdiff_renoise")
        st["jstep"].add_(1)

    def _chain(self, st, noise: Optional[NoiseFn], batch_index: torch.Tensor, mask: torch.Tensor, b: int,
               z_init: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Runs the chain on prepared statics from z_T (or from `z_init`) and decodes z_0: the output of sample /
        inpaint, with the frames in front when the statics have them."""
        lib = _lib.load()
        h = self.net._handle
        if z_init is None:
            # z_T ~ N(0, I) on the zero-CoG subspace (variational_diffusion.py:1322-1328, 1635-1640)
            self._draw(noise, st["nx"], st["nh"])
            _lib.check(h, lib.bdiff_center_noise(h, self.net._stream(), _ptr(st["nx"]), _ptr(st["nh"]), _ptr(st["z"])),
                       "bdiff_center_noise")
        else:
            st["z"].copy_(z_init)
        for name in ("step", "jstep", "frames", "moments"):
            if st.get(name) is not None:
                st[name].zero_()

        bodies = [lambda: self._op(st, noise)]
        if st["num_jumps"]:
            bodies.append(lambda: self._jump(st, noise))
        if self.use_cuda_graph and noise is None:
            # a captured graph bakes in raw pointers: of the statics, and of the library's weights and plan / workspace
            # buffers, which move when a larger topology was planned in between (every bdiff_plan_topology bumps the
            # plan epoch).  The key therefore holds no address of a tensor made per call.
            key = (st["key"], self.net._plan_key, self.net._plan_epoch, self.net._weights_key)
            if self._graph_key != key:
                self._graphs = []
                for body in bodies:
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        body()
                    self._graphs.append(g)
                self._graph_key = key
            bodies = [g.replay for g in self._graphs]
        for jump in st["schedule"]:
            bodies[0]()
            if jump:
                bodies[1]()

        # one forward = prep, node_frames, edge_embed, node_embed, L x (edge_message, node_update), finalize; an op adds
        # k_step (and k_repaint_combine), a jump k_step, the decode k_step
        per_op = self.net.kernels_per_forward + 1 + (1 if st["repaint"] else 0)
        self.kernel_launches += ((1 if z_init is None else 0) + len(st["schedule"]) * per_op + st["num_jumps"]
                                 + self.net.kernels_per_forward + 1)
        # p(x, h | z_0) (variational_diffusion.py:1378-1387, 840-907), then the CoG fix when no frames are returned
        self._draw(noise, st["nx"], st["nh"])
        _lib.check(h, lib.bdiff_decode_z0(h, self.net._stream(), _ptr(st["z"]), _ptr(st["ctx"]), _ptr(st["nx"]),
                                          _ptr(st["nh"]), _ptr(st["dec"]), _ptr(st["xh"])), "bdiff_decode_z0")
        out = self._finish(st["xh"], batch_index, mask, b, cog_fix=st["frames"] is None)
        if st["frames"] is not None:        # out[0] <- the molecules (:1404-1410, 1780-1786); the last row is the dummy
            out = torch.cat((out.unsqueeze(0), st["frames"][1:-1]), dim=0)
        return out

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
        steps = self.cfg.num_timesteps if num_timesteps is None else int(num_timesteps)
        check_frames(steps, return_frames)
        dev = self._device()
        num_nodes = num_nodes.to(dev, non_blocking=True)
        b = int(num_nodes.shape[0])
        batch_index = torch.repeat_interleave(torch.arange(b, device=dev), num_nodes)
        n = int(batch_index.shape[0])
        mask = torch.ones(n, dtype=torch.bool, device=dev) if node_mask is None else node_mask.to(dev)
        st, batch_index, mask = self._prepare(batch_index, mask, b, context, steps, None, return_frames, record_moments)
        if z_init is not None and tuple(z_init.shape) != (n, 3 + self.cfg.num_h):
            raise ValueError(f"z_init must be [{n}, {3 + self.cfg.num_h}]")
        out = self._chain(st, noise, batch_index, mask, b, z_init)
        self.last_moments = st["moments"].clone() if record_moments else None
        return (out, batch_index, mask, st["z"].clone()) if return_z0 else (out, batch_index, mask)

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
        coef = step_coefficient_table(self.gamma, steps).to(dev)
        idx = torch.tensor(row, dtype=torch.int32, device=dev)
        zz = z.detach().to(torch.float32).clone().contiguous()
        ctx = context.to(torch.float32).contiguous() if self.cfg.num_context else None
        self._reverse_step(zz, ctx, noise_x.to(torch.float32).contiguous(), noise_h.to(torch.float32).contiguous(),
                           coef, idx)
        torch.cuda.current_stream().synchronize()
        return zz

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
        z = self._optimize_latent(cfg, samples, num_nodes, self._device(), node_mask)
        return self.sample(num_nodes, context, num_timesteps, node_mask, noise, z_init=z, return_frames=return_frames)

    @staticmethod
    def _optimize_latent(cfg, samples, num_nodes: torch.Tensor, dev: torch.device,
                         node_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The starting latent of `optimize`: the molecules normalised into z [N, 3+F] on `dev`, after the reference's
        mean-zero assertion, which sums the positions of the whole batch."""
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
        return z

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
        steps = self.cfg.num_timesteps if num_timesteps is None else int(num_timesteps)
        r, j, nfr = int(num_resamplings), int(jump_length), int(return_frames)
        check_repaint(r, j, steps, nfr)
        num_nodes, batch_index, parts, fixed, context = self._inpaint_inputs(self.cfg, molecule, node_mask_fixed, context)
        dev = self._device()
        b = int(num_nodes.shape[0])
        n = int(batch_index.shape[0])
        batch_index = batch_index.to(dev)
        mask = torch.ones(n, dtype=torch.bool, device=dev)          # inpaint has no padding mask (:1638)
        st, batch_index, mask = self._prepare(batch_index, mask, b, context, steps, (r, j), nfr)   # context: (:1614-1615)

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
        return self._chain(st, noise, batch_index, mask, b)

"""Denoiser dimensions, derived from the reference's five Hydra config groups.

Mirrors what GCPNetDynamics.__init__ reads (reference src/models/components/gcpnet.py:933-1039) and rejects
loudly every option the CUDA kernels do not implement (they implement exactly the shipped configs:
configs/model/{model_cfg,module_cfg,layer_cfg,diffusion_cfg}/*.yaml).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Any, Dict, Optional, Tuple


def _get(cfg: Any, key: str, default=None):
    if cfg is None:
        return default
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


@dataclass(frozen=True)
class DenoiserConfig:
    num_atom_types: int = 5
    include_charges: bool = True
    num_context: int = 0
    num_layers: int = 9
    h_hidden: int = 256
    chi_hidden: int = 32
    e_hidden: int = 64
    xi_hidden: int = 16
    num_timesteps: int = 1000
    noise_precision: float = 1e-5
    noise_schedule: str = "polynomial_2"
    norm_values: Tuple[float, float, float] = (1.0, 4.0, 10.0)
    norm_biases: Tuple[Optional[float], float, float] = (None, 0.0, 0.0)

    @property
    def num_h(self) -> int:
        return self.num_atom_types + int(self.include_charges)

    @property
    def h_in(self) -> int:
        return self.num_h + 1 + self.num_context

    @staticmethod
    def named(name: str) -> "DenoiserConfig":
        """The three shipped configurations (SURVEY.md §8)."""
        if name == "qm9":
            return DenoiserConfig()
        if name == "qm9_cond":   # configs/experiment/qm9_mol_gen_conditional_ddpm.yaml (alpha)
            return DenoiserConfig(include_charges=False, num_context=1, norm_values=(1.0, 8.0, 1.0))
        if name == "geom":
            return DenoiserConfig(num_atom_types=16, include_charges=False, num_layers=4, e_hidden=16, xi_hidden=8)
        raise ValueError(f"unknown config '{name}'")

    @staticmethod
    def from_reference_cfgs(model_cfg, module_cfg, layer_cfg, diffusion_cfg, dataloader_cfg) -> "DenoiserConfig":
        def require(cond, msg):
            if not cond:
                raise NotImplementedError(f"GCPNetDynamicsB200: unsupported configuration — {msg}")

        require(_get(diffusion_cfg, "diffusion_target", "atom_types_and_coords") == "atom_types_and_coords",
                "diffusion_target must be atom_types_and_coords")
        require(not _get(diffusion_cfg, "self_condition", False), "self_condition=true")
        require(_get(diffusion_cfg, "condition_on_time", True), "condition_on_time=false")
        require(_get(module_cfg, "vector_gate", True), "vector_gate=false")
        require(not _get(module_cfg, "frame_gate", False), "frame_gate=true")
        require(_get(module_cfg, "scalar_gate", 0) == 0, "scalar_gate>0")
        require(not _get(module_cfg, "vector_residual", False), "vector_residual=true")
        require(_get(module_cfg, "bottleneck", 4) == 4 and _get(module_cfg, "default_bottleneck", 4) == 4, "bottleneck!=4")
        require(_get(module_cfg, "norm_x_diff", True), "norm_x_diff=false")
        require(not _get(module_cfg, "ablate_frame_updates", False) and not _get(module_cfg, "ablate_scalars", False)
                and not _get(module_cfg, "ablate_vectors", False), "ablations")
        require(float(_get(module_cfg, "node_positions_weight", 1.0)) == 1.0, "node_positions_weight!=1")
        require(not _get(module_cfg, "update_positions_with_vector_sum", False), "update_positions_with_vector_sum")
        nl = _get(module_cfg, "nonlinearities", ["silu", "silu"])
        require(list(nl) == ["silu", "silu"], "nonlinearities must be (silu, silu)")
        sel = _get(module_cfg, "selected_GCP", None)
        if sel is not None:
            target = getattr(sel, "func", sel)
            require(getattr(target, "__name__", "GCP2") == "GCP2", "selected_GCP must be GCP2")
        require(not _get(layer_cfg, "pre_norm", False) and not _get(layer_cfg, "use_gcp_norm", False)
                and not _get(layer_cfg, "use_gcp_dropout", False), "GCP norm / dropout")
        require(_get(layer_cfg, "use_scalar_message_attention", True), "use_scalar_message_attention=false")
        require(_get(layer_cfg, "num_feedforward_layers", 1) == 1, "num_feedforward_layers!=1")
        mp = _get(layer_cfg, "mp_cfg", None)
        require(_get(mp, "num_message_layers", 4) == 4, "num_message_layers!=4")
        require(_get(mp, "use_residual_message_gcp", True), "use_residual_message_gcp=false")
        require(_get(model_cfg, "h_hidden_dim", 256) == 256 and _get(model_cfg, "chi_hidden_dim", 32) == 32,
                "node hidden dims must be (256, 32)")
        require(_get(model_cfg, "chi_input_dim", 2) == 2 and _get(model_cfg, "e_input_dim", 1) == 1
                and _get(model_cfg, "xi_input_dim", 1) == 1, "input dims must be chi 2, e 1, xi 1")
        require(float(_get(model_cfg, "dropout", 0.0)) == 0.0, "dropout>0")
        require(_get(dataloader_cfg, "num_x_dims", 3) == 3, "num_x_dims!=3")
        nv = _get(diffusion_cfg, "norm_values", [1.0, 4.0, 10.0])
        nb = _get(diffusion_cfg, "norm_biases", [None, 0.0, 0.0])
        return DenoiserConfig(
            num_atom_types=int(_get(dataloader_cfg, "num_atom_types")),
            include_charges=bool(_get(dataloader_cfg, "include_charges")),
            num_context=len(_get(module_cfg, "conditioning", []) or []),
            num_layers=int(_get(model_cfg, "num_encoder_layers")),
            e_hidden=int(_get(model_cfg, "e_hidden_dim")), xi_hidden=int(_get(model_cfg, "xi_hidden_dim")),
            num_timesteps=int(_get(diffusion_cfg, "num_timesteps", 1000)),
            noise_precision=float(_get(diffusion_cfg, "noise_precision", 1e-5)),
            noise_schedule=str(_get(diffusion_cfg, "noise_schedule", "polynomial_2")),
            norm_values=tuple(float(v) for v in nv), norm_biases=tuple(nb))


def parameter_shapes(cfg: DenoiserConfig) -> Dict[str, Tuple[int, ...]]:
    """Reference parameter names -> shapes: the checkpoint contract (`ddpm.dynamics_network.<name>`)."""
    sh: Dict[str, Tuple[int, ...]] = {}

    def gcp(p, s_in, v_in, s_out, v_out, bott, ff=False):
        hid = v_in // bott if bott > 1 else max(v_in, v_out)
        sh[p + "vector_down.weight"] = (hid, v_in)
        fan = hid + s_in + 9
        if ff:
            sh[p + "scalar_out.0.weight"] = (s_out, fan)
            sh[p + "scalar_out.0.bias"] = (s_out,)
            sh[p + "scalar_out.2.weight"] = (s_out, s_out)
            sh[p + "scalar_out.2.bias"] = (s_out,)
        else:
            sh[p + "scalar_out.weight"] = (s_out, fan)
            sh[p + "scalar_out.bias"] = (s_out,)
        sh[p + "vector_down_frames.weight"] = (3, v_in)
        if v_out:
            sh[p + "vector_up.weight"] = (v_out, hid)
            sh[p + "vector_out_scale.weight"] = (v_out, s_out)
            sh[p + "vector_out_scale.bias"] = (v_out,)

    H, Cc, E, X = cfg.h_hidden, cfg.chi_hidden, cfg.e_hidden, cfg.xi_hidden
    gcp("gcp_embedding.edge_embedding.", 1, 1, E, X, 1)
    gcp("gcp_embedding.node_embedding.", cfg.h_in, 2, H, Cc, 1)
    for l in range(cfg.num_layers):
        p = f"interaction_layers.{l}."
        gcp(p + "interaction.message_fusion.0.", 2 * H + E, 2 * Cc + X, H, Cc, 4)
        for k in range(1, 4):
            gcp(p + f"interaction.message_fusion.{k}.", H, Cc, H, Cc, 4)
        sh[p + "interaction.scalar_message_attention.0.weight"] = (1, H)
        sh[p + "interaction.scalar_message_attention.0.bias"] = (1,)
        gcp(p + "feedforward_network.0.", 2 * H, 2 * Cc, H, Cc, 4, ff=True)
        gcp(p + "node_position_update_gcp.", H, Cc, H, 1, 4)
    gcp("scalar_node_projection_gcp.", H, Cc, cfg.h_in, 0, 1)
    return sh

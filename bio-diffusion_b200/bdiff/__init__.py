"""bdiff — H100-native GCPNet denoiser hot path of GCDM (bio-diffusion).

Public surface (mirrors the reference's seam, SURVEY.md §8b):
    GCPNetDynamicsB200   drop-in for src.models.components.gcpnet.GCPNetDynamics
    GCDMSampler          inner loop of EquivariantVariationalDiffusion.mol_gen_sample (sample(seed=) runs it natively)
    philox_noise         NoiseFn replaying the counter-based draws of the native chain (bdiff_sample)
    GCDMEvalNLL          evaluation-mode NLL terms of EquivariantVariationalDiffusion.forward (forward only)
    GCDMTrainLoss        training-mode L2 objective of the same function (value only, no backward)
    check_molecular_stability_batch   the reference's check_molecular_stability for a whole sampled batch in one kernel
    GCDMTrainTail        adaptive clipping + AdamW(amsgrad) + EMA of a training step as three multi-tensor kernels
    training_state / load_training_state            save and resume a library training run bit for bit
    from_reference_checkpoint / to_reference_checkpoint   move a run to and from the reference's Lightning checkpoints
    PropertyClassifier   EDM's EGNN property classifier (inference), packed molecules, drop-in for get_classifier's model
    DenoiserConfig       dims derived from the reference's Hydra config groups
"""
from .config import DenoiserConfig, parameter_shapes
from .dynamics import GCPNetDynamicsB200
from .sampler import GCDMSampler
from .noise import philox_noise
from .loss import GCDMEvalNLL, GCDMTrainLoss
from .optim import GCDMTrainTail
from .checkpoint import (training_state, load_training_state, from_reference_checkpoint, to_reference_checkpoint,
                         reference_to_training_state, training_state_to_reference)
from .stability import check_molecular_stability_batch
from .classifier import PropertyClassifier
from .datasets import QM9_N_NODES, GEOM_N_NODES, sample_num_nodes
from ._lib import BdiffError, load as load_library

__all__ = ["DenoiserConfig", "parameter_shapes", "GCPNetDynamicsB200", "GCDMSampler", "philox_noise", "GCDMEvalNLL", "GCDMTrainLoss", "GCDMTrainTail", "training_state", "load_training_state", "from_reference_checkpoint", "to_reference_checkpoint", "reference_to_training_state", "training_state_to_reference", "check_molecular_stability_batch", "PropertyClassifier", "QM9_N_NODES", "GEOM_N_NODES", "sample_num_nodes", "BdiffError", "load_library"]

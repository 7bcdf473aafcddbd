"""Synthetic padded datasets for the packed-collation tests (tests/test_collate_oracle.py, tests/test_gpu_collate_layouts.py)
and the plain torch expression of the batch the reference builds from them, restricted to the present atoms.

A dataset has M molecules padded to P slots with A atom types, in the reference's layout (positions [M,P,3] float32,
charges [M,P] int64, one_hot [M,P,A] bool, one float32 [M] tensor per property).  The present-atom patterns are what the
collation kernels must get right: a molecule whose only atom is in slot P - 1, molecules with no atom (charges 0, or
negative), a full molecule, dense prefixes as in QM9 / GEOM, and random holes across the 32-slot warp windows.
"""
import torch

PADS = [29, 31, 32, 33, 64, 181, 200]
NUM_TYPES = [5, 16]
PROPS = ("p0", "p1", "p2")
# batches of molecule ids: 1 molecule, exactly one CTA of 8 warps, one warp into a second CTA, and 1 000+ (many CTAs),
# unsorted and with repeats; each gathers 1 to 3 conditioning properties in a different order
BATCHES = {"one": ("p2",), "eight": ("p1", "p0"), "nine": ("p0", "p1", "p2"), "many": ("p2", "p0", "p1")}
LAST_SLOT_ONLY, EMPTY, EMPTY_NEGATIVE, FULL = 0, 1, 2, 3


def padded_dataset(pad: int, num_types: int, num_mols: int = 300, seed: int = 0):
    g = torch.Generator().manual_seed(seed * 1000 + pad * 17 + num_types)
    present = torch.zeros((num_mols, pad), dtype=torch.bool)
    present[LAST_SLOT_ONLY, pad - 1] = True
    present[FULL] = True
    for m in range(FULL + 1, num_mols):
        if m % 2:                                                # dense prefix, as the datasets store molecules
            present[m, : int(torch.randint(1, pad + 1, (1,), generator=g))] = True
        else:                                                    # holes anywhere, with a per-molecule density
            present[m] = torch.rand(pad, generator=g) < float(torch.rand(1, generator=g)) * 0.9 + 0.05
    charges = torch.where(present, torch.randint(1, 36, (num_mols, pad), generator=g), torch.zeros((), dtype=torch.int64))
    charges[EMPTY_NEGATIVE] = -1                                 # no atom: only charge > 0 marks a present slot
    charges[(torch.rand((num_mols, pad), generator=g) < 0.05) & ~present] = -1
    types = torch.randint(0, num_types, (num_mols, pad), generator=g)
    one_hot = torch.nn.functional.one_hot(types, num_types).bool()
    one_hot[~present] = torch.rand((int((~present).sum()), num_types), generator=g) < 0.5   # padding holds garbage
    data = {"positions": torch.randn((num_mols, pad, 3), generator=g) * 3.0, "charges": charges, "one_hot": one_hot}
    norms = {}
    for c, k in enumerate(PROPS):
        data[k] = torch.randn(num_mols, generator=g) * (10.0 ** c) + 5.0 * c
        norms[k] = {"mean": data[k].mean(), "mad": (data[k] - data[k].mean()).abs().mean()}
    return data, norms


def batch_ids(kind: str, num_mols: int, seed: int = 0) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    if kind == "one":
        return torch.tensor([LAST_SLOT_ONLY])
    if kind == "eight":
        return torch.tensor([7, LAST_SLOT_ONLY, 250, 7, EMPTY, 12, FULL, 3])
    if kind == "nine":
        return torch.tensor([num_mols - 1, 40, EMPTY_NEGATIVE, 41, 40, 9, LAST_SLOT_ONLY, 100, 5])
    if kind == "many":
        ids = torch.cat((torch.randint(0, num_mols, (1033,), generator=g),
                         torch.tensor([LAST_SLOT_ONLY, EMPTY, EMPTY_NEGATIVE, FULL])))
        return ids[torch.randperm(ids.numel(), generator=g)]
    raise ValueError(kind)


def packed_reference(data, norms, idx, conditioning):
    """The reference batch (positions, one_hot, charges as float32, batch vector, prepare_context's normalised properties)
    restricted to mask = charges > 0, as plain torch expressions; fp32 (p - mean) / mad rounds each operation once."""
    idx = torch.as_tensor(idx, dtype=torch.int64)
    mask = data["charges"][idx] > 0
    batch = torch.arange(idx.numel()).unsqueeze(1).expand_as(mask)[mask]
    ref = {"x": data["positions"][idx][mask], "one_hot": data["one_hot"][idx][mask].float(),
           "charges": data["charges"][idx][mask].float().unsqueeze(1), "batch": batch, "counts": mask.sum(1)}
    if conditioning:
        p = torch.stack([data[k] for k in conditioning], 1)
        mean = torch.stack([norms[k]["mean"] for k in conditioning])
        mad = torch.stack([norms[k]["mad"] for k in conditioning])
        ref["context"] = (p[idx[batch]] - mean) / mad
    return ref

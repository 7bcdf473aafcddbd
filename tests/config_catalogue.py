"""Denoiser configurations beyond the three shipped ones, shared by test_configs_cpu.py and test_gpu_configs.py.

`bdiff_create` accepts e_hidden in {4, 8, .., 64}, xi_hidden in {4, 8, 12, 16}, Hin = num_h + 1 + num_context in [2, 28]
and 1..64 layers; tensor mode only the (e_hidden, xi_hidden) pairs (64, 16) and (16, 8).  Each entry of CONFIGS names one
such configuration with its weight seed and scale and the LAYOUTS (layout_catalogue.py) it runs on.  `derived_dims`
restates the dims bdiff_create derives (hid0, K0, Ke, Kn), which edge-embedding kernel runs and whether tensor mode
accepts the configuration; `config_classes` says which of CLASSES an entry reaches.
"""
from dataclasses import dataclass
from typing import Tuple

import gcpnet_oracle as O

TPE_PAIRS = ((64, 16), (16, 8))   # (Ed, Xd) of the templated k_edge_embed_tpe (launch_edge_embed)
TC_PAIRS = ((64, 16), (16, 8))    # (Ed, Xd) of tensor mode (tc_supported in bdiff_layers_tc.cu)

# what the catalogue as a whole must reach
CLASSES = {
    "Hin = 2", "Hin = 28", "Kn in (64, 72)", "Kn = 72", "C >= 2 on the QM9 dims", "generic k_edge_embed",
    "(Ed, Xd) = (64, 4)", "(Ed, Xd) = (16, 16)", "Ed = 4, Xd = 4", "Xd = 12", "Ke = 28", "L = 1 parity",
    "L = 1 tensor", "9 < L < 64 tensor", "L = 64 tensor", "tensor with Hin not 7 or 17", "tensor at Hin = 28",
    "parity K0 not 96 or 44",
}


def _round4(v):
    return (v + 3) // 4 * 4


@dataclass(frozen=True)
class ConfigCase:
    name: str
    num_atom_types: int
    include_charges: bool
    num_context: int
    num_layers: int
    e_hidden: int
    xi_hidden: int
    seed: int
    scale: float                    # weight scale of every oracle comparison of the entry (see test_gpu_configs.py)
    layouts: Tuple[str, ...]        # names in layout_catalogue.LAYOUTS; layouts[0] is the training layout

    def oracle(self) -> O.OracleConfig:
        return O.OracleConfig(num_atom_types=self.num_atom_types, include_charges=self.include_charges,
                              num_context=self.num_context, num_layers=self.num_layers, e_hidden=self.e_hidden,
                              xi_hidden=self.xi_hidden)

    def denoiser(self):
        from bdiff.config import DenoiserConfig
        return DenoiserConfig(num_atom_types=self.num_atom_types, include_charges=self.include_charges,
                              num_context=self.num_context, num_layers=self.num_layers, e_hidden=self.e_hidden,
                              xi_hidden=self.xi_hidden)

    @property
    def tensor(self) -> bool:
        return (self.e_hidden, self.xi_hidden) in TC_PAIRS


_P = ("sparse_mask_qm9", "ascending_1_to_29")          # parity entries: a masked batch and every row length 1..29
_T = _P + ("cut_1_127", "empty_mols_qm9")              # tensor entries add a row cut 1 + 127 and empty molecules

CONFIGS = [
    ConfigCase("hin2", 1, False, 0, 2, 20, 8, seed=31, scale=0.7, layouts=_P),
    ConfigCase("hin28_e16x16", 16, True, 10, 2, 16, 16, seed=32, scale=0.7, layouts=_P),
    ConfigCase("hin25_e64x4_l1", 5, False, 19, 1, 64, 4, seed=33, scale=0.7, layouts=_P),
    ConfigCase("e4x4_l1", 5, True, 0, 1, 4, 4, seed=34, scale=0.7, layouts=_P),
    ConfigCase("e32x12_c3", 5, True, 3, 2, 32, 12, seed=35, scale=0.7, layouts=_P),
    ConfigCase("qm9_c2", 5, False, 2, 9, 64, 16, seed=37, scale=0.7, layouts=_T),
    ConfigCase("qm9_l1", 5, True, 0, 1, 64, 16, seed=38, scale=0.7, layouts=_T),
    ConfigCase("geom_l12", 16, False, 0, 12, 16, 8, seed=39, scale=0.7, layouts=_T),
    ConfigCase("geom_l64", 16, False, 0, 64, 16, 8, seed=40, scale=0.4,
               layouts=("sparse_mask_qm9", "tiny_1", "empty_mols_qm9")),
    ConfigCase("geom_hin28", 16, True, 10, 4, 16, 8, seed=41, scale=0.7, layouts=_T),
]
BY_NAME = {c.name: c for c in CONFIGS}


def derived_dims(c: ConfigCase):
    """The dims bdiff_create derives (bdiff_api.cu) and the kernels they select."""
    hin = c.num_atom_types + int(c.include_charges) + 1 + c.num_context
    hid0 = (64 + c.xi_hidden) // 4
    return dict(hin=hin, hid0=hid0, K0=_round4(c.e_hidden + hid0 + 9), Ke=_round4(1 + c.xi_hidden + 9),
                Kn=_round4(hin + 32 + 9),
                edge_embed="tpe" if (c.e_hidden, c.xi_hidden) in TPE_PAIRS else "generic", tensor=c.tensor)


def config_classes(c: ConfigCase):
    d = derived_dims(c)
    ed, xd, L = c.e_hidden, c.xi_hidden, c.num_layers
    got = set()
    if d["hin"] == 2:
        got.add("Hin = 2")
    if d["hin"] == 28:
        got.add("Hin = 28")
    if 64 < d["Kn"] < 72:
        got.add("Kn in (64, 72)")
    if d["Kn"] == 72:
        got.add("Kn = 72")
    if c.num_context >= 2 and (ed, xd) == (64, 16) and c.num_atom_types == 5:
        got.add("C >= 2 on the QM9 dims")
    if d["edge_embed"] == "generic":
        got.add("generic k_edge_embed")
    if (ed, xd) in ((64, 4), (16, 16)):
        got.add(f"(Ed, Xd) = ({ed}, {xd})")
    if (ed, xd) == (4, 4):
        got.add("Ed = 4, Xd = 4")
    if xd == 12:
        got.add("Xd = 12")
    if d["Ke"] == 28 and d["edge_embed"] == "generic":      # the width of EmbedSmem::sA
        got.add("Ke = 28")
    if d["K0"] not in (96, 44):
        got.add("parity K0 not 96 or 44")
    if L == 1:
        got.add("L = 1 parity")
        if c.tensor:
            got.add("L = 1 tensor")
    if 9 < L < 64 and c.tensor:
        got.add("9 < L < 64 tensor")
    if L == 64 and c.tensor:
        got.add("L = 64 tensor")
    if c.tensor and d["hin"] not in (7, 17):
        got.add("tensor with Hin not 7 or 17")
    if c.tensor and d["hin"] == 28:
        got.add("tensor at Hin = 28")
    return got

"""CPU: the stability oracle (oracle/stability_oracle.py) against the unmodified reference function's outputs stored in
tests/golden/stability.pt (tests/golden/make_golden_stability.py): identical integers for every molecule, up to GEOM's
largest (181 atoms), where the reference's torch.cdist uses its matmul formulation and the oracle the direct distance."""
import os

import numpy as np
import pytest
import torch

import stability_oracle as SO
from conftest import GOLDEN


@pytest.mark.parametrize("name", ["qm9", "geom", "geom_large"])
def test_oracle_matches_reference_function(name):
    fx = torch.load(os.path.join(GOLDEN, "stability.pt"), weights_only=False)[name]
    off = np.concatenate(([0], np.cumsum(fx["sizes"])))
    mask = SO.allowed_mask(fx["atom_decoder"], fx["allowed_bonds"])
    nb, ns, ms = SO.check_stability_batch(fx["x"].numpy(), fx["atom_types"].numpy(), off, fx["bonds"], fx["margins"], mask)
    for k, (st, n_st, n) in enumerate(fx["ref"]):
        assert (bool(ms[k]), int(ns[k]), int(off[k + 1] - off[k])) == (st, n_st, n), k
    if name == "geom_large":                    # past one 128-thread stride of the kernel, up to GEOM's largest molecule
        assert fx["sizes"][:3] == [129, 150, 181] and len(fx["sizes"]) > 200
    if name == "qm9":
        assert [r[0] for r in fx["ref"]][-4:] == [True, True, True, False]      # methane, water, H2, stretched H2
    assert nb.min() >= 0


def test_allowed_mask_int_and_list():
    m = SO.allowed_mask(["H", "P"], {"H": 1, "P": [3, 5]})
    assert m.tolist() == [0b10, 0b101000]


@pytest.mark.parametrize("name", ["qm9", "geom", "geom_large"])
def test_bond_order_oracle_matches_reference_graph(name):
    """E of make_mol_edm (rdkit_functions.py:287-296) computed by the reference's own get_bond_order_batch (stored in the
    fixture) vs the oracle restatement: identical integer matrices, including methane's 4 single bonds.  geom_large stores
    the matrices of its first three molecules (129, 150 and 181 atoms) only."""
    fx = torch.load(os.path.join(GOLDEN, "stability.pt"), weights_only=False)[name]
    off = np.concatenate(([0], np.cumsum(fx["sizes"])))
    for k, e_ref in enumerate(fx["bond_E"]):
        a, b = int(off[k]), int(off[k + 1])
        e = SO.bond_order_matrix(fx["x"].numpy()[a:b], fx["atom_types"].numpy()[a:b], fx["bonds"], fx["margins"],
                                 limit_bonds_to_one=fx["limit_bonds_to_one"])
        assert np.array_equal(e, e_ref.numpy().astype(np.int64)), k
    if name == "qm9":
        ch4 = fx["bond_E"][-4].numpy()
        assert ch4.sum() == 4 and (ch4[1:, 0] == 1).all()

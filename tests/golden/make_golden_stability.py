#!/usr/bin/env python
"""Golden fixture for the batched stability check (SURVEY.md §8 f1): inputs, the reference's own tables (as data) and
the outputs of the UNMODIFIED reference function `check_molecular_stability` (src/datamodules/components/edm/
__init__.py:91-124) per molecule, imported through oracle/ref_shim.py in the build container.
Run:  python tests/golden/make_golden_stability.py"""
import os
import sys

import numpy as np
import torch
import torch._dynamo  # noqa: F401  (before the stub modules are installed)

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_shim  # noqa: E402
from stability_oracle import bond_orders_from_distances, direct_distances, lattice_molecule  # noqa: E402

ref_shim.install()
from src.datamodules.components.edm import check_molecular_stability, get_bond_length_arrays, get_bond_order_batch  # noqa: E402
import src.datamodules.components.edm.constants as K  # noqa: E402
from src.datamodules.components.edm.datasets_config import QM9_WITH_H, GEOM_WITH_H  # noqa: E402


def handmade(enc):
    """Methane, water, H2 and a stretched (broken) H2: stable / stable / stable / unstable."""
    t = 1.09 / np.sqrt(3.0)
    ch4 = (np.array([[0, 0, 0], [t, t, t], [t, -t, -t], [-t, t, -t], [-t, -t, t]], dtype=np.float32),
           np.array([enc["C"], enc["H"], enc["H"], enc["H"], enc["H"]]))
    h2o = (np.array([[0, 0, 0], [0.96, 0, 0], [-0.24, 0.93, 0]], dtype=np.float32), np.array([enc["O"], enc["H"], enc["H"]]))
    h2 = (np.array([[0, 0, 0], [0.74, 0, 0]], dtype=np.float32), np.array([enc["H"], enc["H"]]))
    h2x = (np.array([[0, 0, 0], [1.40, 0, 0]], dtype=np.float32), np.array([enc["H"], enc["H"]]))
    return [ch4, h2o, h2, h2x]


def case(info, sizes, seed, spacing, extra=False, num_E=None):
    """num_E: store the bond-order matrices of the first num_E molecules only (all by default), to keep the fixture small."""
    rng = np.random.default_rng(seed)
    dec = list(info["atom_decoder"])
    enc = dict(info["atom_encoder"])
    b = get_bond_length_arrays(enc)
    di = dict(info)
    di["bonds1"], di["bonds2"], di["bonds3"] = b
    xs, ts, outs, es = [], [], [], []
    limit = "GEOM" in info["name"]
    mols = [lattice_molecule(rng, n, len(dec), spacing) for n in sizes] + (handmade(enc) if extra else [])
    sizes = [len(t) for _, t in mols]
    margins = (K.margin1, K.margin2, K.margin3)
    pairs = differ = 0
    for k, (p, t) in enumerate(mols):
        st, ns, nn = check_molecular_stability(torch.from_numpy(p), torch.from_numpy(np.asarray(t, dtype=np.int64)), di)
        xs.append(p); ts.append(np.asarray(t, dtype=np.int64)); outs.append((bool(st), int(ns), int(nn)))
        pt, tt = torch.from_numpy(p), torch.from_numpy(np.asarray(t, dtype=np.int64))
        n = len(tt)
        a1, a2 = torch.cartesian_prod(tt, tt).T if n > 1 else (tt.repeat(1), tt.repeat(1))
        # pairs i != j that the reference's torch.cdist (a matmul formulation above 25 atoms) and the oracle's direct
        # distance put in different bond classes
        ref_order = get_bond_order_batch(a1, a2, torch.cdist(pt, pt, p=2.0).reshape(-1), di).view(n, n).numpy()
        off_diag = ~np.eye(n, dtype=bool)
        differ += int((ref_order != bond_orders_from_distances(direct_distances(p), t, b, margins))[off_diag].sum())
        pairs += n * (n - 1)
        if num_E is not None and k >= num_E:
            continue
        # the (A, E) graph make_mol_edm hands to RDKit (rdkit_functions.py:287-296; RDKit itself is not installed here):
        # the reference's own get_bond_order_batch on cartesian_prod(atom_types, atom_types), then tril(-1)
        dists = torch.cdist(pt.unsqueeze(0), pt.unsqueeze(0), p=2).squeeze(0).view(-1)
        e_full = get_bond_order_batch(a1, a2, dists, di, limit_bonds_to_one=limit).view(n, n)
        es.append(torch.tril(e_full, diagonal=-1).to(torch.int8))
    print(f"{info['name']}: {len(mols)} molecules of {min(sizes)}..{max(sizes)} atoms, {pairs} ordered pairs, "
          f"{differ} classified differently by the reference's cdist and the direct distance")
    return dict(atom_decoder=dec, bonds=[np.asarray(v, dtype=np.float32) for v in b],
                margins=margins, allowed_bonds={k: K.allowed_bonds[k] for k in dec},
                sizes=list(sizes), x=torch.from_numpy(np.concatenate(xs)), atom_types=torch.from_numpy(np.concatenate(ts)),
                ref=outs, bond_E=es, limit_bonds_to_one=limit)


def draw_sizes(rng, hist, count):
    """`count` molecule sizes drawn from a dataset's n_nodes histogram {size: molecules}."""
    n = np.array(sorted(hist))
    w = np.array([hist[k] for k in n], dtype=np.float64)
    return [int(v) for v in rng.choice(n, size=count, p=w / w.sum())]


fx = {"qm9": case(QM9_WITH_H, [19, 5, 23, 1, 12, 29, 2, 17], 3, 1.15, extra=True),
      "geom": case(GEOM_WITH_H, [44, 30, 61, 9, 25], 4, 1.3)}
# GEOM molecules past one 128-thread stride of the stability kernel, then a few hundred of QM9 and GEOM sizes, all with
# the GEOM decoder; the bond-order matrices of the three large ones only
rng = np.random.default_rng(5)
large = [129, 150, 181] + draw_sizes(rng, QM9_WITH_H["n_nodes"], 120) + draw_sizes(rng, GEOM_WITH_H["n_nodes"], 120)
fx["geom_large"] = case(GEOM_WITH_H, large, 6, 1.3, num_E=3)
fx["geom_large"]["n_nodes"] = {int(k): int(v) for k, v in GEOM_WITH_H["n_nodes"].items()}   # for drawing GEOM-size batches
torch.save(fx, os.path.join(os.path.dirname(os.path.abspath(__file__)), "stability.pt"))
for k, v in fx.items():
    print(k, "stable molecules", sum(r[0] for r in v["ref"]), "of", len(v["ref"]))

"""CPU restatement of the molecular-stability check (SURVEY.md §8 f1).  TEST INFRASTRUCTURE ONLY.

Follows /root/reference/src/datamodules/components/edm/__init__.py:
  * `get_bond_order_batch`        :61-88   (distances * 100, three table lookups + margins, later assignments overwrite)
  * `check_molecular_stability`   :91-124  (pairwise distances, diagonal zeroed, row sums, `allowed_bonds` membership;
                                            returns (molecule_stable, nr_stable_bonds, n))
with the tables of edm/constants.py (`bonds1/2/3`, `margin1/2/3` = 10/5/3 pm, `allowed_bonds`) passed in as DATA.
One deliberate difference: distances are the direct fp32 expression sqrt((dx*dx + dy*dy) + dz*dz) for every n, while
`torch.cdist` switches to a matmul formulation above 25 atoms (same value up to fp32 round-off, which can only matter for
a pair sitting exactly on a threshold).  Pinned against the reference's own function on the fixtures of
tests/golden/make_golden_stability.py (identical integers on all of them, including molecules of 129, 150 and 181 atoms;
of their 367 714 ordered atom pairs, none is put in a different bond class by cdist and by the direct distance).
"""
import numpy as np


def lattice_molecule(rng, n, a, spacing):
    """Random test molecule: n atoms on a jittered cubic lattice of the given spacing (Å), so that realistic bond lengths
    (and a few too-short / too-long pairs) occur, with uniform random types in [0, a).  Shared by the stability fixture
    generator and the GPU tests."""
    side = int(np.ceil(n ** (1 / 3))) + 1
    grid = np.stack(np.meshgrid(*[np.arange(side)] * 3, indexing="ij"), -1).reshape(-1, 3)
    pick = rng.choice(len(grid), size=n, replace=False)
    pos = grid[pick] * spacing + rng.normal(0, 0.12, size=(n, 3))
    return pos.astype(np.float32), rng.integers(0, a, size=n)


def direct_distances(x):
    """[n, n] fp32 distances of the kernels: sqrt((dx*dx + dy*dy) + dz*dz), each operation rounded to fp32."""
    p = np.asarray(x, dtype=np.float32)
    d = p[:, None, :] - p[None, :, :]
    return np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])


def bond_orders_from_distances(dist, atom_types, bonds, margins, limit_bonds_to_one=False):
    """get_bond_order_batch on an [n, n] matrix of distances in Å (fp32): 0 none, 1 single, 2 double, 3 triple."""
    tt = np.asarray(atom_types, dtype=np.int64)
    b1, b2, b3 = (np.asarray(b, dtype=np.float32) for b in bonds)
    m1, m2, m3 = (np.float32(m) for m in margins)
    dist = np.float32(100.0) * np.asarray(dist, dtype=np.float32)           # :69 "we change the metric"
    idx = (tt[:, None], tt[None, :])
    order = np.zeros(dist.shape, dtype=np.int64)
    order[dist < b1[idx] + m1] = 1                                           # :76-81
    order[dist < b2[idx] + m2] = 2
    order[dist < b3[idx] + m3] = 3
    if limit_bonds_to_one:
        order[order > 1] = 1
    return order


def allowed_mask(atom_decoder, allowed_bonds):
    """bit c of mask[type] set <=> an atom of that type may have c bonds (constants.py `allowed_bonds`: int or list)."""
    out = np.zeros(len(atom_decoder), dtype=np.uint32)
    for i, sym in enumerate(atom_decoder):
        v = allowed_bonds[sym]
        for c in ([v] if isinstance(v, int) else list(v)):
            out[i] |= np.uint32(1) << np.uint32(c)
    return out


def check_stability_batch(x, atom_types, mol_off, bonds, margins, mask, limit_bonds_to_one=False):
    """x [N,3] fp32, atom_types [N] int, mol_off [B+1]; bonds = (b1, b2, b3) [A,A]; returns nr_bonds [N], nr_stable [B],
    mol_stable [B] (all integer arrays)."""
    x = np.asarray(x, dtype=np.float32)
    t = np.asarray(atom_types, dtype=np.int64)
    nb = np.zeros(len(t), dtype=np.int32)
    nr_stable = np.zeros(len(mol_off) - 1, dtype=np.int32)
    mol_stable = np.zeros(len(mol_off) - 1, dtype=np.int32)
    for k in range(len(mol_off) - 1):
        a, b = int(mol_off[k]), int(mol_off[k + 1])
        p, tt = x[a:b], t[a:b]
        order = bond_orders_from_distances(direct_distances(p), tt, bonds, margins, limit_bonds_to_one)
        np.fill_diagonal(order, 0)                                           # :111
        s = order.sum(axis=1)
        nb[a:b] = s
        ok = [(int(c) < 32 and (int(mask[ti]) >> int(c)) & 1) for ti, c in zip(tt, s)]   # :114-121
        nr_stable[k] = int(sum(ok))
        mol_stable[k] = int(nr_stable[k] == b - a)
    return nb, nr_stable, mol_stable


def bond_order_matrix(x, atom_types, bonds, margins, limit_bonds_to_one=False):
    """E of `make_mol_edm` (rdkit_functions.py:287-296) for ONE molecule: tril(get_bond_order_batch(type_i, type_j, dist), -1)
    as an int [n, n] array (atoms1, atoms2 = cartesian_prod(atom_types, atom_types).T -> (type_i, type_j) at i*n + j)."""
    order = bond_orders_from_distances(direct_distances(x), atom_types, bonds, margins, limit_bonds_to_one)
    return np.tril(order, -1)

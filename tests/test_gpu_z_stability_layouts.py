"""GPU: bdiff_check_stability and bdiff_bond_orders against the oracle (oracle/stability_oracle.py) on the batch layouts
the small fixtures of test_gpu_z_stability.py leave out — integers, bit-exact, with both decoders (QM9, 5 types; GEOM,
16 types) and both `limit_bonds_to_one` settings on both kernels:

  * molecules of 0 .. 300 atoms in one batch, so the stability kernel's 128-thread row stride runs one, two and three
    passes and the bond-order kernel's 256-thread pair stride many, with the empty molecule first, in the middle and last;
  * every threshold of every type pair and bond order, on a 2-atom molecule one float below, on and one float above it;
  * bond counts far above 32 (the bound of the `allowed` bit mask), and counts of 33 .. 36 that a shift taken modulo 32
    would turn into allowed valences;
  * a 4 096-molecule batch of GEOM sizes, the batch `sample_and_analyze` checks at once;
  * GEOM molecules of up to 181 atoms against the unmodified reference's own outputs (tests/golden/stability.pt,
    `geom_large`).
"""
import os

import numpy as np
import pytest
import torch

import stability_oracle as SO
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

F32 = np.float32


def _fixture(name):
    return torch.load(os.path.join(GOLDEN, "stability.pt"), weights_only=False)[name]


def _info(fx, limit):
    """dataset_info for both kernels; bond_orders_batch takes limit_bonds_to_one from the dataset name, as the reference."""
    return {"atom_decoder": fx["atom_decoder"], "bonds1": fx["bonds"][0], "bonds2": fx["bonds"][1],
            "bonds3": fx["bonds"][2], "name": "GEOM" if limit else "QM9"}


def run_and_compare(fx, x, t, sizes, limit, stability=True, bond_orders=True):
    """Both kernels on one batch against the oracle: per-atom bond counts, per-molecule stable-atom counts and stability,
    every molecule's E block and the bond row list.  Returns the oracle's (nr_bonds, nr_stable, mol_stable)."""
    from bdiff.stability import bond_orders_batch, check_molecular_stability_batch
    x = np.asarray(x, dtype=np.float32)
    t = np.asarray(t, dtype=np.int64)
    sizes = [int(s) for s in sizes]
    off = np.concatenate(([0], np.cumsum(sizes))).astype(np.int64)
    mask = SO.allowed_mask(fx["atom_decoder"], fx["allowed_bonds"])
    nb, ns, ms = SO.check_stability_batch(x, t, off, fx["bonds"], fx["margins"], mask, limit_bonds_to_one=limit)
    xd, td = torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda()
    if stability:
        stable, nr_stable, n, nr_bonds = check_molecular_stability_batch(
            xd, td, torch.tensor(sizes), _info(fx, limit), fx["allowed_bonds"], fx["margins"], limit_bonds_to_one=limit)
        assert np.array_equal(nr_bonds.cpu().numpy(), nb)
        assert np.array_equal(nr_stable.cpu().numpy(), ns)
        assert np.array_equal(stable.cpu().numpy().astype(np.int32), ms)
        assert n.cpu().tolist() == sizes
    if bond_orders:
        bonds, e, poff = bond_orders_batch(xd, td, torch.tensor(sizes), _info(fx, limit), fx["margins"])
        assert poff.cpu().tolist() == np.concatenate(([0], np.cumsum(np.square(sizes)))).tolist()
        e = e.cpu().numpy()
        blocks, rows = [], []
        for k, nk in enumerate(sizes):
            e_ref = SO.bond_order_matrix(x[off[k]:off[k + 1]], t[off[k]:off[k + 1]], fx["bonds"], fx["margins"],
                                         limit_bonds_to_one=limit)
            blocks.append(e_ref.reshape(-1))
            rows += [(k, int(i), int(j), int(e_ref[i, j])) for i, j in np.argwhere(e_ref)]
        flat = np.concatenate(blocks)
        assert np.array_equal(e[: flat.size].astype(np.int64), flat)
        assert bonds.cpu().tolist() == [list(r) for r in rows]
    return nb, ns, ms


# ------------------------------------------------------------------------------------------------ sizes across the stride
STRIDE_SIZES = [1, 2, 127, 128, 129, 181, 300]
SPACING = {"qm9": 1.15, "geom": 1.3}


@pytest.mark.parametrize("empty_at", ["first", "middle", "last"])
@pytest.mark.parametrize("limit", [False, True], ids=["all_orders", "limit_to_one"])
@pytest.mark.parametrize("name", ["qm9", "geom"])
def test_sizes_across_the_row_stride(name, limit, empty_at):
    """0, 1, 2, 127, 128, 129, 181 and 300 atoms in one batch: rows past 128 (and past 256) of the stability kernel are
    the second (third) pass of its stride, and their bond counts must be there."""
    fx = _fixture(name)
    sizes = list(STRIDE_SIZES)
    sizes.insert({"first": 0, "middle": 4, "last": len(sizes)}[empty_at], 0)
    rng = np.random.default_rng(11)
    mols = [SO.lattice_molecule(rng, n, len(fx["atom_decoder"]), SPACING[name]) for n in sizes]
    x = np.concatenate([p for p, _ in mols])
    t = np.concatenate([tt for _, tt in mols])
    nb, ns, ms = run_and_compare(fx, x, t, sizes, limit)
    off = np.concatenate(([0], np.cumsum(sizes)))
    for k, n in enumerate(sizes):                          # the later passes carry real bonds, and stable atoms occur
        if n > 128:
            assert nb[off[k] + 128: off[k + 1]].any(), n
        if n > 256:
            assert nb[off[k] + 256: off[k + 1]].any(), n
    assert ns.sum() > 0
    k0 = sizes.index(0)
    assert (ns[k0], ms[k0]) == (0, 1)                      # nr_stable_bonds == n == 0: stable, as in the reference


# ------------------------------------------------------------------------------------------------ thresholds
def _scaled(d):
    """The oracle's (and the kernels') distance of two atoms dx apart along x: 100 * sqrt(dx*dx), in fp32."""
    return F32(100.0) * np.sqrt(F32(d) * F32(d))


def threshold_placements(thr):
    """Separations (d_below, d_at, d_above) along x with _scaled(d_below) the largest value < thr, _scaled(d_at) == thr
    when some float d gives thr exactly (else d_at = d_above), and _scaled(d_above) the smallest value > thr; found by
    stepping np.nextafter from thr / 100."""
    up, down = F32(np.inf), F32(-np.inf)
    d = F32(thr / F32(100.0))
    while _scaled(d) >= thr:
        d = np.nextafter(d, down)
    while _scaled(np.nextafter(d, up)) < thr:
        d = np.nextafter(d, up)
    below = d
    at = np.nextafter(below, up)
    above = at
    while _scaled(above) <= thr:
        above = np.nextafter(above, up)
    return below, at, above


@pytest.mark.parametrize("limit", [False, True], ids=["all_orders", "limit_to_one"])
@pytest.mark.parametrize("name", ["qm9", "geom"])
def test_every_bond_threshold_below_on_and_above(name, limit):
    """For every ordered type pair (ti, tj) and order o: thr = fp32(b_o[ti, tj] + m_o) (the margin alone where the table
    holds 0), and three 2-atom molecules whose distance is one float below, exactly on and one float above thr.  All of
    them (2 304 for GEOM) in one launch of each kernel, every bond order as the oracle gives it."""
    fx = _fixture(name)
    a = len(fx["atom_decoder"])
    tabs = [np.asarray(b, dtype=np.float32) for b in fx["bonds"]]
    xs, ts, meta = [], [], []
    exact = 0
    for o in range(3):
        for ti in range(a):
            for tj in range(a):
                thr = tabs[o][ti, tj] + F32(fx["margins"][o])
                below, at, above = threshold_placements(thr)
                assert _scaled(below) < thr < _scaled(above) and _scaled(at) >= thr
                exact += int(_scaled(at) == thr)
                for side, d in enumerate((below, at, above)):
                    xs.append(np.array([[0, 0, 0], [d, 0, 0]], dtype=np.float32))
                    ts.append([ti, tj])
                    meta.append((o, ti, tj, side))
    meta = np.array(meta)
    assert (tabs[1] == 0).any() and (tabs[2] == 0).any()
    assert exact >= 0.9 * 3 * a * a                        # thresholds no float distance hits are tested on both sides
    nb, _, _ = run_and_compare(fx, np.concatenate(xs), np.concatenate(ts), [2] * len(xs), limit)
    order = nb[0::2]                                       # a 2-atom molecule's bond count is its one pair's order
    assert np.array_equal(order, nb[1::2])
    below, at = order[meta[:, 3] == 0], order[meta[:, 3] == 1]
    o, ti, tj = meta[meta[:, 3] == 0, 0], meta[meta[:, 3] == 0, 1], meta[meta[:, 3] == 0, 2]
    # the single-bond threshold is the largest of the three: every pair is bonded just below it and not on it
    assert (below[o == 0] == 1).all() and (at[o == 0] == 0).all()
    if not limit:                                          # a listed double / triple bond appears just below its threshold
        for oo in (1, 2):
            listed = (o == oo) & (tabs[oo][ti, tj] > 0)
            assert listed.any() and (below[listed] == oo + 1).all() and (at[listed] == oo).all()


# ------------------------------------------------------------------------------------------------ saturated counts
def _ball(rng, n, radius=0.3):
    v = rng.normal(size=(n, 3))
    v *= (radius * rng.random(n) ** (1 / 3) / np.linalg.norm(v, axis=1))[:, None]
    return v.astype(np.float32)


@pytest.mark.parametrize("limit", [False, True], ids=["all_orders", "limit_to_one"])
@pytest.mark.parametrize("name", ["qm9", "geom"])
def test_bond_counts_past_the_allowed_mask(name, limit):
    """181 H/C/N/O atoms inside a 0.3 Å ball (every pair bonded, counts far above 32), and balls of 34 H, 37 C, 35 O and
    36 N atoms, whose counts 33, 36, 34 and 35 are a valence of their type modulo 32: no atom may count as stable."""
    fx = _fixture(name)
    enc = {s: i for i, s in enumerate(fx["atom_decoder"])}
    rng = np.random.default_rng(5)
    hcno = [enc[s] for s in "HCNO"]
    mols = [(_ball(rng, 181), rng.choice(hcno, size=181))]
    mols += [(_ball(rng, n), np.full(n, enc[s])) for s, n in (("H", 34), ("C", 37), ("O", 35), ("N", 36))]
    sizes = [len(tt) for _, tt in mols]
    nb, ns, ms = run_and_compare(fx, np.concatenate([p for p, _ in mols]), np.concatenate([tt for _, tt in mols]),
                                 sizes, limit)
    assert nb.min() >= 33 and not ns.any() and not ms.any()
    if limit:
        assert np.array_equal(nb, np.repeat(np.array(sizes) - 1, sizes))


# ------------------------------------------------------------------------------------------------ a large batch
def test_geom_size_batch_of_4096_molecules():
    """4 096 molecules drawn from GEOM's size histogram, on the jittered lattice: stability as sample_and_analyze
    computes it (all orders) and the bond graph as make_mol_edm builds it for GEOM (orders limited to one)."""
    fx = _fixture("geom")
    hist = _fixture("geom_large")["n_nodes"]
    rng = np.random.default_rng(17)
    n = np.array(sorted(hist))
    sizes = rng.choice(n, size=4096, p=np.array([hist[k] for k in n], dtype=np.float64) / sum(hist.values()))
    mols = [SO.lattice_molecule(rng, int(s), len(fx["atom_decoder"]), 1.3) for s in sizes]
    x = np.concatenate([p for p, _ in mols])
    t = np.concatenate([tt for _, tt in mols])
    nb, ns, _ = run_and_compare(fx, x, t, sizes, limit=False, bond_orders=False)
    assert nb.max() > 0 and ns.sum() > 0
    run_and_compare(fx, x, t, sizes, limit=True, stability=False)


# ------------------------------------------------------------------------------------------------ the reference's outputs
def test_geom_large_fixture_matches_reference():
    """Molecules of 129, 150 and 181 atoms and a few hundred of QM9 and GEOM sizes: (molecule_stable, nr_stable, n) as
    the unmodified reference's check_molecular_stability returned them, and the bond graphs of the three large ones as
    its get_bond_order_batch built them."""
    from bdiff.stability import bond_orders_batch, check_molecular_stability_batch
    fx = _fixture("geom_large")
    info = _info(fx, fx["limit_bonds_to_one"])
    stable, nr_stable, n, _ = check_molecular_stability_batch(
        fx["x"].cuda(), fx["atom_types"].cuda(), torch.tensor(fx["sizes"]), info, fx["allowed_bonds"], fx["margins"])
    got = list(zip(stable.cpu().tolist(), nr_stable.cpu().tolist(), n.cpu().tolist()))
    assert got == [tuple(r) for r in fx["ref"]]
    run_and_compare(fx, fx["x"].numpy(), fx["atom_types"].numpy(), fx["sizes"], limit=False, bond_orders=False)
    bonds, e, poff = bond_orders_batch(fx["x"].cuda(), fx["atom_types"].cuda(), torch.tensor(fx["sizes"]), info,
                                       fx["margins"])
    bonds = bonds.cpu()
    for k, e_ref in enumerate(fx["bond_E"]):
        nk = fx["sizes"][k]
        assert torch.equal(e[int(poff[k]): int(poff[k]) + nk * nk].reshape(nk, nk).cpu(), e_ref), k
        assert bonds[bonds[:, 0] == k, 1:].tolist() == [[i, j, int(e_ref[i, j])] for i, j in torch.nonzero(e_ref).tolist()]


# ------------------------------------------------------------------------------------------------ argument checks
@pytest.mark.parametrize("bad", [-1, "A"])
def test_atom_type_outside_the_decoder_is_rejected(bad):
    """Both entry points reject a type that would index past the [A, A] tables on the device."""
    from bdiff.stability import bond_orders_batch, check_molecular_stability_batch
    fx = _fixture("qm9")
    a = len(fx["atom_decoder"])
    x = torch.zeros((5, 3), device="cuda")
    x[:, 0] = torch.arange(5, dtype=torch.float32)
    t = torch.zeros(5, dtype=torch.int64, device="cuda")
    t[3] = a if bad == "A" else bad
    sizes = torch.tensor([2, 3])
    with pytest.raises(ValueError, match="atom type outside the decoder"):
        bond_orders_batch(x, t, sizes, _info(fx, False), fx["margins"])
    with pytest.raises(ValueError, match="atom type outside the decoder"):
        check_molecular_stability_batch(x, t, sizes, _info(fx, False), fx["allowed_bonds"], fx["margins"])
    t[3] = a - 1                                           # the largest valid type is accepted
    bond_orders_batch(x, t, sizes, _info(fx, False), fx["margins"])

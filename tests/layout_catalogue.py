"""Batch layouts shared by the forward tests (test_gpu_tc_layouts.py) and the training-step tests
(test_gpu_train_layouts.py), with the tiling model of the layer megakernel that says which paths each layout reaches.

A molecule with `na` active atoms has na x na edges, row by row; edge tiles hold 128 edges in eight 16-row windows, node
tiles 32 atoms.  `layout_paths` restates those tiling rules in plain Python (see test_gpu_tc_layouts.py for the paths).
`_inputs` builds a case's seeded inputs: masked xh rows zero, coordinates centred per molecule, t and context per molecule,
for the case's configuration or any other (test_gpu_configs.py).  `host_plan` restates the topology plan with numpy
(test_plan_cpu.py, test_train_hostcheck.py).
"""
from dataclasses import dataclass, field
from typing import List, Tuple

import numpy as np
import torch

import gcpnet_oracle as O

TMT = 128         # edges per edge tile (bdiff_edge_tc.cuh, TMT)
WIN = 16          # rows per segmented-sum window, one warp each (edge_tile_epilogue.inc, wr0 = warp * 16)
R4M = 32          # atoms per node tile (bdiff_node_tc.cuh, R4M)


@dataclass
class Layout:
    name: str
    config: str
    sizes: List[int]
    masked: List[int] = field(default_factory=list)     # masked atom indices (into the concatenated atom list)
    targets: Tuple[str, ...] = ()                        # path classes this case is here to reach
    schedule: bool = False                               # run through profile_forward: a timed-out dependency wait fails
    scale: float = 1.0                                   # weight scale of the oracle comparisons (see below)

    @property
    def n(self):
        return sum(self.sizes)

    def mask(self) -> torch.Tensor:
        m = torch.ones(self.n, dtype=torch.bool)
        m[self.masked] = False
        return m


def _offsets(sizes):
    return np.concatenate(([0], np.cumsum(sizes))).astype(int)


def _mask_mols(sizes, mols):
    """Every atom of molecules `mols`."""
    o = _offsets(sizes)
    return [i for k in mols for i in range(o[k], o[k + 1])]


def _fuzz(config, seed):
    """Fixed-seed random sizes (QM9 1..29, GEOM 1..60 atoms), about 10 % of the atoms masked, 3k..20k edges."""
    rng = np.random.default_rng(1000 + seed + (0 if config == "qm9" else 100))
    hi = 29 if config == "qm9" else 60
    target = int(rng.integers(3000, 20000))
    sizes = []
    while sum(s * s for s in sizes) < target:
        sizes.append(int(rng.integers(1, hi + 1)))
    n = sum(sizes)
    masked = sorted(int(i) for i in np.nonzero(rng.random(n) < 0.1)[0])
    return Layout(f"fuzz_{config}_{seed}", config, sizes, masked, ("row cut once", "masked atom"))


def _sparse(config):
    # [12, 5, 45, 20]: interior masks in molecule 0; molecule 1 has one active atom; molecule 2 (atoms 17..61) keeps its
    # first 5 atoms only, and molecule 3's first two atoms are masked, so node tile 1 (atoms 32..63) has no active atom
    sizes = [12, 5, 45, 20]
    masked = [3, 7, 8] + [12, 13, 15, 16] + list(range(22, 62)) + [62, 63, 70]
    return Layout(f"sparse_mask_{config}", config, sizes, masked,
                  ("masked atom", "one active atom", "node tile without active atoms"))


# The untrained network amplifies round-off with the row length: with full-size random weights, the oracle's own float32
# result misses the float64 one by 8e-5 .. 5e-4 (scaled) on the 128..300-atom molecules, so those cases run with
# half-size weights (float32 vs float64 then within 5e-7), as the teacher-forced steps of test_gpu_parity.py do.
LAYOUTS = [
    Layout("ascending_1_to_29", "qm9", list(range(1, 30)), [],
           ("row inside one window", "row crosses 1 window border", "row crosses 2+ window borders", "row cut once")),
    Layout("row_is_tile", "qm9", [128], [], ("whole-tile row", "row crosses 7 window borders"), scale=0.5),
    Layout("cut_1_127", "qm9", [1, 128], [], ("row cut 1 + 127",), scale=0.5),
    Layout("two_mids", "geom", [1, 258, 3, 300], [], ("2 mid tiles",), scale=0.5),
    Layout("mid_phases", "geom", [130, 131, 129, 181], [], ("1 mid tile", "row cut once"), scale=0.5),
    Layout("empty_mols_qm9", "qm9", [3, 5, 4, 1, 6], _mask_mols([3, 5, 4, 1, 6], [0, 2, 4]),
           ("empty molecule",)),
    Layout("empty_mols_geom", "geom", [40, 27, 64, 50, 33], _mask_mols([40, 27, 64, 50, 33], [0, 2, 4]),
           ("empty molecule", "empty node tile", "masked atom in the GEOM build")),
    _sparse("qm9"),
    _sparse("geom"),
    Layout("node_tile_edges", "geom", [31, 2, 33, 70, 40, 17], [],
           ("molecule straddles a node tile border", "molecule spans 3 node tiles"), schedule=True),
    Layout("tiny_1", "qm9", [1], [], ("E = 1",), schedule=True),
    Layout("tiny_2", "qm9", [2], [], schedule=True),
    Layout("all_masked", "qm9", [3, 4], list(range(7)), ("E = 0",), schedule=True),
    Layout("cond_masked", "qm9_cond", [9, 14, 20, 7], [2, 11, 12, 30, 40, 48], ("masked atom",)),
] + [_fuzz(c, s) for c in ("qm9", "geom") for s in range(3)]

BY_NAME = {c.name: c for c in LAYOUTS}


def layout_paths(sizes, mask, config="qm9"):
    """The paths of k_layers_tc that a batch reaches, from the kernel's tiling rules (see test_gpu_tc_layouts.py)."""
    mask = np.asarray(mask, dtype=bool)
    o = _offsets(sizes)
    paths = set()
    e = 0                          # first edge of the current molecule
    tile_mols = {}                 # edge tile -> molecules with edges in it
    for k in range(len(sizes)):
        act = mask[o[k]:o[k + 1]]
        na = int(act.sum())
        if na == 0:
            paths.add("empty molecule")
        if na == 1 and sizes[k] > 1:
            paths.add("one active atom")
        if na < sizes[k]:
            paths.add("masked atom")
            if config == "geom":
                paths.add("masked atom in the GEOM build")
        if o[k] // R4M != (o[k + 1] - 1) // R4M:
            paths.add("molecule straddles a node tile border")
        if (o[k + 1] - 1) // R4M - o[k] // R4M >= 2:
            paths.add("molecule spans 3 node tiles")
        for a in range(na):
            g0 = e + a * na
            g1 = g0 + na - 1
            t0, t1 = g0 // TMT, g1 // TMT
            for t in range(t0, t1 + 1):
                tile_mols.setdefault(t, set()).add(k)
            if t1 == t0:
                if g0 % TMT == 0 and g1 % TMT == TMT - 1:
                    paths.add("whole-tile row")
            elif t1 == t0 + 1:
                paths.add("row cut once")
                if (t1 * TMT - g0, g1 - t1 * TMT + 1) in ((1, TMT - 1), (TMT - 1, 1)):
                    paths.add("row cut 1 + 127")
            else:
                paths.add(f"{t1 - t0 - 1} mid tile" + ("s" if t1 - t0 > 2 else ""))
            # window borders crossed by each tile's piece of the row (tile borders are not window crossings)
            for t in range(t0, t1 + 1):
                a0, a1 = max(g0, t * TMT), min(g1, t * TMT + TMT - 1)
                c = a1 // WIN - a0 // WIN
                paths.add("row inside one window" if c == 0 else
                          "row crosses 1 window border" if c == 1 else "row crosses 2+ window borders")
                if c == TMT // WIN - 1:
                    paths.add("row crosses 7 window borders")
        e += na * na
    tn = (o[-1] + R4M - 1) // R4M
    if e == 0:
        paths.add("E = 0")
    if e == 1:
        paths.add("E = 1")
    if any(len(m) > 1 for m in tile_mols.values()):
        paths.add("edge tile spans molecules")
    mol_of = np.repeat(np.arange(len(sizes)), sizes)
    for u in range(tn):
        lo, hi = u * R4M, min(o[-1], u * R4M + R4M)
        if not mask[lo:hi].any():
            paths.add("node tile without active atoms")
        # node_dep of bdiff_plan_topology: the edges of the molecules mol_of[lo] .. mol_of[hi - 1]
        if all(mask[o[k]:o[k + 1]].sum() == 0 for k in range(mol_of[lo], mol_of[hi - 1] + 1)):
            paths.add("empty node tile")
    return paths


def host_plan(bi: torch.Tensor, mask: torch.Tensor):
    """The arrays bdiff_plan_topology builds (plan_host in csrc/bdiff_plan.h), restated with numpy: the plan, the per-edge
    records k_edge_rc computes on the device, and the layer megakernel's tables.  edge_dep[t] / node_dep[u] are the
    inclusive ranges of 32-node tiles / 128-edge tiles holding the molecules of edge tile t / node tile u ((0, -1): none);
    node_mid[i] = (first, count) of the edge tiles strictly inside node i's row, for the TN * 32 rows of the node tiles."""
    bi = bi.numpy().astype(np.int64)
    mk = mask.numpy().astype(np.uint8)
    B, N = int(bi.max()) + 1, bi.shape[0]
    mol_off = np.zeros(B + 1, np.int32)
    np.add.at(mol_off, bi + 1, 1)
    mol_off = np.cumsum(mol_off).astype(np.int32)
    act_idx = np.nonzero(mk)[0].astype(np.int32)
    act_off = np.zeros(B + 1, np.int32)
    np.add.at(act_off, bi[act_idx] + 1, 1)
    act_off = np.cumsum(act_off).astype(np.int32)
    na = np.diff(act_off).astype(np.int64)
    edge_off = np.concatenate([[0], np.cumsum(na * na)]).astype(np.int64)
    E = int(edge_off[-1])
    rc = [np.zeros((0, 4), np.int32)]
    for k in range(B):
        act = act_idx[act_off[k]:act_off[k + 1]]
        n = len(act)
        rc.append(np.stack([np.repeat(act, n), np.tile(act, n), np.tile(np.arange(n), n), np.full(n * n, n)], 1))
    rc = np.concatenate(rc).astype(np.int32)
    te, tn = (E + TMT - 1) // TMT, (N + R4M - 1) // R4M
    mol_of_edge = lambda g: np.searchsorted(edge_off[1:], g, side="right")   # molecule holding edge g (g < E)
    g0 = np.arange(te, dtype=np.int64) * TMT
    k0, k1 = mol_of_edge(g0), mol_of_edge(np.minimum(E, g0 + TMT) - 1)
    edge_dep = np.stack([mol_off[k0] // R4M, (mol_off[k1 + 1] - 1) // R4M], 1).astype(np.int32).reshape(te, 2)
    node_dep = np.zeros((tn, 2), np.int32)
    for u in range(tn):
        e0, e1 = edge_off[bi[u * R4M]], edge_off[bi[min(N, u * R4M + R4M) - 1] + 1] - 1
        node_dep[u] = (e0 // TMT, e1 // TMT) if e1 >= e0 else (0, -1)
    node_mid = np.zeros((tn * R4M, 2), np.int32)
    for k in range(B):
        n = int(na[k])
        for a in range(n):
            t0, t1 = (edge_off[k] + a * n) // TMT, (edge_off[k] + a * n + n - 1) // TMT
            if t1 - t0 >= 2:
                node_mid[act_idx[act_off[k] + a]] = (t0 + 1, t1 - t0 - 1)
    return dict(B=B, N=N, E=E, Mact=int(act_idx.shape[0]), TE=te, TN=tn, mol_off=mol_off, act_off=act_off,
                act_idx=act_idx, edge_off=edge_off, node_mol=bi.astype(np.int32), mask=mk, edge_rc=rc,
                edge_dep=edge_dep, node_dep=node_dep, node_mid=node_mid)


def _inputs(c: Layout, ocfg: O.OracleConfig = None):
    """Seeded inputs of a case: masked xh rows are zero, coordinates centred per molecule, t and context per molecule.
    `ocfg` gives the feature and context widths of another configuration than the case's own."""
    ocfg = ocfg or O.config_named(c.config)
    g = torch.Generator().manual_seed(sum(map(ord, c.name)))
    b = len(c.sizes)
    bi = torch.repeat_interleave(torch.arange(b), torch.tensor(c.sizes))
    mask = c.mask()
    xh = torch.randn((c.n, 3 + ocfg.num_h), generator=g) * mask[:, None]
    _, xc = O.centralize(xh[:, :3], bi, mask, b, guard_empty=True)
    xh = torch.cat((xc, xh[:, 3:]), -1)
    t = torch.rand((b, 1), generator=g)[bi]
    ctx = torch.randn((b, ocfg.num_context), generator=g)[bi] if ocfg.num_context else None
    return bi, mask, xh, t, ctx


def _active_mol_rows(c: Layout) -> torch.Tensor:
    """Rows of molecules with at least one active atom."""
    mask = c.mask()
    o = _offsets(c.sizes)
    keep = torch.zeros(c.n, dtype=torch.bool)
    for k in range(len(c.sizes)):
        if mask[o[k]:o[k + 1]].any():
            keep[o[k]:o[k + 1]] = True
    return keep

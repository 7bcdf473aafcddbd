"""Batch layouts of the layer megakernel against the float64 oracle.

Whether a forward of `k_layers_tc` is right depends mostly on where a molecule's edges fall relative to the kernel's tiles.
A molecule with `na` active atoms has na x na edges, row by row; edge tiles hold 128 edges in eight 16-row windows, node
tiles 32 atoms.  The segmented sum of edge_tile_epilogue.inc takes one of several paths for a source atom's row: it lies in
one window, crosses window borders (joined by `finish_crossing`), is cut by one tile border (two `atomicAdd` addends into
`agg`), or a tile lies strictly inside it (the tile's sum goes to `Work::mid`, the node tile adds those in ascending order).
The schedule adds node tiles without edges and dependency ranges spanning molecules.

LAYOUTS names batches that reach each of these paths.  `layout_paths` restates the tiling rules in plain Python (both
live in layout_catalogue.py, shared with the training-step tests of test_gpu_train_layouts.py); the CPU test checks that
every case reaches what it claims and that the catalogue as a whole reaches every path class.  The GPU tests run every case through tensor mode, parity mode and the training forward and compare each molecule's coordinate and
`h` blocks separately with the oracle in float64, each scaled by max(1, |ref|max) of that molecule and block, so that a
small molecule next to a large one is held to its own scale.

Molecules without active atoms: the reference divides 0 by 0 for their centroid, and its NaN guard then zeroes the
velocity of the whole batch.  The CUDA path takes that centroid as 0 (DESIGN.md §2), so the oracle runs with
guard_empty=True here; the empty molecule's own rows must be finite and agree between the two modes.
"""
import pytest
import torch

import gcpnet_oracle as O
from layout_catalogue import BY_NAME, LAYOUTS, Layout, _active_mol_rows, _inputs, _offsets, layout_paths

TENSOR_TOL = 1e-4   # tensor mode (split-bf16 wgmma), as tests/test_gpu_tc.py
PARITY_TOL = 5e-5   # parity mode and the training forward (fp32), as tests/test_gpu_parity.py / test_gpu_train.py
WEIGHT_SEED = {"qm9": 7, "qm9_cond": 5, "geom": 3}

# every path class the catalogue as a whole must reach
PATH_CLASSES = {
    "row inside one window", "row crosses 1 window border", "row crosses 2+ window borders",
    "row crosses 7 window borders", "whole-tile row", "row cut once", "row cut 1 + 127", "1 mid tile", "2 mid tiles",
    "edge tile spans molecules", "E = 0", "E = 1", "empty molecule",
    "empty node tile", "node tile without active atoms", "masked atom", "masked atom in the GEOM build",
    "one active atom", "molecule straddles a node tile border", "molecule spans 3 node tiles",
}


def test_layout_catalogue_reaches_every_path():
    """CPU: each case reaches the paths it is in the catalogue for; together they reach every path class."""
    union = set()
    for c in LAYOUTS:
        got = layout_paths(c.sizes, c.mask().numpy(), c.config)
        e = sum(int(c.mask()[o0:o1].sum()) ** 2 for o0, o1 in zip(_offsets(c.sizes)[:-1], _offsets(c.sizes)[1:]))
        print(f"{c.name:20s} {c.config:8s} N={c.n:4d} E={e:6d}: {', '.join(sorted(got))}")
        missing = set(c.targets) - got
        assert not missing, f"{c.name} does not reach {missing}"
        union |= got
    assert PATH_CLASSES <= union, f"no case reaches {PATH_CLASSES - union}"
    for c in LAYOUTS:
        if c.name.startswith("fuzz_"):
            assert 3000 <= sum(s * s for s in c.sizes) and len(c.masked) > 0


def test_layout_paths_model():
    """CPU: the model on layouts whose paths follow from arithmetic alone."""
    assert "whole-tile row" in layout_paths([128], [True] * 128)
    assert "row cut 1 + 127" in layout_paths([1, 128], [True] * 129)
    assert "2 mid tiles" in layout_paths([1, 258], [True] * 259)     # row 63 of the 258: edges 16255..16512 = tiles 126..129
    assert "2 mid tiles" not in layout_paths([258], [True] * 258)    # a lone molecule needs n >= 259
    assert "2 mid tiles" in layout_paths([259], [True] * 259)
    p = layout_paths([3, 4], [False] * 7)
    assert {"E = 0", "empty molecule", "empty node tile"} <= p


def test_oracle_empty_molecule_guard():
    """CPU: the reference's arithmetic on a batch with an all-masked molecule gives NaN coordinates for that molecule and
    zero velocities everywhere else (its NaN guard); guard_empty=True leaves the other molecules' rows as they are without
    the empty molecule's atoms being active."""
    c = BY_NAME["empty_mols_qm9"]
    bi, mask, xh, t, ctx = _inputs(c)
    ocfg = O.config_named(c.config)
    sd = O.random_state_dict(ocfg, WEIGHT_SEED[c.config])
    raw = O.denoiser_forward(sd, ocfg, bi, mask, xh, t, ctx, dtype=torch.float64)
    guarded = O.denoiser_forward(sd, ocfg, bi, mask, xh, t, ctx, dtype=torch.float64, guard_empty=True)
    empty = ~_active_mol_rows(c)
    assert torch.isnan(raw[empty, :3]).all() and (raw[~empty, :3] == 0).all()
    assert torch.isfinite(guarded).all() and (guarded[empty, :3] == 0).all()
    assert guarded[~empty, :3].abs().max() > 0.01
    assert torch.equal(raw[:, 3:], guarded[:, 3:])
    # without an empty molecule the option changes nothing
    c = BY_NAME["cond_masked"]
    bi, mask, xh, t, ctx = _inputs(c)
    ocfg = O.config_named(c.config)
    sd = O.random_state_dict(ocfg, WEIGHT_SEED[c.config])
    assert torch.equal(O.denoiser_forward(sd, ocfg, bi, mask, xh, t, ctx, dtype=torch.float64),
                       O.denoiser_forward(sd, ocfg, bi, mask, xh, t, ctx, dtype=torch.float64, guard_empty=True))


# ------------------------------------------------------------------------------------------------ oracle
_ORACLE = {}


def _oracle(c: Layout) -> torch.Tensor:
    if c.name not in _ORACLE:
        ocfg = O.config_named(c.config)
        sd = O.random_state_dict(ocfg, WEIGHT_SEED[c.config], scale=c.scale)
        bi, mask, xh, t, ctx = _inputs(c)
        _ORACLE[c.name] = O.denoiser_forward(sd, ocfg, bi, mask, xh, t, ctx, dtype=torch.float64, guard_empty=True)
    return _ORACLE[c.name]


def _net(config, mode, scale=1.0):
    import bdiff
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named(config), mode=mode)
    net.load_state_dict(O.random_state_dict(O.config_named(config), WEIGHT_SEED[config], scale=scale), strict=True)
    return net.cuda()


def _cuda_args(c: Layout):
    return tuple(a.cuda() if a is not None else None for a in _inputs(c))


def _check_per_molecule(c: Layout, out: torch.Tensor, tol: float, what: str):
    """Coordinates and h of every non-empty molecule against the oracle, each scaled by max(1, |ref|max) of that block."""
    ref = _oracle(c)
    out = out.detach().cpu().double()
    assert out.shape == ref.shape
    keep = _active_mol_rows(c)
    assert torch.isfinite(out).all(), f"{c.name}/{what}: non-finite output"
    o = _offsets(c.sizes)
    worst = (0.0, None)
    for k in range(len(c.sizes)):
        if not keep[o[k]]:
            continue
        for blk, cols in (("x", slice(0, 3)), ("h", slice(3, None))):
            r, y = ref[o[k]:o[k + 1], cols], out[o[k]:o[k + 1], cols]
            err = (y - r).abs().max().item() / max(1.0, r.abs().max().item())
            if err > worst[0]:
                worst = (err, (k, blk))
            assert err <= tol, (f"{c.name}/{what}: molecule {k} (n={c.sizes[k]}) block {blk}: scaled error {err:.3e} "
                                f"> {tol:.0e}")
    print(f"{c.name}/{what}: worst per-molecule scaled error {worst[0]:.3e} at {worst[1]}")


# ------------------------------------------------------------------------------------------------ GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.name for c in LAYOUTS])
def test_tensor_layout_matches_fp64_oracle(name):
    """k_layers_tc on the case: per-molecule bar 1e-4, two runs bit-identical (the second through profile_forward on the
    scheduling cases, which fails on a timed-out dependency wait)."""
    c = BY_NAME[name]
    net = _net(c.config, "tensor", c.scale)
    args = _cuda_args(c)
    out = net.denoise(*args)
    if c.schedule:
        prof, out2 = net.profile_forward(*args)
        assert "layers_fused" in prof
    else:
        out2 = net.denoise(*args)
    assert torch.equal(out, out2), f"{name}: tensor mode must be run-to-run deterministic"
    _check_per_molecule(c, out, TENSOR_TOL, "tensor")
    keep = _active_mol_rows(c)
    if not keep.all():
        # the rows of an empty molecule: finite, and the same in both modes
        par = _net(c.config, "parity", c.scale).denoise(*args)
        d = (out[~keep.cuda()] - par[~keep.cuda()]).abs().max().item()
        scale = max(1.0, par[~keep.cuda()].abs().max().item())
        print(f"{name}: empty-molecule rows tensor vs parity max|diff| {d:.3e} (scale {scale:.3g})")
        assert torch.isfinite(par).all() and d <= TENSOR_TOL * scale


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.name for c in LAYOUTS])
def test_parity_layout_matches_fp64_oracle(name):
    c = BY_NAME[name]
    net = _net(c.config, "parity", c.scale)
    _check_per_molecule(c, net.denoise(*_cuda_args(c)), PARITY_TOL, "parity")


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c.name for c in LAYOUTS])
def test_train_forward_layout_matches_fp64_oracle(name):
    c = BY_NAME[name]
    net = _net(c.config, "parity", c.scale)
    out = net.denoise_train(*_cuda_args(c))
    _check_per_molecule(c, out, PARITY_TOL, "train forward")


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["qm9", "geom"])
def test_tensor_workspace_reuse_across_layouts(config):
    """One tensor-mode net runs every case of its config, largest first, then the small ones, then the largest again; each
    output is bit-identical to a fresh net's on the same case (stale agg / mid / schedule / flag state would show)."""
    cases = sorted((c for c in LAYOUTS if c.config == config), key=lambda c: -sum(s * s for s in c.sizes))
    order = [cases[0]] + cases[:0:-1] + [cases[0], cases[1]]
    fresh = {c.name: _net(config, "tensor").denoise(*_cuda_args(c)) for c in cases}
    net = _net(config, "tensor")
    alive = []       # the plan is cached by the address of batch_index / mask: keep every input alive so none is reused
    for c in order:
        alive.append(_cuda_args(c))
        out = net.denoise(*alive[-1])
        assert torch.equal(out, fresh[c.name]), f"{c.name}: output differs after the workspace served other layouts"

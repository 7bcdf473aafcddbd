"""CPU: the host planner of bdiff_plan_topology (csrc/bdiff_plan.h), compiled with g++ into a test harness
(oracle/hostcheck/plan_hostcheck.cpp, test-only).

The layer megakernel claims its work list in order and waits on per-tile completion flags; it cannot deadlock only when
every tile a work item depends on comes earlier in the list.  That is a property of the host-side integer arrays, so it
is checked here for every catalogue layout and two full-size batches, at several layer counts and SM counts, together
with the rest of the staging block (against the numpy restatement `host_plan`) and the planner's rejections."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

from layout_catalogue import LAYOUTS, host_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "oracle", "hostcheck", "plan_hostcheck.cpp")
OUT = os.path.join(ROOT, "oracle", "_build", "libbdiff_plan_hostcheck.so")
HDR = os.path.join(ROOT, "bio-diffusion_b200", "csrc", "bdiff_plan.h")

INFO = ("B", "N", "E", "Mact", "TE", "TN", "nitems", "bytes", "mol_off", "act_off", "act_idx", "node_mol", "edge_off",
        "mask", "edge_dep", "node_dep", "node_mid", "items")


def build_hostcheck():
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    if not os.path.exists(OUT) or os.path.getmtime(OUT) < max(os.path.getmtime(SRC), os.path.getmtime(HDR)):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", OUT, SRC])
    return C.CDLL(OUT)


@pytest.fixture(scope="module")
def lib():
    return build_hostcheck()


def run_planner(lib, bi, mask, L, num_sms, num_mols=None, num_nodes=None):
    """(None, info dict, staging block) or (rejection message, None, None)."""
    bi = np.ascontiguousarray(bi, np.int64)
    mask = np.ascontiguousarray(mask, np.uint8)
    num_mols = int(bi.max()) + 1 if num_mols is None else num_mols
    num_nodes = bi.shape[0] if num_nodes is None else num_nodes
    info = np.zeros(len(INFO), np.int64)
    err = C.create_string_buffer(256)
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib.plan_hostcheck(C.c_int(num_mols), C.c_longlong(num_nodes), P(bi), P(mask), C.c_int(L), C.c_int(num_sms),
                            P(info), err, C.c_int(len(err)))
    if rc != 0:
        return err.value.decode(), None, None
    info = dict(zip(INFO, (int(v) for v in info)))
    block = np.zeros(info["bytes"], np.uint8)
    lib.plan_hostcheck_block(P(block))
    return None, info, block


def _array(block, info, name, dtype, count, cols=None):
    a = np.frombuffer(block, dtype, count * (cols or 1), info[name])
    return a.reshape(count, cols) if cols else a


def _cases():
    cases = [(c.name, c.sizes, c.mask().numpy()) for c in LAYOUTS]
    cases.append(("qm9_128x19", [19] * 128, np.ones(19 * 128, bool)))
    from bdiff.datasets import GEOM_N_NODES, sample_num_nodes
    sizes = [int(s) for s in sample_num_nodes(GEOM_N_NODES, 512, seed=123)]
    cases.append(("geom_hist_512", sizes, np.ones(sum(sizes), bool)))
    return cases


CASES = {name: (sizes, mask) for name, sizes, mask in _cases()}


def _check_order(items, L, te, tn, edge_dep, node_dep):
    """Every (type, layer, tile) once; every dependency before its consumer."""
    assert (items >= 0).all()
    typ, layer, tile = (items >> 30) & 1, (items >> 24) & 63, items & 0xffffff
    assert items.shape[0] == L * (te + tn)
    pos_e = np.full((L, te), -1, np.int64)
    pos_n = np.full((L, tn), -1, np.int64)
    idx = np.arange(items.shape[0])
    e, n = typ == 0, typ == 1
    assert (tile[e] < te).all() and (tile[n] < tn).all() and (layer < L).all()
    pos_e[layer[e], tile[e]] = idx[e]
    pos_n[layer[n], tile[n]] = idx[n]
    assert (pos_e >= 0).all() and (pos_n >= 0).all(), "an item is missing (or appears twice)"
    # node tile (l, u) after edge tiles (l, node_dep[u]); edge tile (l, t), l >= 1, after node tiles (l - 1, edge_dep[t])
    for u in range(tn):
        lo, hi = node_dep[u]
        if hi >= lo:
            assert (pos_e[:, lo:hi + 1].max(1) < pos_n[:, u]).all(), f"node tile {u} claimed before an edge tile it reads"
    for t in range(te):
        lo, hi = edge_dep[t]
        assert (pos_n[:-1, lo:hi + 1].max(1) < pos_e[1:, t]).all(), f"edge tile {t} claimed before a node tile it reads"


@pytest.mark.parametrize("name", list(CASES))
def test_plan_matches_restatement_and_orders_every_dependency_first(lib, name):
    sizes, mask = CASES[name]
    bi = np.repeat(np.arange(len(sizes)), sizes)
    ref = host_plan(torch.from_numpy(bi), torch.from_numpy(mask))
    for L in (1, 4, 9, 64):
        for num_sms in (1, 2, 132):
            err, info, block = run_planner(lib, bi, mask, L, num_sms)
            assert err is None, err
            for k in ("B", "N", "E", "Mact", "TE", "TN"):
                assert info[k] == ref[k], k
            B, N, te, tn = ref["B"], ref["N"], ref["TE"], ref["TN"]
            assert info["nitems"] == L * (te + tn)
            got = dict(mol_off=_array(block, info, "mol_off", np.int32, B + 1),
                       act_off=_array(block, info, "act_off", np.int32, B + 1),
                       act_idx=_array(block, info, "act_idx", np.int32, ref["Mact"]),
                       node_mol=_array(block, info, "node_mol", np.int32, N),
                       edge_off=_array(block, info, "edge_off", np.int64, B + 1),
                       mask=_array(block, info, "mask", np.uint8, N),
                       edge_dep=_array(block, info, "edge_dep", np.int32, te, 2),
                       node_dep=_array(block, info, "node_dep", np.int32, tn, 2),
                       node_mid=_array(block, info, "node_mid", np.int32, tn * 32, 2))
            for k, v in got.items():
                assert np.array_equal(v, ref[k]), f"{name}: {k} differs from the restatement"
            items = _array(block, info, "items", np.int32, info["nitems"]).astype(np.int64)
            _check_order(items, L, te, tn, ref["edge_dep"], ref["node_dep"])


def test_plan_rejections(lib):
    ones = np.ones(6, np.uint8)
    err, _, _ = run_planner(lib, [0, 0, 1, 0, 1, 1], ones, 9, 132)
    assert err == "batch_index must be sorted (node 3)"
    err, _, _ = run_planner(lib, [0, 0, 1, 1, 2, 2], ones, 9, 132, num_mols=2)
    assert err == "batch_index[4]=2 outside [0,2)"
    err, _, _ = run_planner(lib, [-1, 0, 0, 1, 1, 1], ones, 9, 132)
    assert err == "batch_index[0]=-1 outside [0,2)"
    n = 1 << 18                                   # one molecule of 2^18 atoms: 2^36 edges
    err, _, _ = run_planner(lib, np.zeros(n, np.int64), np.ones(n, np.uint8), 9, 132)
    assert err == "too many edges"
    err, _, _ = run_planner(lib, [0, 0, 1, 1, 1, 1], ones, 65, 132)
    assert err == "problem too large for the tile scheduler"
    err, _, _ = run_planner(lib, [0] * 6, ones, 9, 132, num_nodes=(1 << 30) + 1)
    assert err == "too many nodes"
    err, _, _ = run_planner(lib, [0] * 6, ones, 9, 132, num_mols=0)
    assert err == "bad plan arguments"
    assert run_planner(lib, [0, 0, 1, 1, 1, 1], ones, 64, 132)[0] is None

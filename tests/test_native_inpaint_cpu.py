"""CPU: the host half of the native inpainting chain (bdiff_inpaint) — the library's RePaint program against
bdiff/schedule.py's, the centring of the molecules on their fixed atoms against GCDMSampler's, and the argument checks
bdiff_inpaint runs before it touches the device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (T, r, j, F): single steps, jumps longer than the chain, resampling with and without frames, the shipped sizes
PROGRAMS = [(1, 1, 1, 1), (2, 1, 1, 2), (7, 3, 2, 1), (9, 2, 9, 1), (9, 2, 10, 1), (10, 1, 3, 1), (10, 2, 2, 1),
            (10, 3, 1, 5), (12, 4, 5, 1), (50, 10, 10, 1), (100, 10, 1, 10), (1000, 1, 1, 10), (1000, 10, 10, 1)]


def _draws(jump_after):
    """First draw of every op and jump and of the decode, in the order GCDMSampler's chain calls its noise hook: z_T
    (2 draws), per op the known and the unknown part (4), per jump 2, then the decode."""
    d, ops, jumps = 2, [], []
    for jump in jump_after:
        ops.append(d)
        d += 4
        if jump:
            jumps.append(d)
            d += 2
    return ops, jumps, d


@pytest.mark.parametrize("T,r,j,F", PROGRAMS)
def test_repaint_program_matches_schedule_py(T, r, j, F):
    from bdiff import DenoiserConfig
    from bdiff.noise import repaint_tables, schedule_tables
    from bdiff.schedule import gamma_table, repaint_program
    cfg = DenoiserConfig.named("qm9")
    lib = repaint_tables(cfg, T, r, j, F)
    py = repaint_program(gamma_table(cfg.num_timesteps, cfg.noise_precision, cfg.noise_schedule), r, j, T, F)
    assert lib["s_of_op"].tolist() == py["s_of_op"]
    assert lib["jump_after"].tolist() == py["jump_after"]
    assert lib["slot"].tolist() == py["slot"].tolist()
    assert lib["num_jumps"] == py["num_jumps"]
    ops, jumps, dec = _draws(py["jump_after"])
    assert lib["op_draw"].tolist() == ops and lib["jump_draw"].tolist() == jumps and lib["decode_draw"] == dec
    # reverse rows: bdiff_schedule_tables' rows at the op's s, bit for bit; the decode row likewise
    coef, decode = schedule_tables(cfg, T)
    assert torch.equal(lib["rev"], coef[T - 1 - lib["s_of_op"].long()])
    assert torch.equal(lib["decode"], decode)
    # known and jump rows: schedule.py's fp32 torch evaluation, within test_native_sample_cpu.py's bounds
    rel = lambda a, b: ((a.double() - b.double()).abs() / b.double().abs()).max(dim=0).values
    k = rel(lib["known"], py["known"])
    assert k[0] <= 1e-6 and k[1] <= 5e-5, k
    if py["num_jumps"]:
        pj = py["jump"][:py["num_jumps"]]
        assert torch.equal(lib["jump"][:, 2:], pj[:, 2:])
        q = rel(lib["jump"][:, :2], pj[:, :2])
        assert q[0] <= 1e-6 and q[1] <= 5e-5, q


def test_repaint_tables_refuse_bad_arguments():
    from bdiff import DenoiserConfig, _lib
    from bdiff.noise import repaint_tables
    cfg = DenoiserConfig.named("qm9")
    for args in ((10, 0, 1, 1), (10, 1, 0, 1), (10, 1, 2, 2), (10, 1, 1, 3), (10, 1, 1, 11)):
        with pytest.raises(_lib.BdiffError):
            repaint_tables(cfg, *args)


@pytest.fixture(scope="module")
def hostcheck(tmp_path_factory):
    out = tmp_path_factory.mktemp("hostcheck") / "libinpaint_hostcheck.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(out),
                    os.path.join(ROOT, "tests", "native", "inpaint_hostcheck.cpp")], check=True)
    lib = C.CDLL(str(out))
    lib.inpaint_hostcheck.restype = C.c_int
    lib.center_hostcheck.restype = None
    return lib


def test_centring_equals_the_samplers(hostcheck):
    from bdiff import GCDMSampler
    rng = np.random.default_rng(5)
    for trial in range(20):
        b = int(rng.integers(1, 12))
        counts = rng.integers(1, 30, size=b).astype(np.int32)
        n, ld = int(counts.sum()), int(rng.choice([8, 9, 19]))
        xh0 = (rng.standard_normal((n, ld)) * rng.choice([1.0, 3.0, 40.0])).astype(np.float32)
        fixed = (rng.random(n) < rng.choice([0.0, 0.2, 0.6, 1.0])).astype(np.uint8)
        fixed[:counts[0]] = 0                                  # the first molecule has no fixed atom
        bi = torch.repeat_interleave(torch.arange(b), torch.from_numpy(counts.astype(np.int64)))
        want = GCDMSampler._center_on_fixed(torch.from_numpy(xh0), bi, torch.from_numpy(fixed).bool(), b)
        got = xh0.copy()
        hostcheck.center_hostcheck(b, counts.ctypes.data_as(C.POINTER(C.c_int32)), ld,
                                   fixed.ctypes.data_as(C.POINTER(C.c_uint8)), got.ctypes.data_as(C.POINTER(C.c_float)))
        assert torch.equal(torch.from_numpy(got), want), trial
        assert np.array_equal(got[:counts[0]], xh0[:counts[0]])   # not moved


def _check(lib, counts, r=1, j=1, F=1, steps=10, fixed=None, num_h=6, num_context=0, charges=1, has_context=False):
    arr = (C.c_int32 * max(len(counts), 1))(*counts)
    n = sum(c for c in counts if c > 0)
    fx = np.zeros(max(n, 1), dtype=np.uint8) if fixed is None else np.asarray(fixed, dtype=np.uint8)
    msg = C.create_string_buffer(256)
    rc = lib.inpaint_hostcheck(num_h, num_context, 5, charges, len(counts), arr, int(has_context), steps, r, j, F,
                               fx.ctypes.data_as(C.POINTER(C.c_uint8)), msg, 256)
    return rc, msg.value.decode()


def test_inpaint_argument_checks(hostcheck):
    assert _check(hostcheck, [3, 5]) == (0, "")
    assert _check(hostcheck, [3, 5], r=3, j=2, steps=12) == (0, "")
    assert _check(hostcheck, [3, 5], F=5) == (0, "")
    for kw, what in ((dict(r=0), "num_resamplings, jump_length and num_timesteps must be >= 1"),
                     (dict(j=0), "must be >= 1"),
                     (dict(j=2, F=2), "only defined for jump_length == 1"),
                     (dict(F=3), "return_frames=3 does not divide num_timesteps=10"),
                     (dict(F=11), "return_frames must be in [1, num_timesteps=10]"),
                     (dict(fixed=[0, 1, 0, 2, 0, 0, 0, 0]), "fixed_host[3] = 2"),
                     (dict(steps=0), "num_timesteps")):
        rc, msg = _check(hostcheck, [3, 5], **kw)
        assert rc == -1 and what in msg, (kw, msg)
    rc, msg = _check(hostcheck, [3], num_h=5, num_context=1, charges=0)
    assert rc == -1 and "context" in msg
    assert _check(hostcheck, [3], num_h=5, num_context=1, charges=0, has_context=True) == (0, "")
    rc, msg = _check(hostcheck, [3, 0])
    assert rc == -1 and "at least one atom" in msg


def test_inpaint_refuses_a_fixed_mask_of_the_wrong_length():
    """node_mask_fixed is checked against the molecule's atoms on the host, before any chain (seeded or not) starts."""
    from bdiff import DenoiserConfig, GCDMSampler
    cfg = DenoiserConfig.named("qm9")
    mol = dict(x=torch.zeros(5, 3), one_hot=torch.zeros(5, 5), charges=torch.zeros(5, 1), num_nodes=torch.tensor([2, 3]),
               batch_index=torch.tensor([0, 0, 1, 1, 1]))
    with pytest.raises(ValueError, match=r"node_mask_fixed must be \[5\]"):
        GCDMSampler._inpaint_inputs(cfg, mol, torch.zeros(4, dtype=torch.bool), None)

"""CPU: the pieces of the native chain (bdiff_sample) that need no GPU — the numpy restatement of the counter-based noise
against CUDA's own Philox4x32-10, the library's host-side schedule tables (exact against an fp64 evaluation of
bdiff/schedule.py's formulas, close to schedule.py's fp32 torch evaluation), and the argument checks bdiff_sample runs
before it touches the device."""
import ctypes as C
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import philox_mirror as PM
from config_catalogue import CONFIGS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cuda_include():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(nvcc))), "include")
    if not os.path.exists(os.path.join(inc, "curand_philox4x32_x.h")):
        pytest.fail(f"CUDA headers not found under {inc}")
    return inc


CURAND_KAT = r"""
#include <cstdio>
#include <vector_types.h>
#define QUALIFIERS static inline
#include <curand_philox4x32_x.h>
int main() {
  unsigned c0, c1, c2, c3, k0, k1;
  while (scanf("%x %x %x %x %x %x", &c0, &c1, &c2, &c3, &k0, &k1) == 6) {
    uint4 c = {c0, c1, c2, c3}; uint2 k = {k0, k1};
    uint4 o = curand_Philox4x32_10(c, k);
    printf("%08x %08x %08x %08x\n", o.x, o.y, o.z, o.w);
  }
}
"""


def test_philox_mirror_matches_curand(tmp_path):
    """Known answers from the host path of CUDA's curand_Philox4x32_10 (the Random123 authors' code shipped with the
    toolkit), at the all-zero, all-ones and pi-digit vectors and at random (counter, key) pairs."""
    src = tmp_path / "kat.cpp"
    src.write_text(CURAND_KAT)
    exe = tmp_path / "kat"
    subprocess.run(["g++", "-std=c++17", "-I", _cuda_include(), str(src), "-o", str(exe)], check=True)
    rng = np.random.default_rng(3)
    vecs = np.concatenate([np.array([[0] * 6, [0xFFFFFFFF] * 6,
                                     [0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344, 0xA4093822, 0x299F31D0]],
                                    dtype=np.uint32),
                           rng.integers(0, 2 ** 32, size=(200, 6), dtype=np.uint64).astype(np.uint32)])
    inp = "\n".join(" ".join(f"{v:x}" for v in row) for row in vecs)
    out = subprocess.run([str(exe)], input=inp, capture_output=True, text=True, check=True).stdout.split()
    want = np.array([int(w, 16) for w in out], dtype=np.uint32).reshape(-1, 4)
    got = PM.philox4x32_10(vecs[:, :4], vecs[:, 4:])
    assert np.array_equal(got, want)
    # the first one is Random123's published known answer for philox4x32-10 at counter 0, key 0
    assert got[0].tolist() == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]


def test_mirror_layout():
    """Counter = {block, draw}, key = seed: different draws and seeds give different words, element e uses block e>>2."""
    a, b = PM.blocks(7, 0, 4), PM.blocks(7, 1, 4)
    assert not np.array_equal(a, b) and not np.array_equal(a, PM.blocks(8, 0, 4))
    n = PM.normals(7, 0, 16)
    assert np.array_equal(n[:8], PM.normals(7, 0, 8)) and np.isfinite(n).all()


def _tables(cfg, steps):
    from bdiff.noise import schedule_tables
    return schedule_tables(cfg, steps)


def _fp64_tables(gamma, steps):
    """The formulas of schedule.py's transition_terms / _reverse_rows / decode_coefficients evaluated in float64 (the C
    library's exp / log1p / expm1, as the library calls them) at schedule.py's fp32 gamma and grid, rounded once."""
    f32 = np.float32
    g = gamma.numpy()
    T = len(g) - 1
    softplus = lambda x: x if x > 20.0 else math.log1p(math.exp(x))
    logsigmoid = lambda x: min(0.0, x) - math.log1p(math.exp(-abs(x)))
    sigmoid = lambda x: 1.0 / (1.0 + math.exp(-x))
    rows = []
    for r in range(steps):
        s_int = f32(steps - 1 - r)
        s, t = f32(s_int / f32(steps)), f32((s_int + f32(1)) / f32(steps))
        gs, gt = float(g[int(np.rint(f32(s * f32(T))))]), float(g[int(np.rint(f32(t * f32(T))))])
        sigma2 = -math.expm1(softplus(gs) - softplus(gt))
        alpha = math.exp(0.5 * (logsigmoid(-gt) - logsigmoid(-gs)))
        sigma_s, sigma_t = math.sqrt(sigmoid(gs)), math.sqrt(sigmoid(gt))
        rows.append((alpha, sigma2 / alpha / sigma_t, math.sqrt(sigma2) * sigma_s / sigma_t, t))
    return torch.tensor(np.array(rows, dtype=np.float64).astype(np.float32))


def _catalogue():
    from bdiff import DenoiserConfig
    return [DenoiserConfig.named(n) for n in ("qm9", "qm9_cond", "geom")] + [c.denoiser() for c in CONFIGS]


@pytest.mark.parametrize("steps", [1000, 500, 7, 2, 1])
def test_schedule_tables_are_exact(steps):
    """bdiff_schedule_tables, for every configuration: gamma bit-equal to schedule.py's (the rows read it at the grid
    points), every coefficient bit-equal to the fp64 evaluation of schedule.py's formulas at that gamma, and the decode
    row bit-equal to schedule.decode_coefficients."""
    from bdiff.schedule import decode_coefficients, gamma_table
    for cfg in _catalogue():
        gamma = gamma_table(cfg.num_timesteps, cfg.noise_precision, cfg.noise_schedule)
        coef, dec = _tables(cfg, steps)
        assert torch.equal(coef, _fp64_tables(gamma, steps))
        assert torch.equal(dec, decode_coefficients(gamma))


@pytest.mark.parametrize("steps", [1000, 500, 7, 2, 1])
def test_schedule_tables_agree_with_schedule_py(steps):
    """schedule.py evaluates the same formulas in fp32 with torch's CPU kernels (MKL's exp, SLEEF's log1p / expm1 at the
    SIMD width torch dispatches to), which round differently; the cancellation in sigma2_ts = -expm1(softplus(g_s) -
    softplus(g_t)) magnifies that.  t is equal, alpha_ts within 1e-6 and c_eps / sigma within 5e-5 relative."""
    from bdiff.schedule import gamma_table, step_coefficient_table
    for cfg in _catalogue():
        ref = step_coefficient_table(gamma_table(cfg.num_timesteps, cfg.noise_precision, cfg.noise_schedule), steps)
        coef, _ = _tables(cfg, steps)
        assert torch.equal(coef[:, 3], ref[:, 3])
        rel = ((coef.double() - ref.double()).abs() / ref.double().abs()).max(dim=0).values
        assert rel[0] <= 1e-6 and rel[1] <= 5e-5 and rel[2] <= 5e-5, rel


_PY_TABLE = """
import sys
sys.path.insert(0, sys.argv[1])
import torch
from bdiff.schedule import gamma_table, step_coefficient_table
torch.save(step_coefficient_table(gamma_table(1000), 1000), sys.argv[2])
"""


def test_schedule_py_tables_depend_on_torch_cpu_dispatch(tmp_path):
    """Why the library does not promise bit-equality with schedule.py: schedule.py's own table changes when torch runs
    its portable CPU kernels instead of the SIMD ones this machine gets, by as much as the library's table differs from
    it.  A fixed restatement can equal at most one of them; the library's is the fp64 one, the same on every host."""
    if torch.backends.cpu.get_cpu_capability() == "DEFAULT":
        pytest.skip("torch already runs its portable kernels here")
    script = tmp_path / "table.py"
    script.write_text(_PY_TABLE)
    pkg = os.path.join(ROOT, "bio-diffusion_b200")
    tables = {}
    for cap in ("default", None):
        env = dict(os.environ)
        env.pop("ATEN_CPU_CAPABILITY", None)
        if cap:
            env["ATEN_CPU_CAPABILITY"] = cap
        out = tmp_path / f"{cap}.pt"
        subprocess.run([sys.executable, str(script), pkg, str(out)], check=True, env=env)
        tables[cap] = torch.load(out)
    portable, simd = tables["default"], tables[None]
    assert not torch.equal(portable, simd)
    from bdiff import DenoiserConfig
    lib, _ = _tables(DenoiserConfig.named("qm9"), 1000)
    rel = lambda a, b: ((a.double() - b.double()).abs() / b.double().abs()).max().item()
    spread = rel(portable, simd)
    assert rel(lib, simd) <= spread and rel(lib, portable) <= spread


def test_schedule_tables_reject_bad_config():
    from bdiff import _lib
    from bdiff.config import DenoiserConfig
    from bdiff.noise import sample_config
    lib = _lib.load()
    sc = sample_config(DenoiserConfig.named("qm9"))
    buf = (C.c_float * 8)()
    assert lib.bdiff_schedule_tables(C.byref(sc), 0, buf, buf) == -1
    sc.noise_precision = 0.0
    assert lib.bdiff_schedule_tables(C.byref(sc), 2, buf, buf) == -1


@pytest.fixture(scope="module")
def hostcheck(tmp_path_factory):
    out = tmp_path_factory.mktemp("hostcheck") / "libsample_hostcheck.so"
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", str(out),
                    os.path.join(ROOT, "tests", "native", "sample_hostcheck.cpp")], check=True)
    lib = C.CDLL(str(out))
    lib.sample_hostcheck.restype = C.c_int
    return lib


def _check(lib, counts, num_h=6, num_context=0, a=5, charges=1, has_context=False, steps=10, z_shape=None):
    arr = (C.c_int32 * max(len(counts), 1))(*counts)
    shape = (C.c_int64 * 2)(*z_shape) if z_shape is not None else None
    msg = C.create_string_buffer(256)
    rc = lib.sample_hostcheck(num_h, num_context, a, charges, len(counts), arr, int(has_context), steps,
                              int(z_shape is not None), shape, msg, 256)
    return rc, msg.value.decode()


def test_sample_argument_checks(hostcheck):
    assert _check(hostcheck, [3, 5]) == (0, "")
    rc, msg = _check(hostcheck, [])
    assert rc == -1 and "num_mols" in msg
    rc, msg = _check(hostcheck, [3, 0, 2])
    assert rc == -1 and "num_nodes_host[1] = 0" in msg
    rc, msg = _check(hostcheck, [3, -4])
    assert rc == -1 and "at least one atom" in msg
    rc, msg = _check(hostcheck, [3], num_h=5, num_context=1, charges=0)
    assert rc == -1 and "context" in msg
    assert _check(hostcheck, [3], num_h=5, num_context=1, charges=0, has_context=True) == (0, "")
    rc, msg = _check(hostcheck, [3, 5], z_shape=(8, 8))
    assert rc == -1 and "z_init must be [8, 9]" in msg
    assert _check(hostcheck, [3, 5], z_shape=(8, 9)) == (0, "")
    rc, msg = _check(hostcheck, [3], steps=0)
    assert rc == -1 and "num_timesteps" in msg
    rc, msg = _check(hostcheck, [3], num_h=7)
    assert rc == -1 and "num_h" in msg

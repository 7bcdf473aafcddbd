"""Compiler guard of the layer megakernel (bdiff_layers_tc.cu): its wgmmas must issue back to back.

ptxas serializes every wgmma of a kernel (each one waits for its own completion: one WARPGROUP.DEPBAR per HGMMA, warning
C7520) as soon as one of them sits on a path it cannot prove warp-uniform, e.g. inside a lambda it chose to compile as a
called subroutine.  That costs the tensor pipe most of its throughput without changing any result, so only the compiler's
output shows it.  This test compiles the kernel for sm_90a and checks, for both instantiations:
  - no C7520;
  - at most one WARPGROUP.DEPBAR per three HGMMAs (every ring chunk issues at least three products and waits once);
  - stack frame and spills no larger than the bounds below, per instantiation (the figures of CUDA 12.9).
Runs without a GPU; skipped where nvcc is absent."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "bio-diffusion_b200", "csrc")
KERNEL = "k_layers_tc"
INSTANTIATIONS = ("k_layers_tcILi64ELi16E", "k_layers_tcILi16ELi8E")
# bytes per thread: (stack frame, spill stores, spill loads); the serialized build spilled 628 / 1272 and 640 / 1284
MAX_FRAME_SPILLS = {"k_layers_tcILi64ELi16E": (320, 248, 532), "k_layers_tcILi16ELi8E": (272, 200, 472)}


def _nvcc():
    found = shutil.which("nvcc")
    if found:
        return found
    cand = "/usr/local/cuda/bin/nvcc"
    return cand if os.path.exists(cand) else None


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    out = tmp_path_factory.mktemp("layers_sass")
    obj = str(out / "bdiff_layers_tc.o")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                        "-c", os.path.join(CSRC, "bdiff_layers_tc.cu"), "-o", obj],
                       capture_output=True, text=True, cwd=CSRC)
    assert r.returncode == 0, r.stderr[-4000:]
    sass = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    return r.stdout + r.stderr, sass


def _per_function(sass):
    counts, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            counts[cur] = {"HGMMA": 0, "DEPBAR": 0}
            continue
        if cur is None:
            continue
        if "HGMMA." in line:
            counts[cur]["HGMMA"] += 1
        if "WARPGROUP.DEPBAR" in line:
            counts[cur]["DEPBAR"] += 1
    return counts


def test_no_serialized_wgmma(compiled):
    log, _ = compiled
    bad = [ln for ln in log.splitlines() if "C7520" in ln]
    assert not bad, "ptxas serializes the wgmmas of the layer megakernel:\n" + "\n".join(bad)


def test_one_wait_per_chunk(compiled):
    _, sass = compiled
    counts = _per_function(sass)
    for inst in INSTANTIATIONS:
        fn = [c for name, c in counts.items() if inst in name and KERNEL in name]
        assert len(fn) == 1, f"{inst} not found in the SASS"
        c = fn[0]
        assert c["HGMMA"] > 0
        assert 3 * c["DEPBAR"] <= c["HGMMA"], f"{inst}: {c['DEPBAR']} WARPGROUP.DEPBAR for {c['HGMMA']} HGMMA"


def test_spills_bounded(compiled):
    log, _ = compiled
    lines = log.splitlines()
    seen = 0
    for i, ln in enumerate(lines):
        inst = next((x for x in INSTANTIATIONS if x in ln), None)
        if "Compiling entry function" not in ln or inst is None:
            continue
        props = next(x for x in lines[i + 1:] if "spill stores" in x)
        got = tuple(int(v) for v in re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                                               props).groups())
        bound = MAX_FRAME_SPILLS[inst]
        assert all(g <= b for g, b in zip(got, bound)), f"{ln.strip()}: {props.strip()} (bounds {bound})"
        seen += 1
    assert seen == len(INSTANTIATIONS)

"""CPU: the product's training pass (csrc/bdiff_train_engine.cuh — the functors the CUDA kernels of bdiff_train.cu run
and the GEMM orchestration between them) compiled against a host backend (oracle/hostcheck/train_hostcheck.cpp,
test-only) and compared with torch.autograd through the forward oracle: net_out and the gradient of every parameter
tensor, masked atoms, one-atom molecules and the three shipped configurations included.  The CUDA backend itself
(launch wrapper, cuBLAS adapter) is checked on the device by tests/test_gpu_train.py against the reference's fixtures."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import gcpnet_oracle as O
from layout_catalogue import host_plan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "oracle", "hostcheck", "train_hostcheck.cpp")
OUT = os.path.join(ROOT, "oracle", "_build", "libbdiff_train_hostcheck.so")
HDR = os.path.join(ROOT, "bio-diffusion_b200", "csrc", "bdiff_train_engine.cuh")


def build_hostcheck():
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    if not os.path.exists(OUT) or os.path.getmtime(OUT) < max(os.path.getmtime(SRC), os.path.getmtime(HDR)):
        subprocess.check_call(["g++", "-O2", "-fopenmp", "-std=c++17", "-shared", "-fPIC", "-o", OUT, SRC])
    return C.CDLL(OUT)


def run_hostcheck(lib, cfg, sd, bi, mask, xh, t, ctx, d_out):
    pl = host_plan(bi, mask)
    names = list(sd.keys())
    offs, tot = [], 0
    for k in names:
        offs.append(tot)
        tot += (sd[k].numel() + 63) // 64 * 64
    params = np.zeros(tot, np.float32)
    for k, o in zip(names, offs):
        params[o:o + sd[k].numel()] = sd[k].reshape(-1).numpy()
    grads = np.full(tot, 7.0, np.float32)          # the engine must zero its gradient buffer itself
    dims = np.array([cfg.num_h, cfg.num_context, cfg.h_in, cfg.e_hidden, cfg.xi_hidden, cfg.num_layers], np.int32)
    n = bi.shape[0]
    out = np.zeros((n, 3 + cfg.num_h), np.float32)
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    f32 = lambda v: np.ascontiguousarray(v.numpy().astype(np.float32))
    xh_, t_, d_ = f32(xh), f32(t.reshape(-1)), f32(d_out)
    ctx_ = f32(ctx) if ctx is not None else np.zeros(1, np.float32)
    offs_ = np.array(offs, np.int64)
    lib.hostcheck_train.restype = C.c_int
    rc = lib.hostcheck_train(P(dims), C.c_int(pl["B"]), C.c_int(pl["N"]), C.c_longlong(pl["E"]), C.c_int(pl["Mact"]),
                             P(pl["mol_off"]), P(pl["act_off"]), P(pl["act_idx"]), P(pl["edge_off"]), P(pl["node_mol"]),
                             P(pl["mask"]), P(pl["edge_rc"]), C.c_char_p("\n".join(names).encode()), P(offs_),
                             C.c_int(len(names)), P(params), P(grads), C.c_longlong(tot), P(xh_), P(t_), P(ctx_), P(d_),
                             P(out))
    assert rc == 0, f"hostcheck_train: rc {rc} (<0: parameter names not found; >1e6: GEMM calls with illegal leading dimensions)"
    g = {k: torch.from_numpy(grads[o:o + sd[k].numel()].copy()).reshape(sd[k].shape) for k, o in zip(names, offs)}
    return torch.from_numpy(out), g


@pytest.mark.parametrize("cname,sizes,masked", [("qm9", [5, 1, 7], [2]), ("qm9_cond", [4, 6], [5]), ("geom", [9, 3, 1], [0, 10]),
                                                ("geom", [4, 4], []), ("geom", [131, 2], [7]),
                                                ("qm9", [3, 4, 5], [3, 4, 5, 6])])      # molecule 1 has no active atom
def test_training_pass_matches_autograd(cname, sizes, masked):
    lib = build_hostcheck()
    cfg = O.config_named(cname)
    sd = O.random_state_dict(cfg, 21, scale=0.7)
    g = torch.Generator().manual_seed(5)
    nmol = len(sizes)
    bi = torch.repeat_interleave(torch.arange(nmol), torch.tensor(sizes))
    n = bi.shape[0]
    mask = torch.ones(n, dtype=torch.bool)
    for i in masked:
        mask[i] = False
    xh = torch.randn((n, 3 + cfg.num_h), generator=g)
    t = torch.full((n, 1), 0.37)
    ctx = torch.randn((n, cfg.num_context), generator=g) if cfg.num_context else None
    d_out = torch.randn((n, 3 + cfg.num_h), generator=g)
    sda = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    out_a = O.denoiser_forward(sda, cfg, bi, mask, xh, t, ctx, guard_empty=True)    # DESIGN.md §2
    (out_a * d_out).sum().backward()
    out_h, grads = run_hostcheck(lib, cfg, sd, bi, mask, xh, t, ctx, d_out)
    err_f = (out_h - out_a.detach()).abs().max().item() / out_a.detach().abs().max().item()
    assert err_f < 2e-5, err_f
    worst, worst_key = 0.0, None
    for k in sd:
        ref = sda[k].grad
        err = (grads[k] - ref).abs().max().item() / max(ref.abs().max().item(), 1e-12)
        if err > worst:
            worst, worst_key = err, k
    assert worst < 2e-4, (worst_key, worst)

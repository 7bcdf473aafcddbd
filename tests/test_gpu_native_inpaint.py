"""GPU: the native inpainting chain (bdiff_inpaint, GCDMSampler.inpaint(seed=...)) and the frames of the native sampling
chain (bdiff_sample_frames, sample / optimize(seed=..., return_frames=F)).

The key property, as for bdiff_sample: a seeded chain is torch.equal to the Python chain fed the same draws through the
noise hook, `noise=philox_noise(s)`.  Also: the frames, reproducibility, the graph cache, interleaving with bdiff_sample
on one handle, and a C program with no torch in its process."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import gcpnet_oracle as O
from test_gpu_native_sample import _dump_weights, _net

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _molecule(cfg, sizes, seed=2, free=(1,)):
    """Random molecules of `sizes` atoms with ~40 % fixed atoms; the molecules listed in `free` have none."""
    g = torch.Generator().manual_seed(seed)
    n = sum(sizes)
    bi = torch.repeat_interleave(torch.arange(len(sizes)), torch.tensor(sizes))
    types = torch.randint(0, cfg.num_atom_types, (n,), generator=g)
    mol = dict(x=(torch.randn((n, 3), generator=g) * 1.5).cuda(), one_hot=torch.eye(cfg.num_atom_types)[types].cuda(),
               num_nodes=torch.tensor(sizes), batch_index=bi.cuda())
    if cfg.include_charges:
        mol["charges"] = torch.randint(1, 10, (n, 1), generator=g).float().cuda()
    fixed = torch.rand(n, generator=g) < 0.4
    for k in free:
        fixed[bi == k] = False
    return mol, fixed.cuda()


def _context(net, b):
    return torch.randn((b, 1), generator=torch.Generator().manual_seed(1)).cuda() if net.cfg.num_context else None


CASES = [("qm9", "tensor", [9, 7, 1, 12]), ("qm9", "parity", [5, 11, 3]), ("qm9_cond", "tensor", [9, 17, 1, 12]),
         ("geom", "tensor", [30, 45, 12])]


@pytest.mark.parametrize("r,j", [(1, 1), (2, 2), (3, 1), (1, 3)])
@pytest.mark.parametrize("name,mode,sizes", CASES)
def test_native_inpaint_equals_python_chain_fed_the_same_draws(name, mode, sizes, r, j):
    import bdiff
    net = _net(name, mode)
    s = bdiff.GCDMSampler(net)
    mol, fixed = _molecule(net.cfg, sizes)
    ctx = _context(net, len(sizes))
    for seed in (5, 2 ** 40 + 3):
        out = s.inpaint(mol, fixed, r, j, num_timesteps=5, context=ctx, seed=seed)
        ref = s.inpaint(mol, fixed, r, j, num_timesteps=5, context=ctx, noise=bdiff.philox_noise(seed))
        assert torch.isfinite(out).all()
        assert torch.equal(out, ref)


def test_frames_equal_python_chain():
    """sample / optimize / inpaint with seed= and return_frames = F: every frame bit-equal to the noise-hook chain; frame 0
    is the molecules without the CoG fix."""
    import bdiff
    net = _net("qm9")
    s = bdiff.GCDMSampler(net)
    sizes = torch.tensor([19, 7, 12])
    out = s.sample(sizes, num_timesteps=6, return_frames=3, seed=8)[0]
    ref = s.sample(sizes, num_timesteps=6, return_frames=3, noise=bdiff.philox_noise(8))[0]
    assert out.shape == (3, 38, 9) and torch.equal(out, ref)
    assert not torch.equal(out[1], out[2])
    mol, fixed = _molecule(net.cfg, [9, 7, 12], free=(2,))
    out = s.inpaint(mol, fixed, 2, 1, return_frames=2, num_timesteps=4, seed=3)
    ref = s.inpaint(mol, fixed, 2, 1, return_frames=2, num_timesteps=4, noise=bdiff.philox_noise(3))
    assert out.shape == (2, 28, 9) and torch.equal(out, ref)
    # optimize from existing molecules (a configuration without charges)
    gnet = _net("geom")
    gs = bdiff.GCDMSampler(gnet)
    g = torch.Generator().manual_seed(3)
    sz = [30, 21]
    bi = torch.repeat_interleave(torch.arange(2), torch.tensor(sz))
    n = bi.shape[0]
    _, x = O.centralize(torch.randn((n, 3), generator=g) * 1.5, bi, torch.ones(n, dtype=torch.bool), 2)
    one_hot = torch.nn.functional.one_hot(torch.randint(0, gnet.cfg.num_atom_types, (n,), generator=g),
                                          gnet.cfg.num_atom_types).float()
    samples = [(x[:30], one_hot[:30]), (x[30:], one_hot[30:])]
    out = gs.optimize(samples, torch.tensor(sz), num_timesteps=4, return_frames=2, seed=12)[0]
    ref = gs.optimize(samples, torch.tensor(sz), num_timesteps=4, return_frames=2, noise=bdiff.philox_noise(12))[0]
    assert out.shape[0] == 2 and torch.equal(out, ref)


def test_seed_refusals():
    import bdiff
    net = _net("qm9")
    s = bdiff.GCDMSampler(net)
    mol, fixed = _molecule(net.cfg, [5, 6])
    with pytest.raises(ValueError, match="noise"):
        s.inpaint(mol, fixed, num_timesteps=3, seed=1, noise=bdiff.philox_noise(1))
    for kw in (dict(noise=bdiff.philox_noise(1)), dict(node_mask=torch.ones(11, dtype=torch.bool)), dict(return_z0=True),
               dict(record_moments=True)):
        with pytest.raises(ValueError, match="native chain"):
            s.sample(torch.tensor([5, 6]), num_timesteps=3, seed=1, **kw)


def test_reproducible_graph_cache_and_interleaving():
    import bdiff
    from bdiff import _lib
    lib = _lib.load()
    net = _net("qm9")
    s = bdiff.GCDMSampler(net)
    mol, fixed = _molecule(net.cfg, [9, 7, 1, 12])
    builds = lambda: lib.bdiff_inpaint_graph_builds(net._handle)
    a = s.inpaint(mol, fixed, 2, 2, num_timesteps=6, seed=1)
    assert builds() == 1
    b = s.inpaint(mol, fixed, 2, 2, num_timesteps=6, seed=1)
    c = s.inpaint(mol, fixed, 2, 2, num_timesteps=6, seed=2)
    assert torch.equal(a, b) and not torch.equal(a[:, :3], c[:, :3])
    s.inpaint(mol, fixed, 2, 2, num_timesteps=4, seed=3)             # a shorter chain and another seed: the same graphs
    assert builds() == 1
    big, bfixed = _molecule(net.cfg, [19, 25, 29, 12, 8])
    s.inpaint(big, bfixed, 2, 2, num_timesteps=4, seed=3)             # a larger batch: rebuilt
    assert builds() == 2
    # alternating with bdiff_sample on the same handle gives what fresh handles give
    sizes = torch.tensor([9, 17, 1, 12])
    alt = []
    for _ in range(2):
        alt.append(s.sample(sizes, num_timesteps=5, seed=4)[0])
        alt.append(s.inpaint(mol, fixed, 2, 2, num_timesteps=6, seed=1))
    fresh_sample = bdiff.GCDMSampler(_net("qm9")).sample(sizes, num_timesteps=5, seed=4)[0]
    fresh_inpaint = bdiff.GCDMSampler(_net("qm9")).inpaint(mol, fixed, 2, 2, num_timesteps=6, seed=1)
    for k in range(0, 4, 2):
        assert torch.equal(alt[k], fresh_sample) and torch.equal(alt[k + 1], fresh_inpaint)
    assert torch.equal(alt[1], a)
    n = builds()
    with torch.no_grad():                                              # new weights: rebuilt
        next(net.parameters()).mul_(0.5)
    s.inpaint(mol, fixed, 2, 2, num_timesteps=6, seed=1)
    assert builds() == n + 1


def test_bad_arguments_are_rejected():
    from bdiff import _lib
    from bdiff.noise import sample_config
    net = _net("qm9_cond")
    net.sync_weights()
    lib = _lib.load()
    h = net._handle
    assert lib.bdiff_sample_setup(h, C.byref(sample_config(net.cfg))) == 0
    out = torch.empty((4, 64, 3 + net.cfg.num_h), device="cuda")
    ctx = torch.zeros((4, 1), device="cuda")
    xh0 = np.zeros((64, 3 + net.cfg.num_h), dtype=np.float32)
    fixed = np.zeros(64, dtype=np.uint8)

    def call(counts=(3, 5), context=ctx, T=4, r=1, j=1, F=1):
        arr = (C.c_int32 * max(len(counts), 1))(*counts)
        rc = lib.bdiff_inpaint(h, None, len(counts), arr, C.c_void_p(context.data_ptr()) if context is not None else None,
                               T, r, j, 1, C.c_void_p(xh0.ctypes.data), C.c_void_p(fixed.ctypes.data), F, None,
                               C.c_void_p(out.data_ptr()), None)
        return rc, lib.bdiff_last_error(h).decode()

    for kw, what in ((dict(r=0), "must be >= 1"), (dict(j=2, F=2), "jump_length == 1"), (dict(F=3), "does not divide"),
                     (dict(context=None), "context"), (dict(counts=(3, 0)), "at least one atom")):
        rc, msg = call(**kw)
        assert rc == -1 and what in msg, msg
    assert call(F=2)[0] == 0


def test_c_program_without_torch_inpaints_like_python(tmp_path):
    import bdiff
    from bdiff.schedule import decode_coefficients, repaint_program
    cuda = os.path.dirname(os.path.dirname(os.path.realpath(shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc")))
    libdir = os.path.join(ROOT, "bio-diffusion_b200", "bdiff")
    exe = tmp_path / "inpaint_main"
    subprocess.run(["gcc", "-std=c11", "-O2", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(cuda, "include"),
                    os.path.join(ROOT, "tests", "native", "inpaint_main.c"), "-o", str(exe), "-L", libdir, "-lbdiff_sm90",
                    "-L", os.path.join(cuda, "lib64"), "-lcudart", f"-Wl,-rpath,{libdir}",
                    f"-Wl,-rpath,{os.path.join(cuda, 'lib64')}"], check=True)
    net = _net("qm9")
    s = bdiff.GCDMSampler(net)
    sizes, steps, r, j, seed = [9, 7, 1, 12], 6, 2, 2, 4242
    mol, fixed = _molecule(net.cfg, sizes)
    _dump_weights(net, tmp_path / "w.bin")
    prog = repaint_program(s.gamma, r, j, steps)
    tables = torch.cat((prog["rev"].reshape(-1), prog["known"].reshape(-1), prog["jump"][:prog["num_jumps"]].reshape(-1),
                        decode_coefficients(s.gamma)))
    (tmp_path / "t.bin").write_bytes(tables.float().numpy().tobytes())
    xh0 = torch.cat((mol["x"], mol["one_hot"], mol["charges"]), dim=1).float().cpu()
    (tmp_path / "m.bin").write_bytes(xh0.numpy().tobytes() + fixed.cpu().to(torch.uint8).numpy().tobytes())
    env = {k: v for k, v in os.environ.items() if k not in ("LD_PRELOAD", "PYTHONPATH")}
    subprocess.run([str(exe), str(tmp_path / "w.bin"), str(tmp_path / "t.bin"), str(tmp_path / "m.bin"),
                    str(tmp_path / "o.bin"), str(seed), str(steps), str(r), str(j)] + [str(v) for v in sizes],
                   check=True, env=env)
    got = torch.from_numpy(np.fromfile(tmp_path / "o.bin", dtype=np.float32).reshape(sum(sizes), -1).copy())
    ref = s.inpaint(mol, fixed, r, j, num_timesteps=steps, seed=seed).cpu()
    assert torch.equal(got, ref)

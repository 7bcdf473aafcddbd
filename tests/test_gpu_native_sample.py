"""GPU: the native chain (bdiff_sample, GCDMSampler.sample(seed=...)) and its counter-based noise.

The key property: sample(seed=s) is torch.equal to the Python chain fed the same draws through the existing noise hook,
sample(noise=philox_noise(s)) — the native chain runs the same arithmetic in the same order.  Also: the noise against the
numpy restatement, its statistics, reproducibility, the launch count per step, the graph cache, the argument checks, and
a C program with no torch in its process."""
import ctypes as C
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest
import torch

import gcpnet_oracle as O
import philox_mirror as PM

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _net(name, mode="tensor", seed=7):
    import bdiff
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named(name), mode=mode)
    net.load_state_dict(O.random_state_dict(O.config_named(name), seed, scale=0.5), strict=True)
    return net.cuda()


def _ulps(a, b):
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


def test_noise_fill_matches_mirror():
    from bdiff.noise import noise_fill, philox_words
    for seed, draw in ((0, 0), (12345, 7), (2 ** 63 + 11, 2 ** 33 + 5)):
        words = philox_words(seed, draw, 4096).cpu().numpy().astype(np.uint32)
        assert np.array_equal(words, PM.blocks(seed, draw, 4096))
        got = noise_fill(seed, draw, (4099, 3)).cpu().numpy().reshape(-1)
        want = PM.normals(seed, draw, got.size)
        assert _ulps(got, want).max() <= 2


def test_noise_statistics():
    from scipy import stats
    from bdiff.noise import noise_fill
    n = 10_000_000
    x = noise_fill(99, 3, (n,)).double()
    m, v = x.mean().item(), x.var().item()
    assert abs(m) < 5 / n ** 0.5 and abs(v - 1) < 5 * (2 / n) ** 0.5
    assert abs((x ** 3).mean().item()) < 5 * (15 / n) ** 0.5 and abs((x ** 4).mean().item() - 3) < 5 * (96 / n) ** 0.5
    assert stats.kstest(x[:2_000_000].cpu().numpy(), "norm").pvalue > 1e-3
    y = noise_fill(99, 4, (n,)).double()               # the next draw
    lim = 5 / n ** 0.5
    for a, b in ((x, y), (x[:-1], x[1:]), (x[:-2], x[2:]), (x[:-4], x[4:])):
        assert abs(torch.corrcoef(torch.stack((a, b)))[0, 1].item()) < lim
    z = noise_fill(100, 3, (n,)).double()              # another seed, same draw
    assert abs(torch.corrcoef(torch.stack((x, z)))[0, 1].item()) < lim


CASES = [("qm9", "tensor", [9, 17, 1, 12, 19]), ("qm9", "parity", [5, 11, 3]), ("qm9_cond", "tensor", [9, 17, 1, 12]),
         ("geom", "tensor", [30, 45, 12])]


@pytest.mark.parametrize("name,mode,sizes", CASES)
def test_native_chain_equals_python_chain_fed_the_same_draws(name, mode, sizes):
    import bdiff
    net = _net(name, mode)
    s = bdiff.GCDMSampler(net)
    num_nodes = torch.tensor(sizes)
    ctx = torch.randn((len(sizes), 1), generator=torch.Generator().manual_seed(1)).cuda() if net.cfg.num_context else None
    for seed in (5, 2 ** 40 + 3):
        out, bi, mask = s.sample(num_nodes, ctx, 6, seed=seed)
        ref, rbi, rmask = s.sample(num_nodes, ctx, 6, noise=bdiff.philox_noise(seed))
        assert torch.isfinite(out).all()
        assert torch.equal(out, ref) and torch.equal(bi, rbi) and torch.equal(mask, rmask)
    # the centred noise and the re-centred steps leave every molecule's centre of gravity at the origin
    x = out[:, :3].double()
    cog = torch.zeros((len(sizes), 3), dtype=torch.float64, device=x.device).index_add_(0, bi, x)
    assert cog.abs().max().item() < 1e-4 * max(1.0, x.abs().max().item()) * max(sizes)


@pytest.mark.parametrize("name", ["qm9_cond", "geom"])
def test_native_chain_from_z_init(name):
    import bdiff
    net = _net(name)
    s = bdiff.GCDMSampler(net)
    sizes = torch.tensor([7, 13, 4])
    g = torch.Generator().manual_seed(3)
    z = torch.randn((int(sizes.sum()), 3 + net.cfg.num_h), generator=g)
    bi = torch.repeat_interleave(torch.arange(3), sizes)
    z[:, :3] -= (torch.zeros((3, 3)).index_add_(0, bi, z[:, :3]) / sizes[:, None])[bi]
    z = z.cuda()
    ctx = torch.randn((3, 1), generator=g).cuda() if net.cfg.num_context else None
    out = s.sample(sizes, ctx, 5, z_init=z, seed=17)[0]
    ref = s.sample(sizes, ctx, 5, z_init=z, noise=bdiff.philox_noise(17))[0]
    assert torch.equal(out, ref)


def test_reproducible_and_seed_dependent():
    import bdiff
    s = bdiff.GCDMSampler(_net("qm9"))
    sizes = torch.tensor([9, 17, 1, 12])
    a = s.sample(sizes, num_timesteps=8, seed=1)[0]
    b = s.sample(sizes, num_timesteps=8, seed=1)[0]
    c = s.sample(sizes, num_timesteps=8, seed=2)[0]
    assert torch.equal(a, b)
    assert not torch.equal(a[:, :3], c[:, :3])
    # the output is discretised like mol_gen_sample's: one-hot types and integer charges
    assert torch.equal(a[:, 3:8].sum(1), torch.ones(a.shape[0], device=a.device))
    assert torch.equal(a[:, 8], a[:, 8].round())


def test_launches_per_step_and_graph_cache():
    import bdiff
    from bdiff import _lib
    net = _net("qm9")
    s = bdiff.GCDMSampler(net)
    lib = _lib.load()
    sizes, larger = torch.tensor([9, 17, 1, 12]), torch.tensor([19, 25, 29, 12, 8])

    def launches(steps, sz=sizes, seed=1):
        before = net.launch_count()
        s.sample(sz, num_timesteps=steps, seed=seed)
        return net.launch_count() - before

    builds = lambda: lib.bdiff_sample_graph_builds(net._handle)
    launches(6)                                         # first call: also packs the weights
    assert builds() == 1
    d6 = launches(6)
    d3 = launches(3)                                    # a shorter chain and another seed: the same graph
    launches(3, seed=9)
    assert builds() == 1
    assert d6 - d3 == 3 * (net.kernels_per_forward + 1)
    launches(3, larger)                                 # a larger topology: rebuilt
    assert builds() == 2
    launches(3, larger, seed=4)
    assert builds() == 2
    with torch.no_grad():                               # new weights: rebuilt
        next(net.parameters()).mul_(0.5)
    launches(3, larger)
    assert builds() == 3
    launches(3, larger)
    assert builds() == 3


def test_batch_index_after_a_longer_chain():
    """A longer chain than any before grows (and so reallocates) the chain buffers while the plan of the same batch is
    reused: the returned batch_index must still be the batch's, and the molecules those of a fresh handle."""
    import bdiff
    s = bdiff.GCDMSampler(_net("qm9"))
    sizes = torch.tensor([9, 17, 1, 12])
    want = torch.repeat_interleave(torch.arange(4), sizes).cuda()
    for steps in (3, 8, 30):
        out, bi, _ = s.sample(sizes, num_timesteps=steps, seed=11)
        assert torch.equal(bi, want)
    fresh = bdiff.GCDMSampler(_net("qm9")).sample(sizes, num_timesteps=30, seed=11)[0]
    assert torch.equal(out, fresh)


def test_bad_arguments_are_rejected():
    from bdiff import _lib
    from bdiff.noise import sample_config
    net = _net("qm9_cond")
    net.sync_weights()
    lib = _lib.load()
    h = net._handle
    sc = sample_config(net.cfg)
    assert lib.bdiff_sample_setup(h, C.byref(sc)) == 0
    out = torch.empty((64, 3 + net.cfg.num_h), device="cuda")
    ctx = torch.zeros((4, 1), device="cuda")

    def call(counts, context, z_init=None, shape=None):
        arr = (C.c_int32 * max(len(counts), 1))(*counts)
        zs = (C.c_int64 * 2)(*shape) if shape else None
        rc = lib.bdiff_sample(h, None, len(counts), arr, C.c_void_p(context.data_ptr()) if context is not None else None,
                              4, 1, C.c_void_p(z_init.data_ptr()) if z_init is not None else None, zs, None,
                              C.c_void_p(out.data_ptr()), None)
        return rc, lib.bdiff_last_error(h).decode()

    for counts, context, z, shape, what in (([], ctx, None, None, "num_mols"), ([3, 0], ctx, None, None, "at least one"),
                                            ([3, -2], ctx, None, None, "at least one"), ([3, 5], None, None, None, "context"),
                                            ([3, 5], ctx, out, (8, 5), f"z_init must be [8, {3 + net.cfg.num_h}]")):
        rc, msg = call(counts, context, z, shape)
        assert rc == -1 and what in msg, msg
    assert call([3, 5], ctx)[0] == 0


def _dump_weights(net, path):
    cfg = net.cfg
    with open(path, "wb") as f:
        f.write(struct.pack("8i", cfg.num_h, cfg.num_context, cfg.num_layers, cfg.h_hidden, cfg.chi_hidden, cfg.e_hidden,
                            cfg.xi_hidden, 1 if net.mode == "tensor" else 0))
        f.write(struct.pack("3i", cfg.num_atom_types, int(cfg.include_charges), cfg.num_timesteps))
        f.write(struct.pack("2d", float(cfg.noise_schedule.split("_")[1]), cfg.noise_precision))
        f.write(struct.pack("3f", *cfg.norm_values))
        f.write(struct.pack("3f", *[0.0 if v is None else v for v in cfg.norm_biases]))
        params = list(net.state_dict().items())
        f.write(struct.pack("i", len(params)))
        for name, t in params:
            f.write(struct.pack("i", len(name)) + name.encode())
            f.write(struct.pack("i", t.dim()) + struct.pack(f"{t.dim()}q", *t.shape))
            f.write(t.detach().float().contiguous().cpu().numpy().tobytes())


def test_c_program_without_torch_samples_like_python(tmp_path):
    import bdiff
    from bdiff.schedule import decode_coefficients, step_coefficient_table
    cuda = os.path.dirname(os.path.dirname(os.path.realpath(shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc")))
    libdir = os.path.join(ROOT, "bio-diffusion_b200", "bdiff")
    exe = tmp_path / "sample_main"
    subprocess.run(["gcc", "-std=c11", "-O2", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(cuda, "include"),
                    os.path.join(ROOT, "tests", "native", "sample_main.c"), "-o", str(exe), "-L", libdir, "-lbdiff_sm90",
                    "-L", os.path.join(cuda, "lib64"), "-lcudart", f"-Wl,-rpath,{libdir}",
                    f"-Wl,-rpath,{os.path.join(cuda, 'lib64')}"], check=True)
    net = _net("qm9")
    s = bdiff.GCDMSampler(net)
    sizes, steps, seed = [9, 17, 1, 12], 5, 4242
    _dump_weights(net, tmp_path / "w.bin")
    tables = torch.cat((step_coefficient_table(s.gamma, steps).reshape(-1), decode_coefficients(s.gamma)))
    (tmp_path / "t.bin").write_bytes(tables.float().numpy().tobytes())
    env = {k: v for k, v in os.environ.items() if k not in ("LD_PRELOAD", "PYTHONPATH")}
    lib_coef, lib_dec = bdiff.noise.schedule_tables(net.cfg, steps)
    (tmp_path / "l.bin").write_bytes(torch.cat((lib_coef.reshape(-1), lib_dec)).numpy().tobytes())
    outs = {}
    for tab in ("t.bin", "-", "l.bin"):
        subprocess.run([str(exe), str(tmp_path / "w.bin"), str(tmp_path / tab) if tab != "-" else "-",
                        str(tmp_path / "o.bin"), str(seed), str(steps)] + [str(v) for v in sizes], check=True, env=env)
        got = torch.from_numpy(np.fromfile(tmp_path / "o.bin", dtype=np.float32).reshape(sum(sizes), -1).copy())
        if tab == "t.bin":     # the Python chain's tables: bit-identical to sample(seed=)
            ref = s.sample(torch.tensor(sizes), num_timesteps=steps, seed=seed)[0].cpu()
            assert torch.equal(got, ref)
        else:                  # the library's own tables: a valid sample (one-hot types, integer charges) ...
            assert torch.isfinite(got).all()
            assert torch.equal(got[:, 3:8].sum(1), torch.ones(sum(sizes)))
        outs[tab] = got
    # ... and exactly the run on bdiff_schedule_tables' output handed in explicitly
    assert torch.equal(outs["-"], outs["l.bin"])

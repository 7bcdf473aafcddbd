"""CPU: the configurations of config_catalogue.py, and the boundaries of what bdiff_create accepts.

The catalogue must reach every class of config_catalogue.CLASSES; parameter shapes and the module's state dict must match
the oracle's for every entry; and the training engine's host build (test_train_hostcheck.py) must match float64 autograd
through the oracle on every entry but the 64-layer one (too slow on the host; the GPU tests run it) — net_out within 2e-5
of max|ref|, each gradient within 2e-4 of its max|ref|.
"""
import ctypes as C

import pytest
import torch

import gcpnet_oracle as O
from config_catalogue import BY_NAME, CLASSES, CONFIGS, config_classes, derived_dims
from layout_catalogue import BY_NAME as LAYOUTS, _inputs
from test_gpu_train_layouts import oracle_grads
from test_train_hostcheck import build_hostcheck, run_hostcheck


def test_catalogue_reaches_every_class():
    union = set()
    for c in CONFIGS:
        got = config_classes(c)
        print(f"{c.name:16s} {derived_dims(c)}: {', '.join(sorted(got))}")
        union |= got
    assert CLASSES <= union, f"no entry reaches {CLASSES - union}"
    for c in CONFIGS:       # every entry is there for a class no other entry reaches
        rest = set().union(*(config_classes(o) for o in CONFIGS if o is not c))
        assert not CLASSES <= rest, f"{c.name} reaches no class of its own"
    assert len({c.name for c in CONFIGS}) == len(CONFIGS)
    for c in CONFIGS:
        assert derived_dims(c)["hin"] == c.oracle().h_in == c.denoiser().h_in
        assert all(n in LAYOUTS for n in c.layouts)


def test_derived_dims_of_the_shipped_configs():
    """The restated dims on the shipped configurations, whose values DESIGN.md and the kernels' comments quote."""
    from config_catalogue import ConfigCase
    qm9 = derived_dims(ConfigCase("qm9", 5, True, 0, 9, 64, 16, 0, 1.0, ()))
    geom = derived_dims(ConfigCase("geom", 16, False, 0, 4, 16, 8, 0, 1.0, ()))
    assert qm9 == dict(hin=7, hid0=20, K0=96, Ke=28, Kn=48, edge_embed="tpe", tensor=True)
    assert geom == dict(hin=17, hid0=18, K0=44, Ke=20, Kn=60, edge_embed="tpe", tensor=True)


@pytest.mark.parametrize("name", [c.name for c in CONFIGS])
def test_parameter_shapes_and_state_dict(name):
    import bdiff
    from bdiff.config import parameter_shapes
    c = BY_NAME[name]
    sd = O.random_state_dict(c.oracle(), c.seed, scale=c.scale)
    assert parameter_shapes(c.denoiser()) == {k: tuple(v.shape) for k, v in sd.items()} == O.param_shapes(c.oracle())
    net = bdiff.GCPNetDynamicsB200(config=c.denoiser())
    net.load_state_dict(sd, strict=True)


@pytest.mark.parametrize("name", [c.name for c in CONFIGS if c.num_layers < 64])
def test_host_training_engine_matches_fp64_autograd(name):
    c = BY_NAME[name]
    ocfg = c.oracle()
    lay = LAYOUTS[c.layouts[0]]
    inputs = _inputs(lay, ocfg)
    d_out = torch.randn((lay.n, 3 + ocfg.num_h), generator=torch.Generator().manual_seed(c.seed))
    sd = O.random_state_dict(ocfg, c.seed, scale=c.scale)
    ref_out, ref_grads = oracle_grads(sd, ocfg, inputs, d_out)
    out, grads = run_hostcheck(build_hostcheck(), ocfg, sd, *inputs, d_out)
    err = (out.double() - ref_out).abs().max().item() / ref_out.abs().max().item()
    worst = max(((grads[k].double() - r).abs().max().item() / max(r.abs().max().item(), 1e-30), k)
                for k, r in ref_grads.items())
    print(f"{name}: net_out {err:.2e}, worst gradient {worst[0]:.2e} ({worst[1]})")
    assert err < 2e-5, err
    assert worst[0] < 2e-4, worst


def test_from_reference_cfgs_two_conditioning_keys():
    """The reference's QM9 module config documents `conditioning: [H_thermo, homo]`: one context column per key."""
    import bdiff
    model = dict(chi_input_dim=2, e_input_dim=1, xi_input_dim=1, h_hidden_dim=256, chi_hidden_dim=32, e_hidden_dim=64,
                 xi_hidden_dim=16, num_encoder_layers=9, dropout=0.0)
    module = dict(conditioning=["H_thermo", "homo"])
    diff = dict(norm_values=[1.0, 8.0, 1.0])
    data = dict(num_atom_types=5, include_charges=False, num_x_dims=3)
    cfg = bdiff.DenoiserConfig.from_reference_cfgs(model, module, {}, diff, data)
    assert cfg.num_context == 2 and cfg.h_in == 8
    assert (cfg.e_hidden, cfg.xi_hidden, cfg.num_h) == (BY_NAME["qm9_c2"].e_hidden, BY_NAME["qm9_c2"].xi_hidden, 5)


def _create(**kw):
    """bdiff_create's return code for the qm9 dims with `kw` changed; a handle it makes is destroyed."""
    from bdiff import _lib
    lib = _lib.load()
    args = dict(num_h=6, num_context=0, num_layers=9, h_hidden=256, chi_hidden=32, e_hidden=64, xi_hidden=16, mode=0)
    args.update(kw)
    h = C.c_void_p()
    rc = lib.bdiff_create(C.byref(_lib.Config(**args)), C.byref(h))
    if h.value:
        lib.bdiff_destroy(h)
    return rc, lib.bdiff_last_error(None).decode()


@pytest.mark.parametrize("kw", [dict(e_hidden=0), dict(e_hidden=2), dict(e_hidden=6), dict(e_hidden=68),
                                dict(xi_hidden=2), dict(xi_hidden=6), dict(xi_hidden=20),
                                dict(num_h=28, num_context=0), dict(num_h=6, num_context=22),
                                dict(num_layers=0), dict(num_layers=65)])
def test_create_refuses_out_of_range_configs(kw):
    rc, msg = _create(**kw)
    assert rc == -1, (kw, rc, msg)


@pytest.mark.parametrize("kw", [dict(e_hidden=4), dict(e_hidden=64), dict(xi_hidden=4), dict(xi_hidden=16),
                                dict(num_h=1, num_context=0), dict(num_h=6, num_context=21), dict(num_layers=1),
                                dict(num_layers=64), dict(mode=1, num_h=17, num_context=10, e_hidden=16, xi_hidden=8)])
def test_create_accepts_the_edges_of_the_range(kw):
    rc, msg = _create(**kw)
    assert rc == (0 if torch.cuda.is_available() else -2), (kw, rc, msg)


@pytest.mark.parametrize("name", [c.name for c in CONFIGS if not c.tensor])
def test_tensor_mode_refuses_other_edge_dims(name):
    """Before it touches a device: the same refusal with and without a GPU."""
    import bdiff
    net = bdiff.GCPNetDynamicsB200(config=BY_NAME[name].denoiser(), mode="tensor")
    with pytest.raises(bdiff.BdiffError, match=r"\(64,16\), \(16,8\)"):
        net._ensure_handle()
    rc, _ = _create(mode=1, e_hidden=BY_NAME[name].e_hidden, xi_hidden=BY_NAME[name].xi_hidden)
    assert rc == -1

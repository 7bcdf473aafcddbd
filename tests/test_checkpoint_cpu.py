"""CPU: the reference-checkpoint converters of bdiff/checkpoint.py on synthesised Lightning checkpoints.

The layout fixture (tests/golden/checkpoint_layout.pt) is the reference's own state_dict / parameters() order; the
checkpoint contents come from torch.optim.AdamW and the EMA callback's arithmetic (tests/checkpoint_synth.py)."""
import copy
import warnings

import pytest
import torch

import bdiff
from bdiff.checkpoint import DYNAMICS_PREFIX, reference_parameter_names, reference_to_training_state, \
    training_state_to_reference
from checkpoint_synth import assert_same, layout, synth_checkpoint

CONFIGS = ("qm9", "qm9_cond", "geom")
HYPER = dict(lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-12, amsgrad=True, ema_decay=0.9999, clip=True,
             queue_len=50)


def names_of(cname):
    return list(bdiff.parameter_shapes(bdiff.DenoiserConfig.named(cname)))


@pytest.mark.parametrize("cname", CONFIGS)
def test_fixture_orders_agree_with_parameter_shapes(cname):
    lay = layout(cname)
    shapes = bdiff.parameter_shapes(bdiff.DenoiserConfig.named(cname))
    dyn = {k[len(DYNAMICS_PREFIX):]: s for k, s, _ in lay["state_dict"] if k.startswith(DYNAMICS_PREFIX)}
    assert dyn == {k: tuple(s) for k, s in shapes.items()}
    params = [k[len(DYNAMICS_PREFIX):] for k in lay["parameters"] if k.startswith(DYNAMICS_PREFIX)]
    assert set(params) == set(shapes) and len(params) == len(shapes)
    assert lay["parameters"][-1] == "ddpm.gamma.gamma"
    assert reference_parameter_names([k for k, _, _ in lay["state_dict"]]) == lay["parameters"]
    assert set(lay["buffers"]) == {k for k, _, _ in lay["state_dict"]} - set(lay["parameters"])


@pytest.mark.parametrize("cname", CONFIGS)
def test_import_matches_torch_adamw_and_export_reproduces_the_template(cname):
    ckpt, params = synth_checkpoint(cname, steps=3, seed=1)
    lay = layout(cname)
    order = names_of(cname)[::-1]              # any order of the tail's parameters: mapping is by name
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        st = reference_to_training_state(ckpt, bdiff.DenoiserConfig.named(cname), order, HYPER)
    adam = ckpt["optimizer_states"][0]["state"]
    ema = dict(zip([k for k, _, _ in lay["state_dict"]], ckpt["callbacks"]["EMA"]["ema_weights"]))
    pos = {k: i for i, k in enumerate(lay["parameters"])}
    o = st["optimizer"]
    for i, n in enumerate(order):
        k = DYNAMICS_PREFIX + n
        assert torch.equal(st["model"][n], params[pos[k]].detach())
        assert torch.equal(o["exp_avg"][i], adam[pos[k]]["exp_avg"])
        assert torch.equal(o["exp_avg_sq"][i], adam[pos[k]]["exp_avg_sq"])
        assert torch.equal(o["max_exp_avg_sq"][i], adam[pos[k]]["max_exp_avg_sq"])
        assert torch.equal(o["ema"][i], ema[k])
    assert int(o["state"][0]) == 3 and int(o["state"][1]) == 1 and int(o["state"][2]) == 1
    assert o["state"][8:9].view(torch.float32).item() == 3000.0
    assert o["hyperparameters"]["lr"] == 1e-4 and o["hyperparameters"]["weight_decay"] == 1e-12

    out, ema_ckpt = training_state_to_reference(st, ckpt, bdiff.DenoiserConfig.named(cname))
    assert_same(out, ckpt)
    assert list(ema_ckpt["state_dict"].keys()) == list(ckpt["state_dict"].keys())
    assert_same(list(ema_ckpt["state_dict"].values()), ckpt["callbacks"]["EMA"]["ema_weights"])
    assert_same({k: v for k, v in ema_ckpt.items() if k != "state_dict"}, {k: v for k, v in out.items() if k != "state_dict"})
    fresh = [torch.nn.Parameter(p.detach().clone(), requires_grad=p.requires_grad) for p in params]
    torch.optim.AdamW(fresh, lr=1e-4, weight_decay=1e-12, amsgrad=True).load_state_dict(out["optimizer_states"][0])


def test_export_writes_new_values_and_keeps_the_rest():
    cname = "geom"
    cfg = bdiff.DenoiserConfig.named(cname)
    ckpt, _ = synth_checkpoint(cname, steps=2, seed=2)
    st = reference_to_training_state(ckpt, cfg, names_of(cname), HYPER)
    o = st["optimizer"]
    for t in list(st["model"].values()) + o["exp_avg"] + o["ema"]:
        t.add_(1.0)
    o["state"][0] = 7
    o["hyperparameters"]["lr"] = 3e-4
    out, ema_ckpt = training_state_to_reference(st, ckpt, cfg, epoch=5, global_step=7)
    assert out["epoch"] == 5 and out["global_step"] == 7
    assert out["optimizer_states"][0]["param_groups"][0]["lr"] == 3e-4
    lay = layout(cname)
    for i, n in enumerate(names_of(cname)):
        k = DYNAMICS_PREFIX + n
        p = lay["parameters"].index(k)
        s = out["optimizer_states"][0]["state"][p]
        assert torch.equal(out["state_dict"][k], st["model"][n]) and torch.equal(s["exp_avg"], o["exp_avg"][i])
        assert s["step"].dtype == ckpt["optimizer_states"][0]["state"][p]["step"].dtype and float(s["step"]) == 7.0
        assert torch.equal(ema_ckpt["state_dict"][k], o["ema"][i])
    for k in lay["buffers"] + ["ddpm.gamma.gamma"]:
        assert out["state_dict"][k] is ckpt["state_dict"][k]
    ref_ema = dict(zip(ckpt["state_dict"].keys(), ckpt["callbacks"]["EMA"]["ema_weights"]))
    assert torch.equal(ema_ckpt["state_dict"]["ddpm.num_nodes_distribution.prob"], ref_ema["ddpm.num_nodes_distribution.prob"])
    for key in ("loops", "lr_schedulers", "hyper_parameters"):
        assert out[key] is ckpt[key]
    assert_same(out["callbacks"]["EMAModelCheckpoint{'monitor': 'val/loss', 'mode': 'min'}"],
                ckpt["callbacks"]["EMAModelCheckpoint{'monitor': 'val/loss', 'mode': 'min'}"])
    assert out["callbacks"]["EMA"]["cur_step"] == ckpt["callbacks"]["EMA"]["cur_step"]


def test_ema_precedence_companion_then_callback_then_warning():
    cname = "geom"
    cfg = bdiff.DenoiserConfig.named(cname)
    names = names_of(cname)
    ckpt, _ = synth_checkpoint(cname, steps=2, seed=3)
    companion = {"state_dict": {k: v + 1.0 if v.is_floating_point() else v for k, v in ckpt["state_dict"].items()}}
    st = reference_to_training_state(ckpt, cfg, names, HYPER, ema_ckpt=companion)
    assert all(torch.equal(e, companion["state_dict"][DYNAMICS_PREFIX + n]) for e, n in zip(st["optimizer"]["ema"], names))
    cb = dict(zip(ckpt["state_dict"].keys(), ckpt["callbacks"]["EMA"]["ema_weights"]))
    st = reference_to_training_state(ckpt, cfg, names, HYPER)
    assert all(torch.equal(e, cb[DYNAMICS_PREFIX + n]) for e, n in zip(st["optimizer"]["ema"], names))
    bare = dict(ckpt, callbacks={"EMA": {"cur_step": 1}})
    with pytest.warns(UserWarning, match="unable to find the associated EMA weights"):
        st = reference_to_training_state(bare, cfg, names, HYPER)
    assert all(torch.equal(e, ckpt["state_dict"][DYNAMICS_PREFIX + n]) for e, n in zip(st["optimizer"]["ema"], names))


def _broken(ckpt, what):
    c = copy.deepcopy(ckpt)
    sd = c["state_dict"]
    if what == "learned":
        sd["ddpm.gamma.gamma_0"] = torch.tensor([-5.0])
    elif what == "gamma":
        sd["ddpm.gamma.gamma"] = sd["ddpm.gamma.gamma"] * 1.001
    elif what == "no_optimizer":
        del c["optimizer_states"]
    elif what == "param_count":
        c["optimizer_states"][0]["param_groups"][0]["params"].append(10 ** 6)
    elif what == "shape":
        k = next(k for k in sd if k.startswith(DYNAMICS_PREFIX))
        sd[k] = torch.zeros(sd[k].shape[0] + 1, *sd[k].shape[1:])
    elif what == "missing":
        del sd[next(k for k in sd if k.startswith(DYNAMICS_PREFIX))]
    elif what == "mixed_steps":
        st = c["optimizer_states"][0]["state"]
        st[0]["step"] = st[0]["step"] + 1
    elif what == "partial_state":
        del c["optimizer_states"][0]["state"][0]
    elif what == "ema_list":
        c["callbacks"]["EMA"]["ema_weights"] = c["callbacks"]["EMA"]["ema_weights"][:-1]
    return c


TEMPLATE_ERRORS = ("learned", "gamma", "no_optimizer", "param_count", "shape", "missing")


@pytest.mark.parametrize("what", TEMPLATE_ERRORS + ("mixed_steps", "partial_state", "ema_list"))
def test_errors_raise_and_load_nothing(what):
    cname = "geom"
    cfg = bdiff.DenoiserConfig.named(cname)
    ckpt, _ = synth_checkpoint(cname, steps=2, seed=4)
    bad = _broken(ckpt, what)
    with pytest.raises(ValueError):
        reference_to_training_state(bad, cfg, names_of(cname), HYPER)
    if what in ("learned", "gamma", "shape", "missing"):        # the weight-only import checks these too
        net = bdiff.GCPNetDynamicsB200(config=cfg)
        before = {k: v.clone() for k, v in net.state_dict().items()}
        with pytest.raises(ValueError):
            bdiff.from_reference_checkpoint(bad, net)
        assert all(torch.equal(before[k], v) for k, v in net.state_dict().items())
    if what in TEMPLATE_ERRORS:
        good = reference_to_training_state(ckpt, cfg, names_of(cname), HYPER)
        with pytest.raises(ValueError):
            training_state_to_reference(good, bad, cfg)


def test_weight_only_import_on_a_cpu_net():
    cname = "qm9_cond"
    ckpt, _ = synth_checkpoint(cname, steps=1, seed=5)
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named(cname))
    bdiff.from_reference_checkpoint(ckpt, net)
    for n, p in net.named_parameters():
        assert torch.equal(p.detach(), ckpt["state_dict"][DYNAMICS_PREFIX + n])


def test_a_different_schedule_length_is_rejected():
    ckpt, _ = synth_checkpoint("geom", steps=1, seed=6)
    cfg = bdiff.DenoiserConfig(num_atom_types=16, include_charges=False, num_layers=4, e_hidden=16, xi_hidden=8,
                               num_timesteps=500)
    with pytest.raises(ValueError, match="ddpm.gamma.gamma"):
        reference_to_training_state(ckpt, cfg, names_of("geom"), HYPER)

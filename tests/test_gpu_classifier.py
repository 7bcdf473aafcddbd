"""GPU: bdiff.PropertyClassifier (the EGNN property classifier on the CUDA path) against the reference fixture and the
float64 oracle.  Tolerance 1e-4 * max(1, |ref|): the edge GEMM runs on split-bf16 wgmma (~2^-16 relative per product),
the node GEMMs in fp32 FFMA, the activations with ex2 / rcp approximations."""
import pytest
import torch

import classifier_oracle as CO
import gcpnet_oracle as O
from conftest import load_golden

pytestmark = pytest.mark.gpu


def _clf(n_layers, attention, node_attr, sd):
    import bdiff
    clf = bdiff.PropertyClassifier(n_layers=n_layers, attention=attention, node_attr=int(node_attr))
    clf.load_state_dict(sd, strict=True)
    return clf.cuda().requires_grad_(False)


def _close(got, ref):
    tol = 1e-4 * max(1.0, ref.abs().max().item())
    err = (got.double().cpu() - ref.double().cpu()).abs().max().item()
    assert err <= tol, f"max |diff| {err:.3e} > {tol:.1e}"


def _sd64(sd):
    return {k: v.double() for k, v in sd.items()}


@pytest.mark.parametrize("name", ["l7_att", "l2_nodeattr"])
def test_fixture_predictions_and_mae(name):
    fx = load_golden("classifier_qm9")
    c = fx["configs"][name]
    clf = _clf(c["n_layers"], c["attention"], c["node_attr"], CO.random_state_dict(c["seed"], c["n_layers"], c["attention"],
                                                                                   c["node_attr"]))
    loss, count = 0.0, 0
    for b, ref in zip(fx["batches"], c["pred"]):
        packed = clf.predict(b["x"].cuda(), b["one_hot"].cuda(), b["num_nodes"])
        _close(packed, ref)
        d = CO.dense_batch(b["x"].cuda(), b["one_hot"].cuda(), b["num_nodes"])
        bs, n, _ = d["positions"].shape
        # exactly the call of test_with_property_classifier (src/__init__.py:170-183)
        dense = clf(h0=d["one_hot"].view(bs * n, -1), x=d["positions"].view(bs * n, -1), edges=None, edge_attr=None,
                    node_mask=d["atom_mask"].view(bs * n, -1).float(), edge_mask=d["edge_mask"].float(), n_nodes=n)
        assert torch.equal(dense, packed)
        loss += (fx["mad"] * dense.cpu() + fx["mean"] - b["label"]).abs().mean().item() * bs
        count += bs
    assert abs(loss / count - c["mae"]) <= 1e-4 * max(1.0, c["mae"])


@pytest.mark.parametrize("n_layers,attention,node_attr", [(7, True, False), (2, False, True)])
def test_qm9_batch_against_float64_oracle_and_rerun(n_layers, attention, node_attr):
    import bdiff
    sd = CO.random_state_dict(21, n_layers, attention, node_attr)
    clf = _clf(n_layers, attention, node_attr, sd)
    sizes = bdiff.sample_num_nodes(bdiff.QM9_N_NODES, 128, seed=4)
    sizes[0], sizes[1] = 1, 29
    g = torch.Generator().manual_seed(8)
    n = int(sizes.sum())
    x = torch.randn((n, 3), generator=g) * 1.5
    oh = torch.nn.functional.one_hot(torch.randint(0, 5, (n,), generator=g), 5).double()
    ref = CO.packed_forward(_sd64(sd), n_layers, attention, node_attr, x.double(), oh, sizes)
    p1 = clf.predict(x.cuda(), oh.float().cuda(), sizes)
    p2 = clf.predict(x.cuda(), oh.float().cuda(), sizes)
    _close(p1, ref)
    assert torch.equal(p1, p2), "two runs differ"


def test_rows_cut_by_tile_borders():
    """Molecules of 127 / 128 atoms and odd sizes: rows of pairs cut by tile borders and by the tile's middle row."""
    sd = CO.random_state_dict(4, 2, True, False)
    clf = _clf(2, True, False, sd)
    sizes = torch.tensor([128, 3, 127, 1, 65, 64, 2])
    g = torch.Generator().manual_seed(2)
    n = int(sizes.sum())
    x = torch.randn((n, 3), generator=g) * 2.0
    oh = torch.nn.functional.one_hot(torch.randint(0, 5, (n,), generator=g), 5).double()
    ref = CO.packed_forward(_sd64(sd), 2, True, False, x.double(), oh, sizes)
    p = clf.predict(x.cuda(), oh.float().cuda(), sizes)
    _close(p, ref)
    assert torch.equal(p, clf.predict(x.cuda(), oh.float().cuda(), sizes))


def test_weights_repacked_after_update():
    sd = CO.random_state_dict(6, 1, True, False)
    clf = _clf(1, True, False, sd)
    x, oh, sizes = torch.randn(9, 3).cuda(), torch.eye(5)[torch.arange(9) % 5].cuda(), torch.tensor([4, 5])
    p0 = clf.predict(x, oh, sizes).clone()
    with torch.no_grad():
        clf.graph_dec._modules["2"].bias.add_(1.0)
    p1 = clf.predict(x, oh, sizes)
    _close(p1, p0 + 1.0)


def test_sample_and_optimize_scored_by_predict():
    """End to end: a T = 4 qm9_cond sample, then one optimisation iteration (optimize with 4 steps), both scored by
    predict on the sampler's packed output and compared with the oracle on the same molecules."""
    import bdiff
    ocfg = O.config_named("qm9_cond")
    net = bdiff.GCPNetDynamicsB200(config=bdiff.DenoiserConfig.named("qm9_cond"), mode="tensor")
    net.load_state_dict(O.random_state_dict(ocfg, 7, scale=0.5), strict=True)
    net.cuda()
    sampler = bdiff.GCDMSampler(net)
    sd = CO.random_state_dict(9)
    clf = _clf(7, True, False, sd)
    sizes = torch.tensor([9, 1, 17, 29, 12])
    ctx = torch.randn((len(sizes), 1), generator=torch.Generator().manual_seed(3)).cuda()
    torch.manual_seed(0)
    out, bi, _ = sampler.sample(sizes, ctx, num_timesteps=4)
    for it in range(2):
        x, oh = out[:, :3], out[:, 3:8]
        pred = clf.predict(x, oh, sizes)
        ref = CO.packed_forward(_sd64(sd), 7, True, False, x.double().cpu(), oh.double().cpu(), sizes)
        _close(pred, ref)
        if it == 0:
            samples, o = [], 0
            for k in sizes.tolist():
                samples.append((out[o:o + k, :3], out[o:o + k, 3:8]))
                o += k
            out, _, _ = sampler.optimize(samples, sizes, ctx, num_timesteps=4)

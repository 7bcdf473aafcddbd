"""GPU: the training pass of bdiff.PropertyClassifier (forward with tape + hand-written reverse sweep behind autograd)
against the reference training fixture and the float64 oracle, its reproducibility, the reference's training loop
restated through the dense drop-in, and the one-tape rule."""
import pytest
import torch

import classifier_backward as CB
import classifier_oracle as CO
from conftest import load_golden

pytestmark = pytest.mark.gpu

# ||g - g_ref||_inf / ||g_ref||_2 per parameter tensor: the bar of the denoiser's training pass.  The edge GEMMs (z2 and
# da) run on split-bf16 wgmma (~2^-16 relative per product), the rest in fp32 FFMA, activations with ex2 / rcp.
GRAD_TOL = 2e-4


def _clf(n_layers, attention, node_attr, sd):
    import bdiff
    clf = bdiff.PropertyClassifier(n_layers=n_layers, attention=attention, node_attr=int(node_attr))
    clf.load_state_dict(sd, strict=True)
    return clf.cuda()


def _dense(d):
    bs, n, _ = d["positions"].shape
    return dict(h0=d["one_hot"].view(bs * n, -1), x=d["positions"].view(bs * n, -1), edges=None, edge_attr=None,
                node_mask=d["atom_mask"].view(bs * n, -1).float(), edge_mask=d["edge_mask"].float(), n_nodes=n)


def _molecules(sizes, seed):
    sizes = torch.as_tensor(sizes)
    g = torch.Generator().manual_seed(seed)
    n = int(sizes.sum())
    x = torch.randn((n, 3), generator=g) * 1.5
    oh = torch.nn.functional.one_hot(torch.randint(0, 5, (n,), generator=g), 5).float()
    return sizes, x, oh


@pytest.mark.parametrize("name", ["l7_att", "l2_nodeattr"])
def test_gradients_match_reference_fixture(name):
    """loss.backward() of the train branch of train_with_property_classifier (:188-190) on batch 0, every parameter."""
    fx = load_golden("classifier_train_qm9")
    c = fx["configs"][name]
    clf = _clf(c["n_layers"], c["attention"], c["node_attr"],
               CO.random_state_dict(c["seed"], c["n_layers"], c["attention"], c["node_attr"]))
    b = fx["batches"][0]
    d = CO.dense_batch(b["x"].cuda(), b["one_hot"].cuda(), b["num_nodes"])
    pred = clf(**_dense(d))
    assert pred.requires_grad
    loss = torch.nn.L1Loss()(pred, ((b["label"] - fx["mean"]) / fx["mad"]).cuda())
    loss.backward()
    assert abs(loss.item() - c["loss0"]) <= 1e-4 * max(1.0, c["loss0"])
    worst, worst_key = 0.0, None
    for k, p in clf.named_parameters():
        assert p.grad is not None, k
        ref = c["grads"][k]
        f = p.grad.detach().double().reshape(-1).cpu()
        scale = max(ref["norm"], 1e-12)
        err = max(abs(float(f.norm()) - ref["norm"]) / scale, abs(float(f.sum()) - ref["sum"]) / scale,
                  float((f[ref["idx"]].float() - ref["vals"]).abs().max()) / scale)
        if err > worst:
            worst, worst_key = err, k
    print(f"{name}: worst gradient error {worst:.3e} ({worst_key})")
    assert worst < GRAD_TOL, (worst_key, worst)


def _layouts():
    import bdiff
    hist = bdiff.sample_num_nodes(bdiff.QM9_N_NODES, 128, seed=4)
    hist[0], hist[1] = 1, 29
    return {
        "qm9_hist_128": (hist, (7, True, False)),
        "with_128_atoms": ([128, 3, 127, 1, 65, 64, 2], (2, True, False)),
        "one_atom_molecules": ([1, 1, 5, 1, 1], (2, True, True)),
        "pairs_fill_tiles": ([8, 8, 11, 2, 1, 1, 1], (3, False, True)),    # 64 + 64 | 121 + 4 + 1 + 1 + 1: two full tiles
        "pairs_cross_tiles": ([9, 8, 8, 7, 13], (2, True, False)),
    }


@pytest.mark.parametrize("layout", ["qm9_hist_128", "with_128_atoms", "one_atom_molecules", "pairs_fill_tiles",
                                    "pairs_cross_tiles"])
def test_gradients_against_float64_oracle(layout):
    sizes, (n_layers, attention, node_attr) = _layouts()[layout]
    sizes, x, oh = _molecules(sizes, 8)
    sd = CO.random_state_dict(21, n_layers, attention, node_attr)
    clf = _clf(n_layers, attention, node_attr, sd)
    d_pred = torch.randn(sizes.numel(), generator=torch.Generator().manual_seed(3))
    ref_pred, ref = CB.packed_backward({k: v.double() for k, v in sd.items()}, n_layers, attention, node_attr,
                                       x.double(), oh.double(), sizes, d_pred.double())
    pred = clf.predict(x.cuda(), oh.cuda(), sizes)
    (pred * d_pred.cuda()).sum().backward()
    assert (pred.detach().double().cpu() - ref_pred).abs().max().item() <= 1e-4 * max(1.0, ref_pred.abs().max().item())
    worst, worst_key = 0.0, None
    for k, p in clf.named_parameters():
        r = ref[k]
        err = (p.grad.double().cpu() - r).abs().max().item() / max(r.norm().item(), 1e-12)
        if err > worst:
            worst, worst_key = err, k
    print(f"{layout}: worst gradient error {worst:.3e} ({worst_key})")
    assert worst < GRAD_TOL, (worst_key, worst)


def test_reproducible_and_training_pred_equals_predict():
    import bdiff
    sizes = bdiff.sample_num_nodes(bdiff.QM9_N_NODES, 64, seed=2)
    sizes, x, oh = _molecules(sizes, 5)
    clf = _clf(7, True, False, CO.random_state_dict(7))
    x, oh = x.cuda(), oh.cuda()
    with torch.no_grad():
        infer = clf.predict(x, oh, sizes)
    runs = []
    for _ in range(2):
        clf.zero_grad(set_to_none=True)
        pred = clf.predict(x, oh, sizes)
        assert torch.equal(pred.detach(), infer)
        (pred * torch.linspace(-1, 1, pred.numel(), device="cuda")).sum().backward()
        runs.append({k: p.grad.clone() for k, p in clf.named_parameters()})
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k


def _loop(clf, fx, data, labels):
    """The train branch of train_with_property_classifier (:160-190), restated line for line: scheduler first, then per
    batch zero_grad, the dense call, L1 loss against the normalised label, backward, step."""
    loss_l1 = torch.nn.L1Loss()
    optimizer = torch.optim.Adam(clf.parameters(), lr=fx["lr"])
    lr_scheduler = torch.optim.lr_scheduler.CosineAnnealingLR(optimizer, fx["t_max"])
    lr_scheduler.step()
    loss_arr = []
    for d, label in zip(data, labels):
        clf.train()
        optimizer.zero_grad()
        pred = clf(**_dense(d))
        loss = loss_l1(pred, (label - fx["mean"]) / fx["mad"])
        loss.backward()
        optimizer.step()
        loss_arr.append(loss.item())
    return loss_arr, optimizer


# Measured on an H100 80GB HBM3 (700 W): the largest |loss - loss_arr| over both configurations and all three batches
# is 2.5e-5 (DESIGN §4d), 4x under the tolerance.  Losses are O(1); batch 0 differs only by the forward's fp32 /
# split-bf16 rounding (~1e-6); batches 1 and 2 follow one and two Adam steps, whose update m / sqrt(v) carries the
# gradients' ~1e-5 relative error into the weights.
LOSS_TOL = 1e-4


@pytest.mark.parametrize("name", ["l7_att", "l2_nodeattr"])
def test_reference_training_loop(name):
    fx = load_golden("classifier_train_qm9")
    c = fx["configs"][name]
    clf = _clf(c["n_layers"], c["attention"], c["node_attr"],
               CO.random_state_dict(c["seed"], c["n_layers"], c["attention"], c["node_attr"]))
    data = [CO.dense_batch(b["x"].cuda(), b["one_hot"].cuda(), b["num_nodes"]) for b in fx["batches"]]
    labels = [b["label"].cuda() for b in fx["batches"]]
    loss_arr, optimizer = _loop(clf, fx, data, labels)
    diff = max(abs(a - b) for a, b in zip(loss_arr, c["loss_arr"]))
    print(f"{name}: loss_arr {loss_arr} vs reference {c['loss_arr']}: max |diff| {diff:.3e}")
    assert diff <= LOSS_TOL, (loss_arr, c["loss_arr"])
    # 50 further steps on batch 0 lower the loss
    d, label = data[0], (labels[0] - fx["mean"]) / fx["mad"]
    losses = []
    for _ in range(50):
        optimizer.zero_grad()
        loss = torch.nn.L1Loss()(clf(**_dense(d)), label)
        loss.backward()
        optimizer.step()
        losses.append(loss.item())
    print(f"{name}: 50 steps on batch 0: {losses[0]:.4f} -> {losses[-1]:.4f}")
    assert losses[-1] < 0.5 * losses[0]


def test_backward_after_newer_forward_raises():
    import bdiff
    sizes, x, oh = _molecules([4, 9], 1)
    clf = _clf(1, True, False, CO.random_state_dict(2, 1, True, False))
    p1 = clf.predict(x.cuda(), oh.cuda(), sizes)
    p2 = clf.predict(x.cuda(), oh.cuda(), sizes)
    with pytest.raises(bdiff.BdiffError):
        p1.sum().backward()
    p2.sum().backward()
    assert all(p.grad is not None for p in clf.parameters())

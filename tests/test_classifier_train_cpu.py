"""CPU: the classifier's hand-derived float64 backward (classifier_backward.packed_backward, the formula sheet of the CUDA
training pass) against torch.autograd, the oracle against the reference training fixture (gradients and the loss
trajectory of train_with_property_classifier), and a compile guard of the reverse-sweep kernels."""
import os
import re
import shutil
import subprocess

import pytest
import torch

import classifier_backward as CB
import classifier_oracle as CO
from conftest import ROOT, load_golden


def _cases():
    fx = load_golden("classifier_train_qm9")
    return fx, list(fx["configs"].items())


def _dense_pred(sd, c, d):
    bs, n, _ = d["positions"].shape
    return CO.dense_forward(sd, c["n_layers"], c["attention"], c["node_attr"], d["one_hot"].view(bs * n, -1),
                            d["positions"].view(bs * n, -1), d["atom_mask"].view(bs * n, 1).float(), d["edge_mask"].float(), n)


@pytest.mark.parametrize("name", ["l7_att", "l2_nodeattr"])
def test_hand_backward_matches_autograd_float64(name):
    fx, _ = _cases()
    c = fx["configs"][name]
    sd = {k: v.double() for k, v in CO.random_state_dict(c["seed"], c["n_layers"], c["attention"], c["node_attr"]).items()}
    g = torch.Generator().manual_seed(1)
    for b in fx["batches"]:
        x, oh, nn = b["x"].double(), b["one_hot"].double(), b["num_nodes"]
        d_pred = torch.randn(nn.numel(), generator=g, dtype=torch.float64)
        pred, grads = CB.packed_backward(sd, c["n_layers"], c["attention"], c["node_attr"], x, oh, nn, d_pred)
        sda = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
        ref = CO.packed_forward(sda, c["n_layers"], c["attention"], c["node_attr"], x, oh, nn)
        (ref * d_pred).sum().backward()
        assert (pred - ref.detach()).abs().max().item() <= 1e-12 * max(1.0, ref.abs().max().item())
        assert set(grads) == set(sd)
        for k in sd:
            scale = sda[k].grad.abs().max().item()
            assert (grads[k] - sda[k].grad).abs().max().item() <= 1e-10 * max(scale, 1e-30), k


@pytest.mark.parametrize("name", ["l7_att", "l2_nodeattr"])
def test_oracle_reproduces_reference_training_fixture(name):
    """Gradient fingerprints of the train branch's L1 loss on batch 0 (oracle autograd in float64), then the reference
    loop restated on the oracle in float32 (Adam lr 1e-3, CosineAnnealingLR stepped before the batches): the same losses
    as the reference's loss_arr."""
    fx, _ = _cases()
    c = fx["configs"][name]
    sd = CO.random_state_dict(c["seed"], c["n_layers"], c["attention"], c["node_attr"])
    assert abs(CO.checksum(sd) - c["checksum"]) <= 1e-9 * abs(c["checksum"])
    b0 = fx["batches"][0]
    d64 = CO.dense_batch(b0["x"].double(), b0["one_hot"].double(), b0["num_nodes"])
    params = {k: v.double().requires_grad_(True) for k, v in sd.items()}
    loss = torch.nn.functional.l1_loss(_dense_pred(params, c, d64), ((b0["label"] - fx["mean"]) / fx["mad"]).double())
    loss.backward()
    assert abs(loss.item() - c["loss0"]) <= 1e-6
    for k, p in params.items():
        ref = c["grads"][k]
        f = p.grad.reshape(-1)
        scale = max(ref["norm"], 1e-12)
        err = max(abs(float(f.norm()) - ref["norm"]), abs(float(f.sum()) - ref["sum"]),
                  float((f[ref["idx"]].float() - ref["vals"]).abs().max())) / scale
        # the bar is the fixture's own float32 error: at most 1.1e-5 of the norm (gcl_0.att_mlp.0.weight of l7_att, a
        # sum over pairs with heavy cancellation) against these float64 gradients
        assert err < 5e-5, (k, err)
    data = [CO.dense_batch(b["x"], b["one_hot"], b["num_nodes"]) for b in fx["batches"]]
    labels = [(b["label"] - fx["mean"]) / fx["mad"] for b in fx["batches"]]
    params = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    opt = torch.optim.Adam(list(params.values()), lr=fx["lr"])
    sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, fx["t_max"])
    sched.step()
    for d, y, ref in zip(data, labels, c["loss_arr"]):
        opt.zero_grad()
        loss = torch.nn.functional.l1_loss(_dense_pred(params, c, d), y)
        loss.backward()
        opt.step()
        assert abs(loss.item() - ref) <= 1e-5 * max(1.0, abs(ref)), (loss.item(), ref)


def _nvcc():
    found = shutil.which("nvcc")
    if found:
        return found
    cand = "/usr/local/cuda/bin/nvcc"
    return cand if os.path.exists(cand) else None


def test_reverse_sweep_kernels_compile_without_spills(tmp_path):
    """Every kernel of bdiff_classifier.cu (the reverse sweep included) compiles for sm_90a with no spills and no C7520;
    k_clf_bwd_edge issues its two K = 128 GEMMs (z2 and da) as 48 HGMMAs per tile."""
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    csrc = os.path.join(ROOT, "bio-diffusion_b200", "csrc")
    obj = str(tmp_path / "bdiff_classifier.o")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                        os.path.join(csrc, "bdiff_classifier.cu"), "-o", obj], capture_output=True, text=True, cwd=csrc)
    assert r.returncode == 0, r.stderr[-4000:]
    log = r.stdout + r.stderr
    assert "C7520" not in log, log
    kernels = re.findall(r"Compiling entry function '(\w+)'", log)
    for name in ("k_clf_bwd_edge", "k_clf_bwd_node", "k_clf_bwd_nodedec", "k_clf_bwd_dh_edge", "k_clf_bwd_pairs",
                 "k_clf_bwd_readout", "k_clf_wgrad", "k_clf_nodeILb1", "k_clf_readoutILb1"):
        assert any(name in k for k in kernels), name
    spills = re.findall(r"(\d+) bytes spill stores, (\d+) bytes spill loads", log)
    assert spills and all(int(a) == 0 and int(b) == 0 for a, b in spills), spills
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", obj], capture_output=True, text=True,
                          check=True).stdout
    cur, hg = None, 0
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        if cur and "k_clf_bwd_edge" in cur:
            hg += "HGMMA." in line
    assert hg >= 48, hg

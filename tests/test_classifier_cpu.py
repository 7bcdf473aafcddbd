"""CPU: the EGNN property classifier's oracle against the reference fixture, its dense and packed forms against each
other, the checkpoint contract of bdiff.PropertyClassifier, input validation, and a compile guard of the edge kernel."""
import os
import pickle
import re
import shutil
import subprocess
from argparse import Namespace

import pytest
import torch

import classifier_oracle as CO
from conftest import ROOT, load_golden


def _cases():
    fx = load_golden("classifier_qm9")
    return fx, list(fx["configs"].items())


def test_oracle_matches_reference_fixture():
    fx, cases = _cases()
    for name, c in cases:
        sd = CO.random_state_dict(c["seed"], c["n_layers"], c["attention"], c["node_attr"])
        assert abs(CO.checksum(sd) - c["checksum"]) <= 1e-9 * abs(c["checksum"]), f"{name}: regenerated weights differ"
        for b, ref in zip(fx["batches"], c["pred"]):
            d = CO.dense_batch(b["x"], b["one_hot"], b["num_nodes"])
            bs, n, _ = d["positions"].shape
            dense = CO.dense_forward(sd, c["n_layers"], c["attention"], c["node_attr"], d["one_hot"].view(bs * n, -1),
                                     d["positions"].view(bs * n, -1), d["atom_mask"].view(bs * n, 1).float(),
                                     d["edge_mask"].float(), n)
            packed = CO.packed_forward(sd, c["n_layers"], c["attention"], c["node_attr"], b["x"], b["one_hot"], b["num_nodes"])
            assert (dense - ref).abs().max().item() <= 1e-6 * max(1.0, ref.abs().max().item()), name
            assert (packed - ref).abs().max().item() <= 1e-6 * max(1.0, ref.abs().max().item()), name


def test_oracle_dense_equals_packed_in_float64():
    fx, _ = _cases()
    sd = {k: v.double() for k, v in CO.random_state_dict(3, 3, True, True).items()}
    b = fx["batches"][1]
    x, oh = b["x"].double(), b["one_hot"].double()
    d = CO.dense_batch(x, oh, b["num_nodes"])
    bs, n, _ = d["positions"].shape
    dense = CO.dense_forward(sd, 3, True, True, d["one_hot"].view(bs * n, -1), d["positions"].view(bs * n, -1),
                             d["atom_mask"].view(bs * n, 1).double(), d["edge_mask"].double(), n)
    packed = CO.packed_forward(sd, 3, True, True, x, oh, b["num_nodes"])
    assert dense.dtype == torch.float64
    assert (dense - packed).abs().max().item() <= 1e-12 * max(1.0, dense.abs().max().item())


def test_checkpoint_contract():
    import bdiff
    clf = bdiff.PropertyClassifier(in_node_nf=5, in_edge_nf=0, hidden_nf=128, n_layers=7, attention=1, node_attr=0)
    sd = clf.state_dict()
    assert len(sd) == 80 and sum(v.numel() for v in sd.values()) == 743944
    assert {k: tuple(v.shape) for k, v in sd.items()} == CO.param_shapes(7, True, False)
    clf.load_state_dict(CO.random_state_dict(1), strict=True)
    small = bdiff.PropertyClassifier(n_layers=2, attention=0, node_attr=1)
    assert {k: tuple(v.shape) for k, v in small.state_dict().items()} == CO.param_shapes(2, False, True)


def test_from_dir(tmp_path):
    import bdiff
    with open(tmp_path / "args.pickle", "wb") as f:
        pickle.dump(Namespace(nf=128, n_layers=2, attention=0, node_attr=1, model_name="egnn"), f)
    sd = CO.random_state_dict(5, 2, False, True)
    torch.save(sd, str(tmp_path / "best_checkpoint.npy"))
    clf = bdiff.PropertyClassifier.from_dir(str(tmp_path))
    assert clf.n_layers == 2 and not clf.attention and clf.node_attr == 1
    for k, v in clf.state_dict().items():
        assert torch.equal(v, sd[k])


def test_unsupported_options_raise():
    import bdiff
    for kw in (dict(hidden_nf=64), dict(in_edge_nf=1), dict(in_node_nf=6), dict(act_fn=torch.nn.ReLU())):
        with pytest.raises(NotImplementedError):
            bdiff.PropertyClassifier(**kw)


def test_bad_input_is_rejected():
    import bdiff
    clf = bdiff.PropertyClassifier(n_layers=1).requires_grad_(False)
    x, oh = torch.zeros(10, 3), torch.zeros(10, 5)
    with pytest.raises(ValueError):
        clf.predict(x, torch.zeros(10, 6), torch.tensor([4, 6]))           # one-hot width
    with pytest.raises(ValueError):
        clf.predict(x, oh, torch.tensor([4, 5]))                           # num_nodes does not sum to N
    with pytest.raises(ValueError):
        clf.predict(torch.zeros(130, 3), torch.zeros(130, 5), torch.tensor([129, 1]))   # more than 128 atoms
    with pytest.raises(bdiff.BdiffError):
        clf.predict(x, oh, torch.tensor([4, 6]))                           # valid, but no CPU fallback
    nm = torch.tensor([[1, 1, 1, 0], [1, 1, 0, 0]], dtype=torch.bool)
    em = nm.unsqueeze(1) & nm.unsqueeze(2)                                 # diagonal kept: not the standard mask
    with pytest.raises(ValueError):
        clf(h0=torch.zeros(8, 5), x=torch.zeros(8, 3), edges=None, edge_attr=None, node_mask=nm.view(8, 1).float(),
            edge_mask=em.view(32, 1).float(), n_nodes=4)
    trainable = bdiff.PropertyClassifier(n_layers=1)
    with pytest.raises(RuntimeError):
        trainable.predict(x, oh, torch.tensor([4, 6]))                     # inference only


# ---------------------------------------------------------------------------------------------- compile guard
def _nvcc():
    found = shutil.which("nvcc")
    if found:
        return found
    cand = "/usr/local/cuda/bin/nvcc"
    return cand if os.path.exists(cand) else None


def test_edge_kernel_compiles_to_back_to_back_wgmma(tmp_path):
    """k_clf_edge: HGMMA present, no C7520 (wgmmas serialized on a path ptxas cannot prove warp-uniform), one
    WARPGROUP.DEPBAR for its 24 HGMMAs per tile, and no spills."""
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
    sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", obj], capture_output=True, text=True,
                          check=True).stdout
    cur, hg, dep = None, 0, 0
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        if cur and "k_clf_edge" in cur:
            hg += "HGMMA." in line
            dep += "WARPGROUP.DEPBAR" in line
    assert hg >= 24 and 0 < dep <= hg // 24, (hg, dep)
    lines = log.splitlines()
    i = next(i for i, ln in enumerate(lines) if "Compiling entry function" in ln and "k_clf_edge" in ln)
    props = next(x for x in lines[i + 1:] if "spill stores" in x)
    st, ld = (int(v) for v in re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", props).groups())
    assert st == 0 and ld == 0, props

#!/usr/bin/env python
"""Golden fixture for the EGNN property classifier: predictions of the UNMODIFIED reference `EGNN` (src/__init__.py:
368-419) and the MAE of its `test_with_property_classifier` (:144-230), imported through oracle/ref_shim.py.  Dense
batches are built exactly as ConditionalDiffusionDataLoader.sample builds them (mol_gen_eval_conditional_qm9.py:124-139),
with molecule sizes that include n = 1 and n = 29.  Weights are not stored: they are regenerated from the seed by
classifier_oracle.random_state_dict, and the fixture keeps their checksum.
Run:  python tests/golden/make_golden_classifier.py"""
import os
import sys

import torch
import torch._dynamo  # noqa: F401  (before the stub modules are installed)

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ref_shim  # noqa: E402

ref_shim.install()
from src import EGNN, test_with_property_classifier  # noqa: E402
import classifier_oracle as CO  # noqa: E402

CONFIGS = [  # (name, n_layers, attention, node_attr, seed)
    ("l7_att", 7, True, False, 11),
    ("l2_nodeattr", 2, False, True, 12),
]
BATCHES = [[1, 7, 29, 19], [12, 29, 3, 9, 5, 1]]
MEAN, MAD = 75.2, 6.3          # an alpha-like normaliser (mean, mean absolute deviation)


def molecules(seed, sizes):
    g = torch.Generator().manual_seed(seed)
    n = sum(sizes)
    x = torch.randn((n, 3), generator=g) * 1.6
    one_hot = torch.nn.functional.one_hot(torch.randint(0, 5, (n,), generator=g), 5).float()
    label = MEAN + MAD * torch.randn((len(sizes),), generator=g)
    return x, one_hot, torch.tensor(sizes, dtype=torch.int64), label


def main():
    out = {"batches": [], "configs": {}, "mean": MEAN, "mad": MAD, "property": "alpha"}
    data = []
    for b, sizes in enumerate(BATCHES):
        x, one_hot, nn, label = molecules(100 + b, sizes)
        out["batches"].append({"x": x, "one_hot": one_hot, "num_nodes": nn, "label": label})
        d = CO.dense_batch(x, one_hot, nn)
        d["alpha"] = label
        data.append(d)
    for name, n_layers, attention, node_attr, seed in CONFIGS:
        sd = CO.random_state_dict(seed, n_layers, attention, node_attr)
        model = EGNN(in_node_nf=5, in_edge_nf=0, hidden_nf=128, device="cpu", n_layers=n_layers, coords_weight=1.0,
                     attention=attention, node_attr=int(node_attr))
        model.load_state_dict(sd, strict=True)
        model.eval()
        preds = []
        with torch.no_grad():
            for d in data:
                bs, n_nodes, _ = d["positions"].shape
                rows, cols = [], []
                for bi in range(bs):                # get_classifier_adj_matrix (:117-141)
                    for i in range(n_nodes):
                        for j in range(n_nodes):
                            rows.append(i + bi * n_nodes)
                            cols.append(j + bi * n_nodes)
                edges = [torch.LongTensor(rows), torch.LongTensor(cols)]
                pred = model(h0=d["one_hot"].view(bs * n_nodes, -1), x=d["positions"].view(bs * n_nodes, -1), edges=edges,
                             edge_attr=None, node_mask=d["atom_mask"].view(bs * n_nodes, -1).float(),
                             edge_mask=d["edge_mask"].float(), n_nodes=n_nodes)
                preds.append(pred.clone())
            mae = test_with_property_classifier(model=model, epoch=0, dataloader=data, mean=MEAN, mad=MAD, property="alpha",
                                                device="cpu", log_interval=1000)
        out["configs"][name] = {"n_layers": n_layers, "attention": attention, "node_attr": node_attr, "seed": seed,
                                "checksum": CO.checksum(sd), "pred": preds, "mae": float(mae)}
        print(f"{name}: mae {mae:.6f}, pred[0][:4] {preds[0][:4].tolist()}")
    torch.save(out, os.path.join(ROOT, "tests", "golden", "classifier_qm9.pt"))


if __name__ == "__main__":
    main()

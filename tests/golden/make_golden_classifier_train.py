#!/usr/bin/env python
"""Golden fixture for training the EGNN property classifier, from the UNMODIFIED reference `EGNN` (src/__init__.py:
368-419) and its own `train_with_property_classifier` (:144-204), imported through oracle/ref_shim.py.  Both configurations
of make_golden_classifier.py (weights regenerated from the seed, checksum kept), dense batches built as that script
builds them (ConditionalDiffusionDataLoader.sample, mol_gen_eval_conditional_qm9.py:124-139), n = 1 and n = 29 included.
Stores per configuration:
  grads     per-parameter fingerprints (L2 norm, sum, 8 strided entries) of the train branch's L1 loss on batch 0;
  loss_arr  the per-batch losses of train_with_property_classifier(partition="train") over the 3 batches with
            torch.optim.Adam(lr=1e-3) and CosineAnnealingLR(T_max=10) (the loop steps the scheduler first).
Run:  python tests/golden/make_golden_classifier_train.py"""
import os
import sys

import torch

import make_golden_classifier as MG          # installs ref_shim (the reference `src` package)
from src import EGNN, train_with_property_classifier  # noqa: E402
import classifier_oracle as CO  # noqa: E402

BATCHES = [[1, 7, 29, 19], [12, 29, 3, 9, 5, 1], [17, 9, 23, 4, 11]]
LR, T_MAX = 1e-3, 10


def grad_fingerprint(g):
    f = g.detach().double().reshape(-1)
    idx = torch.linspace(0, f.numel() - 1, steps=min(8, f.numel())).long()
    return dict(norm=float(f.norm()), sum=float(f.sum()), idx=idx, vals=f[idx].float().clone())


def dense_call(model, d):
    """The model call of train_with_property_classifier (:176-186), edges from get_classifier_adj_matrix (:117-141)."""
    bs, n_nodes, _ = d["positions"].shape
    rows = [i + bi * n_nodes for bi in range(bs) for i in range(n_nodes) for _ in range(n_nodes)]
    cols = [j + bi * n_nodes for bi in range(bs) for _ in range(n_nodes) for j in range(n_nodes)]
    return model(h0=d["one_hot"].view(bs * n_nodes, -1), x=d["positions"].view(bs * n_nodes, -1),
                 edges=[torch.LongTensor(rows), torch.LongTensor(cols)], edge_attr=None,
                 node_mask=d["atom_mask"].view(bs * n_nodes, -1).float(), edge_mask=d["edge_mask"].float(), n_nodes=n_nodes)


def main():
    out = {"batches": [], "configs": {}, "mean": MG.MEAN, "mad": MG.MAD, "property": "alpha", "lr": LR, "t_max": T_MAX}
    data = []
    for b, sizes in enumerate(BATCHES):
        x, one_hot, nn, label = MG.molecules(200 + b, sizes)
        out["batches"].append({"x": x, "one_hot": one_hot, "num_nodes": nn, "label": label})
        d = CO.dense_batch(x, one_hot, nn)
        d["alpha"] = label
        data.append(d)
    for name, n_layers, attention, node_attr, seed in MG.CONFIGS:
        sd = CO.random_state_dict(seed, n_layers, attention, node_attr)

        def make():
            m = EGNN(in_node_nf=5, in_edge_nf=0, hidden_nf=128, device="cpu", n_layers=n_layers, coords_weight=1.0,
                     attention=attention, node_attr=int(node_attr))
            m.load_state_dict(sd, strict=True)
            return m

        # gradient of the train branch's loss on batch 0 (:188-190)
        model = make()
        model.train()
        d = data[0]
        loss = torch.nn.L1Loss()(dense_call(model, d), (d["alpha"] - MG.MEAN) / MG.MAD)
        loss.backward()
        grads = {k: grad_fingerprint(p.grad) for k, p in model.named_parameters()}
        # the reference loop itself; a forward hook records each prediction to restate loss_arr (local to the loop)
        model = make()
        preds = []
        model.register_forward_hook(lambda mod, args, res: preds.append(res.detach().clone()))
        opt = torch.optim.Adam(model.parameters(), lr=LR)
        sched = torch.optim.lr_scheduler.CosineAnnealingLR(opt, T_MAX)
        avg = train_with_property_classifier(model=model, epoch=0, dataloader=data, mean=MG.MEAN, mad=MG.MAD,
                                             property="alpha", device="cpu", partition="train", optimizer=opt,
                                             lr_scheduler=sched, log_interval=1000)
        loss_arr = [float(torch.nn.L1Loss()(p, (dd["alpha"] - MG.MEAN) / MG.MAD)) for p, dd in zip(preds, data)]
        sizes = [len(s) for s in BATCHES]
        assert abs(sum(l * s for l, s in zip(loss_arr, sizes)) / sum(sizes) - avg) < 1e-6
        out["configs"][name] = {"n_layers": n_layers, "attention": attention, "node_attr": node_attr, "seed": seed,
                                "checksum": CO.checksum(sd), "loss0": loss.item(), "grads": grads, "loss_arr": loss_arr,
                                "avg_loss": float(avg)}
        print(f"{name}: loss0 {loss.item():.6f}, loss_arr {loss_arr}")
    torch.save(out, os.path.join(MG.ROOT, "tests", "golden", "classifier_train_qm9.pt"))


if __name__ == "__main__":
    sys.exit(main())

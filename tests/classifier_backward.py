"""Hand-derived backward of EDM's EGNN property classifier (reference: src/__init__.py:233-419) in plain torch,
dtype-generic (float64 works): the formula sheet of the CUDA training pass (bdiff_classifier_train.cuh).  The forward
is classifier_oracle's packed form (real atoms only, the pairs of each molecule in (row, col) order, diagonal masked);
tests/test_classifier_train_cpu.py checks the sweep against torch.autograd through that oracle."""
import torch
import torch.nn.functional as F

from classifier_oracle import packed_pairs


def _dsilu(z):
    s = torch.sigmoid(z)
    return s * (1 + z * (1 - s))


def packed_backward(sd, n_layers, attention, node_attr, x, one_hot, num_nodes, d_pred):
    """Hand-derived reverse sweep of classifier_oracle.packed_forward: {name: d(sum_k pred_k d_pred_k) / d name} for
    every parameter (x and one_hot are data).  Plain torch ops, no autograd.  Returns (pred, grads)."""
    H = 128
    rows, cols, mol = packed_pairs(num_nodes, x.device)
    B = int(num_nodes.numel())
    W = {k: v.to(x) for k, v in sd.items()}
    mask = (rows != cols).to(x.dtype)[:, None]
    h0 = one_hot.to(x)
    radial = ((x[rows] - x[cols]) ** 2).sum(1, keepdim=True)
    lin = lambda n, v: F.linear(v, W[n + ".weight"], W[n + ".bias"])   # noqa: E731
    # ---- forward, keeping the tape
    h = lin("embedding", h0)
    tape = []
    for i in range(n_layers):
        p = f"gcl_{i}."
        W1 = W[p + "edge_mlp.0.weight"]
        z1 = (h @ W1[:, :H].T + W[p + "edge_mlp.0.bias"])[rows] + (h @ W1[:, H:2 * H].T)[cols] + radial * W1[:, 2 * H]
        a = F.silu(z1)
        z2 = lin(p + "edge_mlp.2", a)
        s = F.silu(z2)
        g = torch.sigmoid(lin(p + "att_mlp.0", s)) if attention else torch.ones_like(s[:, :1])
        agg = torch.zeros_like(h).index_add_(0, rows, s * g * mask)
        inp = torch.cat([h, agg, h0] if node_attr else [h, agg], dim=1)
        v = lin(p + "node_mlp.0", inp)
        u = F.silu(v)
        tape.append((h, z1, a, z2, s, g, inp, v, u))
        h = h + lin(p + "node_mlp.2", u)
    q = lin("node_dec.0", h)
    qs = F.silu(q)
    S = torch.zeros((B, H), dtype=x.dtype, device=x.device).index_add_(0, mol, lin("node_dec.2", qs))
    w = lin("graph_dec.0", S)
    ws = F.silu(w)
    pred = lin("graph_dec.2", ws).squeeze(1)
    # ---- reverse sweep
    G = {}

    def put(name, dW, db):
        G[name + ".weight"], G[name + ".bias"] = dW, db

    dp = d_pred.to(x)[:, None]                                          # [B, 1]
    put("graph_dec.2", dp.T @ ws, dp.sum(0))
    dw = (dp @ W["graph_dec.2.weight"]) * _dsilu(w)
    put("graph_dec.0", dw.T @ S, dw.sum(0))
    dy = (dw @ W["graph_dec.0.weight"])[mol]                             # the molecule sum
    put("node_dec.2", dy.T @ qs, dy.sum(0))
    dq = (dy @ W["node_dec.2.weight"]) * _dsilu(q)
    put("node_dec.0", dq.T @ h, dq.sum(0))
    dh = dq @ W["node_dec.0.weight"]
    for i in reversed(range(n_layers)):
        p = f"gcl_{i}."
        hl, z1, a, z2, s, g, inp, v, u = tape[i]
        put(p + "node_mlp.2", dh.T @ u, dh.sum(0))                       # h' = h + W4 u + b4
        dv = (dh @ W[p + "node_mlp.2.weight"]) * _dsilu(v)
        put(p + "node_mlp.0", dv.T @ inp, dv.sum(0))
        dinp = dv @ W[p + "node_mlp.0.weight"]
        dh = dh + dinp[:, :H]
        dm = dinp[:, H:2 * H][rows] * mask                               # agg_i = sum_j m_ij [i != j]
        if attention:                                                    # m = s g, g = sigmoid(w_att . s + b_att)
            dt = (dm * s).sum(1, keepdim=True) * g * (1 - g)
            put(p + "att_mlp.0", dt.T @ s, dt.sum(0))
            ds = dm * g + dt @ W[p + "att_mlp.0.weight"]
        else:
            ds = dm
        dz2 = ds * _dsilu(z2)
        put(p + "edge_mlp.2", dz2.T @ a, dz2.sum(0))
        dz1 = (dz2 @ W[p + "edge_mlp.2.weight"]) * _dsilu(z1)
        dP = torch.zeros_like(hl).index_add_(0, rows, dz1)               # z1 = P_i + Q_j + w_r r_ij
        dQ = torch.zeros_like(hl).index_add_(0, cols, dz1)
        W1 = W[p + "edge_mlp.0.weight"]
        put(p + "edge_mlp.0", torch.cat([dP.T @ hl, dQ.T @ hl, (dz1 * radial).sum(0)[:, None]], dim=1), dP.sum(0))
        dh = dh + dP @ W1[:, :H] + dQ @ W1[:, H:2 * H]
    put("embedding", dh.T @ h0, dh.sum(0))
    return pred, {k: G[k].reshape(W[k].shape) for k in sd}

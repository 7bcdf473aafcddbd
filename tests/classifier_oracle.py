"""Functional restatement of EDM's EGNN property classifier (reference: src/__init__.py:233-419), the oracle of the CUDA
classifier (bdiff.PropertyClassifier).  Plain torch, dtype-generic (float64 works), CPU or GPU.

Two entry points over the same layer code:
  dense_forward   the reference's call: h0 [B*n, 5], x [B*n, 3], node_mask [B*n, 1], edge_mask [B*n*n, 1] over the full
                  n x n pair list of every padded molecule (get_classifier_adj_matrix, :117-141);
  packed_forward  real atoms only (x [N, 3], one_hot [N, 5], num_nodes [B]), the pairs of each molecule in (row, col) order
                  with the diagonal masked — what the CUDA path computes.
"""
import math
from typing import Dict, Tuple

import torch
import torch.nn.functional as F

IN_NODE_NF = 5


def param_shapes(n_layers: int = 7, attention: bool = True, node_attr: bool = False, hidden_nf: int = 128
                 ) -> Dict[str, Tuple[int, ...]]:
    """State-dict names and shapes of EGNN(in_node_nf=5, in_edge_nf=0, hidden_nf, n_layers, attention, node_attr)
    (:385-403; E_GCL_mask deletes coord_mlp, :345)."""
    h = hidden_nf
    out = {"embedding.weight": (h, IN_NODE_NF), "embedding.bias": (h,)}
    for i in range(n_layers):
        p = f"gcl_{i}."
        out.update({p + "edge_mlp.0.weight": (h, 2 * h + 1), p + "edge_mlp.0.bias": (h,),
                    p + "edge_mlp.2.weight": (h, h), p + "edge_mlp.2.bias": (h,),
                    p + "node_mlp.0.weight": (h, 2 * h + (IN_NODE_NF if node_attr else 0)), p + "node_mlp.0.bias": (h,),
                    p + "node_mlp.2.weight": (h, h), p + "node_mlp.2.bias": (h,)})
        if attention:
            out.update({p + "att_mlp.0.weight": (1, h), p + "att_mlp.0.bias": (1,)})
    for m in ("node_dec", "graph_dec"):
        out.update({m + ".0.weight": (h, h), m + ".0.bias": (h,),
                    m + ".2.weight": ((1 if m == "graph_dec" else h), h), m + ".2.bias": ((1 if m == "graph_dec" else h),)})
    return out


def random_state_dict(seed: int, n_layers: int = 7, attention: bool = True, node_attr: bool = False
                      ) -> Dict[str, torch.Tensor]:
    """nn.Linear's default init range (uniform, bound 1/sqrt(fan_in)), drawn name by name in sorted order from one seeded
    generator: the same tensors on every machine."""
    shapes = param_shapes(n_layers, attention, node_attr)
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name in sorted(shapes):
        shape = shapes[name]
        fan_in = shape[1] if name.endswith("weight") else shapes[name[:-4] + "weight"][1]
        bound = 1.0 / math.sqrt(fan_in)
        sd[name] = (torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1).mul_(bound).to(torch.float32)
    return sd


def checksum(sd: Dict[str, torch.Tensor]) -> float:
    """Order-independent fingerprint of a state dict (float64 sum of |w| weighted by the position in the tensor)."""
    tot = 0.0
    for name in sorted(sd):
        v = sd[name].detach().double().reshape(-1)
        tot += float((v.abs() * torch.arange(1, v.numel() + 1, dtype=torch.float64).sqrt()).sum())
    return tot


def _lin(sd, name, v):
    return F.linear(v, sd[name + ".weight"].to(v), sd[name + ".bias"].to(v))


def _egnn(sd, n_layers, attention, node_attr, h0, x, rows, cols, edge_mask, node_mask, mol, num_mols):
    """EGNN.forward (:405-419) on an explicit pair list; pred [num_mols] = graph_dec(sum over molecule of node_dec(h))."""
    h = _lin(sd, "embedding", h0)
    radial = ((x[rows] - x[cols]) ** 2).sum(1, keepdim=True)                 # coord2radial, norm_diff=False (:331-340)
    for i in range(n_layers):
        p = f"gcl_{i}."
        m = F.silu(_lin(sd, p + "edge_mlp.0", torch.cat([h[rows], h[cols], radial], dim=1)))   # edge_model (:306-316)
        m = F.silu(_lin(sd, p + "edge_mlp.2", m))
        if attention:
            m = m * torch.sigmoid(_lin(sd, p + "att_mlp.0", m))
        m = m * edge_mask                                                      # E_GCL_mask.forward (:357)
        agg = torch.zeros_like(h).index_add_(0, rows, m)                       # unsorted_segment_sum over row (:320)
        inp = torch.cat([h, agg, h0] if node_attr else [h, agg], dim=1)
        h = h + _lin(sd, p + "node_mlp.2", F.silu(_lin(sd, p + "node_mlp.0", inp)))    # node_model, recurrent (:318-328)
    h = _lin(sd, "node_dec.2", F.silu(_lin(sd, "node_dec.0", h))) * node_mask
    hs = torch.zeros((num_mols, h.shape[1]), dtype=h.dtype, device=h.device).index_add_(0, mol, h)
    return _lin(sd, "graph_dec.2", F.silu(_lin(sd, "graph_dec.0", hs))).squeeze(1)


def dense_forward(sd, n_layers, attention, node_attr, h0, x, node_mask, edge_mask, n_nodes):
    """The reference's dense call EGNN(h0, x, edges, None, node_mask, edge_mask, n_nodes)."""
    nt = h0.shape[0]
    b = nt // n_nodes
    dev = h0.device
    loc = torch.arange(n_nodes, device=dev)
    base = (torch.arange(b, device=dev) * n_nodes)[:, None, None]
    rows = (base + loc[None, :, None].expand(b, n_nodes, n_nodes)).reshape(-1)
    cols = (base + loc[None, None, :].expand(b, n_nodes, n_nodes)).reshape(-1)
    mol = torch.arange(b, device=dev).repeat_interleave(n_nodes)
    return _egnn(sd, n_layers, attention, node_attr, h0, x, rows, cols, edge_mask.to(h0), node_mask.to(h0), mol, b)


def packed_pairs(num_nodes: torch.Tensor, device=None):
    """(rows, cols, mol) of the block-diagonal pair list in (row, col) order, self pairs included."""
    nn = num_nodes.to("cpu", torch.int64)
    rows, cols = [], []
    off = 0
    for n in nn.tolist():
        r = torch.arange(n).repeat_interleave(n) + off
        c = torch.arange(n).repeat(n) + off
        rows.append(r)
        cols.append(c)
        off += n
    mol = torch.arange(len(nn)).repeat_interleave(nn)
    return torch.cat(rows).to(device), torch.cat(cols).to(device), mol.to(device)


def packed_forward(sd, n_layers, attention, node_attr, x, one_hot, num_nodes):
    rows, cols, mol = packed_pairs(num_nodes, x.device)
    edge_mask = (rows != cols).to(x.dtype)[:, None]
    node_mask = torch.ones((x.shape[0], 1), dtype=x.dtype, device=x.device)
    return _egnn(sd, n_layers, attention, node_attr, one_hot, x, rows, cols, edge_mask, node_mask, mol, int(num_nodes.numel()))


def dense_batch(x, one_hot, num_nodes):
    """The dense batch ConditionalDiffusionDataLoader.sample builds from packed molecules
    (mol_gen_eval_conditional_qm9.py:124-139): positions [B, n, 3], atom_mask [B, n], edge_mask [B*n*n, 1], one_hot [B, n, 5]."""
    dev = x.device
    nn = num_nodes.to(dev)
    bs, n_max = int(nn.shape[0]), int(nn.max())
    node_mask = torch.arange(n_max, device=dev).unsqueeze(0) < nn.unsqueeze(-1)
    dense_x = torch.zeros((bs, n_max, x.shape[-1]), dtype=x.dtype, device=dev)
    dense_x[node_mask] = x
    dense_one_hot = torch.zeros((bs, n_max, one_hot.shape[-1]), dtype=one_hot.dtype, device=dev)
    dense_one_hot[node_mask] = one_hot
    edge_mask = node_mask.unsqueeze(1) * node_mask.unsqueeze(2)
    edge_mask *= ~torch.eye(n_max, dtype=torch.bool, device=dev).unsqueeze(0)
    return {"positions": dense_x, "atom_mask": node_mask, "edge_mask": edge_mask.view(bs * n_max * n_max, 1),
            "one_hot": dense_one_hot}

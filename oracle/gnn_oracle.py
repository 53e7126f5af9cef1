"""float64 edge-list torch layers of GCN and GraphSAGE (mean / gcn aggregators) on the unpartitioned graph: the
autograd reference that a distributed training step of adaqp_b200.model.DistGCN / DistSAGE is compared with.

    GCN        y = D_in^-1/2 A D_out^-1/2 x W + b                          (W stored [in, out], distGCN.py)
    SAGE mean  y = x Ws^T + (A x / clamp(in_deg, 1)) Wn^T + b              (nn.Linear weights [out, in])
    SAGE gcn   y = ((A x + x) / (clamp(in_deg, 1) + 1)) Wn^T + b           (no fc_self)

A[v, u] = 1 for every edge u -> v (src u, dst v); degrees are counted on the given edge list and clamped to 1 as in
the reference (AdaQP/model/ops.py:17-67).  The distributed backward aggregates with out-degree norms; on the
symmetric graphs used here they equal the in-degree norms autograd differentiates, which
tests/test_gnn_oracle_cpu.py checks against the numpy oracle.
"""
from __future__ import annotations

from .gat_oracle import global_from_layouts


def degrees(src, dst, n):
    """(in_deg, out_deg) of the edge list as float64 tensors, unclamped."""
    import torch
    ones = torch.ones(src.numel(), dtype=torch.float64)
    return (torch.zeros(n, dtype=torch.float64).index_add(0, dst, ones),
            torch.zeros(n, dtype=torch.float64).index_add(0, src, ones))


def _sum_in(src, dst, x):
    """(A x)[v] = sum_{u->v} x[u] as a sparse product (a dense x[src] of a dense graph would not fit in memory)."""
    import torch
    A = torch.sparse_coo_tensor(torch.stack([dst, src]), torch.ones(src.numel(), dtype=x.dtype), (x.shape[0],) * 2,
                                check_invariants=True)
    return torch.sparse.mm(A.coalesce(), x)


def torch_gcn_layer(src, dst, x, W, b):
    """D_in^-1/2 A D_out^-1/2 x W + b."""
    in_deg, out_deg = degrees(src, dst, x.shape[0])
    h = _sum_in(src, dst, x * out_deg.clamp(min=1).pow(-0.5).unsqueeze(1)) * in_deg.clamp(min=1).pow(-0.5).unsqueeze(1)
    return h @ W + b


def torch_sage_layer(src, dst, x, Wn, b, Ws=None, agg: str = "mean"):
    """fc_self(x) + fc_neigh(h_neigh) + bias for agg 'mean'; fc_neigh(h_neigh) + bias for 'gcn' (Ws unused)."""
    in_deg, _ = degrees(src, dst, x.shape[0])
    if agg == "mean":
        h = _sum_in(src, dst, x) / in_deg.clamp(min=1).unsqueeze(1)
        return x @ Ws.T + h @ Wn.T + b
    if agg == "gcn":
        h = (_sum_in(src, dst, x) + x) / (in_deg.clamp(min=1) + 1).unsqueeze(1)
        return h @ Wn.T + b
    raise ValueError(agg)


def mono_step(layouts, state, model: str, agg: str = "mean", n_layers: int = 3):
    """One training step of the float64 model on the unpartitioned graph behind `layouts` (dropout off, LayerNorm +
    ReLU between layers, cross entropy summed over the training nodes and divided by their number).
    `state` maps the distributed model's state_dict names to arrays.  Returns (logits in rank order, loss, gradient
    of every state entry, global (in_deg, out_deg) as numpy)."""
    import numpy as np
    import torch
    import torch.nn.functional as F
    indptr, indices, base = global_from_layouts(layouts)
    N = int(base[-1])
    dst = torch.from_numpy(np.repeat(np.arange(N), np.diff(indptr)))
    src = torch.from_numpy(indices)
    x = torch.from_numpy(np.concatenate([L.feat for L in layouts]).astype(np.float64))
    y = torch.from_numpy(np.concatenate([L.label for L in layouts]).astype(np.int64))
    train = torch.from_numpy(np.concatenate([L.train_mask for L in layouts]).astype(bool))
    P = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in state.items()}
    h = x
    for i in range(n_layers):
        if model == "gcn":
            h = torch_gcn_layer(src, dst, h, P[f"convs.{i}.weight"], P[f"convs.{i}.bias"])
        else:
            s = f"sages.{i}."
            h = torch_sage_layer(src, dst, h, P[s + "fc_neigh.weight"], P[s + "bias"], P.get(s + "fc_self.weight"), agg)
        if i < n_layers - 1:
            h = F.relu(F.layer_norm(h, (h.shape[1],), P[f"norms.{i}.weight"], P[f"norms.{i}.bias"], 1e-5))
    loss = F.cross_entropy(h[train], y[train], reduction="sum") / int(train.sum())
    loss.backward()
    in_deg, out_deg = degrees(src, dst, N)
    return (h.detach().numpy(), float(loss.detach()), {k: v.grad.numpy() for k, v in P.items()},
            (in_deg.numpy(), out_deg.numpy()))

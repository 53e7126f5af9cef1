"""DistSAGE: GraphSAGE layers (mean / gcn aggregators) over the distributed aggregation op
(reference: AdaQP/model/distSAGE.py:14-97), plus DGL's max-pool aggregator ('pool', an extension beyond the reference):
p = relu(fc_pool(x)) on the wgmma GEMM, the column-wise neighbourhood max of p over the halo exchange
(ops.DistAggSAGEPool, csrc/sage_pool.cu), then fc_self(x) + fc_neigh(max) + bias."""
from __future__ import annotations

from typing import Any

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch import Tensor
from torch.nn import init
from torch.nn.parameter import Parameter

from .. import dense, fused
from .ops import DistAggSAGE, DistAggSAGEPool

AGGREGATORS = ("mean", "gcn", "pool")


class DistSAGEConv(nn.Module):
    def __init__(self, in_feats: int, out_feats: int, aggregator_type: str = "mean", bias: int = True,
                 activation: Any = None):
        super().__init__()
        if aggregator_type not in AGGREGATORS:
            raise ValueError(f"Invalid aggregator_type. Must be one of {AGGREGATORS}. But got {aggregator_type!r} instead.")
        self._in_feats, self._out_feats = in_feats, out_feats
        self._activation, self._aggregator_type = activation, aggregator_type
        self.bias = Parameter(torch.zeros(out_feats)) if bias else None
        if aggregator_type == "pool":
            self.fc_pool = nn.Linear(in_feats, in_feats)
        if aggregator_type != "gcn":
            self.fc_self = nn.Linear(in_feats, out_feats, bias=False)
        self.fc_neigh = nn.Linear(in_feats, out_feats, bias=False)

    def reset_parameters(self):
        gain = nn.init.calculate_gain("relu")
        if self._aggregator_type == "pool":
            init.xavier_uniform_(self.fc_pool.weight, gain=gain)
            init.zeros_(self.fc_pool.bias)
        if self._aggregator_type != "gcn":
            init.xavier_uniform_(self.fc_self.weight, gain=gain)
        init.xavier_uniform_(self.fc_neigh.weight, gain=gain)
        if self.bias is not None:
            init.zeros_(self.bias)

    def forward(self, local_feats: Tensor, graph, layer: int) -> Tensor:
        if self._aggregator_type == "pool":
            p = F.relu(dense.linear_nk(local_feats, self.fc_pool.weight, self.fc_pool.bias))
            h_neigh = DistAggSAGEPool.apply(p, graph, layer, self.training)
        else:
            h_neigh = DistAggSAGE.apply(local_feats, graph, layer, self.training)
        rst = dense.linear_nk(h_neigh, self.fc_neigh.weight)           # wgmma 3xTF32 (adaqp_b200/dense.py)
        if self._aggregator_type != "gcn":
            rst = dense.linear_nk(local_feats, self.fc_self.weight) + rst
        if self.bias is not None:
            rst = rst + self.bias
        return self._activation(rst) if self._activation is not None else rst


class DistSAGE(nn.Module):
    def __init__(self, in_feats: int, h_feats: int, num_classes: int, num_layers: int, drop_rate: float,
                 use_norm: bool = True, aggregator_type: str = "mean"):
        super().__init__()
        dims = [in_feats] + [h_feats] * (num_layers - 1) + [num_classes]
        self.sages = nn.ModuleList(DistSAGEConv(dims[i], dims[i + 1], aggregator_type=aggregator_type)
                                   for i in range(num_layers))
        if use_norm:
            self.norms = nn.ModuleList(nn.LayerNorm(h_feats) for _ in range(num_layers - 1))
        self.drop_rate = drop_rate

    def reset_parameters(self):
        for m in list(self.sages) + list(getattr(self, "norms", [])):
            m.reset_parameters()

    def forward(self, g, feats: Tensor) -> Tensor:
        last = len(self.sages) - 1
        for i in range(last):
            feats = self.sages[i](feats, g, i)
            feats = F.dropout(feats, p=self.drop_rate, training=self.training)
            if hasattr(self, "norms"):
                feats = fused.layer_norm_relu(feats, self.norms[i])      # relu(norms[i](feats)), one pass (csrc/norm.cu)
            else:
                feats = F.relu(feats)
        return self.sages[last](feats, g, last)

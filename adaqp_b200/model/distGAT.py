"""DistGAT: graph attention layers over the distributed attention aggregation (an extension beyond the reference,
whose models are GCN and SAGE).

Each layer is DGL's GATConv with one projection shared by sources and destinations, negative slope 0.2, no attention
dropout and no residual: z = x W on the wgmma GEMM (adaqp_b200.dense, no bias), attention aggregation of z over the
halo exchange (ops.DistAggGAT, csrc/gat.cu), then + b.  Hidden layers concatenate `heads` heads of width
h_feats / heads; the last layer has one head of width num_classes.  Layers stack as in DistGCN: conv, dropout, fused
LayerNorm + ReLU.  Initialisation follows DGL: xavier_normal_(gain=calculate_gain('relu')) for W, a_l and a_r, zeros
for b."""
from __future__ import annotations

from typing import List, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch import Tensor
from torch.nn import init
from torch.nn.parameter import Parameter

from .. import dense, fused
from .ops import DistAggGAT


def gat_layer_shapes(h_feats: int, num_classes: int, num_layers: int, heads: int) -> Tuple[List[int], List[int]]:
    """(row width H * D, heads H) of every layer's z: what each layer exchanges."""
    if heads <= 0 or h_feats % heads != 0:
        raise ValueError(f"hidden_dim={h_feats} is not divisible by gat_heads={heads}")
    return [h_feats] * (num_layers - 1) + [num_classes], [heads] * (num_layers - 1) + [1]


class DistGATConv(nn.Module):
    def __init__(self, in_feats: int, out_feats: int, num_heads: int, bias: bool = True):
        super().__init__()
        self._in_feats, self._out_feats, self._num_heads = in_feats, out_feats, num_heads
        self.weight = Parameter(torch.empty(in_feats, num_heads * out_feats))
        self.attn_l = Parameter(torch.empty(num_heads, out_feats))
        self.attn_r = Parameter(torch.empty(num_heads, out_feats))
        self.bias = Parameter(torch.empty(num_heads * out_feats)) if bias else None
        self.reset_parameters()

    def reset_parameters(self):
        gain = init.calculate_gain("relu")
        init.xavier_normal_(self.weight, gain=gain)
        # DGL keeps the attention vectors as [1, H, D]: same fans
        init.xavier_normal_(self.attn_l.data.view(1, self._num_heads, self._out_feats), gain=gain)
        init.xavier_normal_(self.attn_r.data.view(1, self._num_heads, self._out_feats), gain=gain)
        if self.bias is not None:
            init.zeros_(self.bias)

    def forward(self, feats: Tensor, graph, layer: int) -> Tensor:
        z = dense.linear(feats, self.weight)                       # projection first: the exchange moves z
        rst = DistAggGAT.apply(z, self.attn_l, self.attn_r, graph, layer, self.training, self._num_heads)
        return rst + self.bias if self.bias is not None else rst


class DistGAT(nn.Module):
    def __init__(self, in_feats: int, h_feats: int, num_classes: int, num_layers: int, drop_rate: float,
                 use_norm: bool = True, heads: int = 4):
        super().__init__()
        widths, hs = gat_layer_shapes(h_feats, num_classes, num_layers, heads)
        dims_in = [in_feats] + widths[:-1]
        self.convs = nn.ModuleList(DistGATConv(dims_in[i], widths[i] // hs[i], hs[i]) for i in range(num_layers))
        if use_norm:
            self.norms = nn.ModuleList(nn.LayerNorm(h_feats) for _ in range(num_layers - 1))
        self.drop_rate = drop_rate

    def reset_parameters(self):
        for m in list(self.convs) + list(getattr(self, "norms", [])):
            m.reset_parameters()

    def forward(self, g, feats: Tensor) -> Tensor:
        last = len(self.convs) - 1
        for i in range(last):
            feats = self.convs[i](feats, g, i)
            feats = F.dropout(feats, p=self.drop_rate, training=self.training)
            if hasattr(self, "norms"):
                feats = fused.layer_norm_relu(feats, self.norms[i])
            else:
                feats = F.relu(feats, inplace=True)
        return self.convs[last](feats, g, last)

"""DistGATv2: GATv2 attention layers over the distributed attention aggregation (an extension beyond the reference,
whose models are GCN and SAGE).

Each layer is DGL's GATv2Conv with share_weights=False, negative slope 0.2, no attention dropout and no residual
(every node has a self-loop): zs = x W_s + b_s and zd = x W_d + b_d on the wgmma GEMM (two adaqp_b200.dense calls,
each at most 256 wide), then the attention aggregation of zs over the halo exchange (ops.DistAggGATv2,
csrc/gatv2.cu).  Layer shapes come from gat_layer_shapes: hidden layers concatenate `heads` heads of width
h_feats / heads, the last layer has one head of width num_classes.  Layers stack as in DistGAT: conv, dropout, fused
LayerNorm + ReLU.  Initialisation follows DGL: xavier_normal_(gain=calculate_gain('relu')) for W_s, W_d and attn,
zeros for the biases."""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch import Tensor
from torch.nn import init
from torch.nn.parameter import Parameter

from .. import dense, fused
from .distGAT import gat_layer_shapes
from .ops import DistAggGATv2


class DistGATv2Conv(nn.Module):
    def __init__(self, in_feats: int, out_feats: int, num_heads: int):
        super().__init__()
        self._in_feats, self._out_feats, self._num_heads = in_feats, out_feats, num_heads
        self.W_s = Parameter(torch.empty(in_feats, num_heads * out_feats))
        self.b_s = Parameter(torch.empty(num_heads * out_feats))
        self.W_d = Parameter(torch.empty(in_feats, num_heads * out_feats))
        self.b_d = Parameter(torch.empty(num_heads * out_feats))
        self.attn = Parameter(torch.empty(num_heads, out_feats))
        self.reset_parameters()

    def reset_parameters(self):
        gain = init.calculate_gain("relu")
        # DGL's fc_src / fc_dst are nn.Linear(in, H * D) (weight [H * D, in]): the same fans as W stored [in, H * D]
        init.xavier_normal_(self.W_s, gain=gain)
        init.xavier_normal_(self.W_d, gain=gain)
        init.xavier_normal_(self.attn.data.view(1, self._num_heads, self._out_feats), gain=gain)   # DGL: [1, H, D]
        init.zeros_(self.b_s)
        init.zeros_(self.b_d)

    def forward(self, feats: Tensor, graph, layer: int) -> Tensor:
        zs = dense.linear(feats, self.W_s, self.b_s)            # projections first: the exchange moves zs
        zd = dense.linear(feats, self.W_d, self.b_d)
        return DistAggGATv2.apply(zs, zd, self.attn, graph, layer, self.training, self._num_heads)


class DistGATv2(nn.Module):
    def __init__(self, in_feats: int, h_feats: int, num_classes: int, num_layers: int, drop_rate: float,
                 use_norm: bool = True, heads: int = 4):
        super().__init__()
        widths, hs = gat_layer_shapes(h_feats, num_classes, num_layers, heads)
        dims_in = [in_feats] + widths[:-1]
        self.convs = nn.ModuleList(DistGATv2Conv(dims_in[i], widths[i] // hs[i], hs[i]) for i in range(num_layers))
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

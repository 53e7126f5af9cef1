"""DistGCNII: GCNII (Chen et al., "Simple and Deep Graph Convolutional Networks"; PyG GCN2Conv, DGL GCN2Conv) with
shared weights over the distributed exchange, an extension beyond the reference, whose models are GCN and SAGE.

    x   = dropout(x)
    h_0 = relu(x W_in + b_in)
    for l = 1 .. L:
        d   = dropout(h_{l-1})
        s_l = (1 - alpha) A d + alpha h_0                     A = D^-1/2 A D^-1/2, the GCN norms
        h_l = relu(s_l W'_l),   W'_l = (1 - beta_l) I + beta_l W_l,   beta_l = log(theta / l + 1)
    logits = dropout(h_L) W_out + b_out

as PyG's examples/gcn2_cora.py.  The propagation is ops.DistGCNIIProp (the teleport step of csrc/spmm.cu, column-sliced
at hidden widths that are multiples of 128 above 128): 2L exchanges of hidden-width rows per training step.  The
identity mapping is folded into W'_l, an H x H autograd expression of every forward pass, so the existing wgmma GEMM
(adaqp_b200.dense) runs it and autograd gives dW_l = beta_l s_l^T dpre.  W_in, W_out and W_l are xavier_uniform_,
biases zero.  H is the yaml `hidden_dim`; GCNII has no LayerNorm, and `num_layers` / `use_norm` do not apply."""
from __future__ import annotations

import math
from numbers import Integral, Real
from typing import Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch import Tensor
from torch.nn import init
from torch.nn.parameter import Parameter

from .. import dense
from .distAPPNP import APPNPLinear
from .ops import DistGCNIIProp

GCNII_LAYERS = 8      # default of the yaml `model: gcnii_layers`
GCNII_ALPHA = 0.1     # default of the yaml `model: gcnii_alpha`
GCNII_THETA = 0.5     # default of the yaml `model: gcnii_theta`


def gcnii_params(layers, alpha, theta) -> Tuple[int, float, float]:
    """(L, alpha, theta) checked: L an integer >= 1, alpha a number in [0, 1], theta a finite number > 0."""
    if isinstance(layers, bool) or not (isinstance(layers, Integral)
                                        or (isinstance(layers, Real) and float(layers).is_integer())):
        raise ValueError(f"gcnii_layers={layers!r} is not an integer")
    if int(layers) < 1:
        raise ValueError(f"gcnii_layers={layers} must be at least 1")
    if isinstance(alpha, bool) or not isinstance(alpha, Real) or not 0.0 <= float(alpha) <= 1.0:
        raise ValueError(f"gcnii_alpha={alpha!r} is outside [0, 1]")
    if isinstance(theta, bool) or not isinstance(theta, Real) or not (math.isfinite(float(theta)) and float(theta) > 0):
        raise ValueError(f"gcnii_theta={theta!r} is not a finite number above 0")
    return int(layers), float(alpha), float(theta)


def gcnii_beta(theta: float, layer: int) -> float:
    """beta_l = log(theta / l + 1) of layer l = 1 .. L."""
    return math.log(theta / layer + 1.0)


class GCNIIConv(nn.Module):
    """The H x H weight W_l of one layer; the identity mapping W'_l is built in DistGCNII.forward."""

    def __init__(self, h_feats: int):
        super().__init__()
        self.weight = Parameter(torch.empty(h_feats, h_feats))
        self.reset_parameters()

    def reset_parameters(self):
        init.xavier_uniform_(self.weight)


class DistGCNII(nn.Module):
    def __init__(self, in_feats: int, h_feats: int, num_classes: int, drop_rate: float, layers: int = GCNII_LAYERS,
                 alpha: float = GCNII_ALPHA, theta: float = GCNII_THETA):
        super().__init__()
        self.layers, self.alpha, self.theta = gcnii_params(layers, alpha, theta)
        self.lins = nn.ModuleList([APPNPLinear(in_feats, h_feats), APPNPLinear(h_feats, num_classes)])
        self.convs = nn.ModuleList(GCNIIConv(h_feats) for _ in range(self.layers))
        self.drop_rate = drop_rate

    def reset_parameters(self):
        for m in list(self.lins) + list(self.convs):
            m.reset_parameters()

    def forward(self, g, feats: Tensor) -> Tensor:
        x = F.dropout(feats, p=self.drop_rate, training=self.training)
        h0 = F.relu(self.lins[0](x))
        h = h0
        for i, conv in enumerate(self.convs):
            d = F.dropout(h, p=self.drop_rate, training=self.training)
            s = DistGCNIIProp.apply(d, h0, g, self.alpha, self.training, i)    # exchanges d on forward{i}
            beta = gcnii_beta(self.theta, i + 1)
            eye = torch.eye(conv.weight.shape[0], dtype=conv.weight.dtype, device=conv.weight.device)
            h = F.relu(dense.linear(s, (1.0 - beta) * eye + beta * conv.weight))
        h = F.dropout(h, p=self.drop_rate, training=self.training)
        return self.lins[1](h)

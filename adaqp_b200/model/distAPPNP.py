"""DistAPPNP: APPNP (Klicpera et al., "Predict then Propagate"; DGL APPNPConv, PyG APPNP) over the distributed
exchange, an extension beyond the reference, whose models are GCN and SAGE.

An MLP transforms each node's features with no exchange, then K personalized-PageRank steps propagate its output:

    z = MLP(x)       h_0 = z       h_{k+1} = (1 - alpha) A h_k + alpha z       logits = h_K

with A = D^-1/2 A D^-1/2, the GCN norms (the graphs carry one self-loop per node).  The MLP has `num_layers` linear
layers num_feats -> hidden ... -> num_classes on the wgmma GEMM (adaqp_b200.dense), stacked as in DistGCN: linear,
dropout, fused LayerNorm + ReLU.  Weights are xavier_uniform_, biases zero, as DistGCNConv.  The propagation is
ops.DistAPPNPProp (csrc/spmm.cu appnp_prop_kernel): 2K exchanges of num_classes-wide rows per training step."""
from __future__ import annotations

from numbers import Integral, Real
from typing import Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F
from torch import Tensor
from torch.nn import init
from torch.nn.parameter import Parameter

from .. import dense, fused
from .ops import DistAPPNPProp

APPNP_K = 10          # default of the yaml `model: appnp_k`
APPNP_ALPHA = 0.1     # default of the yaml `model: appnp_alpha`


def appnp_params(k, alpha) -> Tuple[int, float]:
    """(K, alpha) checked: K an integer >= 1, alpha a number in [0, 1]."""
    if isinstance(k, bool) or not (isinstance(k, Integral) or (isinstance(k, Real) and float(k).is_integer())):
        raise ValueError(f"appnp_k={k!r} is not an integer")
    if int(k) < 1:
        raise ValueError(f"appnp_k={k} must be at least 1")
    if isinstance(alpha, bool) or not isinstance(alpha, Real) or not 0.0 <= float(alpha) <= 1.0:
        raise ValueError(f"appnp_alpha={alpha!r} is outside [0, 1]")
    return int(k), float(alpha)


class APPNPLinear(nn.Module):
    def __init__(self, in_feats: int, out_feats: int):
        super().__init__()
        self.weight = Parameter(torch.empty(in_feats, out_feats))
        self.bias = Parameter(torch.empty(out_feats))
        self.reset_parameters()

    def reset_parameters(self):
        init.xavier_uniform_(self.weight)
        init.zeros_(self.bias)

    def forward(self, x: Tensor) -> Tensor:
        return dense.linear(x, self.weight, self.bias)


class DistAPPNP(nn.Module):
    def __init__(self, in_feats: int, h_feats: int, num_classes: int, num_layers: int, drop_rate: float,
                 use_norm: bool = True, k: int = APPNP_K, alpha: float = APPNP_ALPHA):
        super().__init__()
        self.k, self.alpha = appnp_params(k, alpha)
        dims = [in_feats] + [h_feats] * (num_layers - 1) + [num_classes]
        self.lins = nn.ModuleList(APPNPLinear(dims[i], dims[i + 1]) for i in range(num_layers))
        if use_norm:
            self.norms = nn.ModuleList(nn.LayerNorm(h_feats) for _ in range(num_layers - 1))
        self.drop_rate = drop_rate

    def reset_parameters(self):
        for m in list(self.lins) + list(getattr(self, "norms", [])):
            m.reset_parameters()

    def forward(self, g, feats: Tensor) -> Tensor:
        last = len(self.lins) - 1
        for i in range(last):
            feats = self.lins[i](feats)
            feats = F.dropout(feats, p=self.drop_rate, training=self.training)
            if hasattr(self, "norms"):
                feats = fused.layer_norm_relu(feats, self.norms[i])
            else:
                feats = F.relu(feats, inplace=True)
        z = self.lins[last](feats)
        return DistAPPNPProp.apply(z, g, self.k, self.alpha, self.training)

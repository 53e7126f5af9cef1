"""float64 numpy restatement of GCNII (DESIGN.md §14), forward and backward, and of its distributed exchange protocol.

    h_0 = relu(x W_in + b_in)
    s_l = (1 - alpha) A h_{l-1} + alpha h_0,   p_l = s_l W'_l,   h_l = relu(p_l)      l = 1 .. L
    W'_l = (1 - beta_l) I + beta_l W_l,   beta_l = log(theta / l + 1)
    logits = h_L W_out + b_out

with dropout off and A = D^-1/2 A D^-1/2 (appnp_oracle.matrix).  Backward from G = dL/dlogits:

    dh_L = G W_out^T;  per layer l = L .. 1: dp = dh_l * [p_l > 0],  dW_l = beta_l s_l^T dp,  ds = dp W'_l^T,
    dh_{l-1} = (1 - alpha) A^T ds,  dh_0 += alpha ds;   dW_in = x^T (dh_0 * [x W_in + b_in > 0])

Parameters are keyed as the model's state_dict: lins.0.*, convs.{l-1}.weight, lins.1.*.  `dist_step` runs every rank
over prepared layouts (manager.layout) with each exchange simulated exactly (gat_oracle.exchange): layer l moves
h_{l-1} on forward{l-1} and ds_l on backward{l-1}; the weight gradients are the sums of the ranks' shares.
"""
from __future__ import annotations

import math
from typing import Dict, List, Sequence

import numpy as np

from .appnp_oracle import _local, _pow, exchange, global_from_layouts, matrix  # noqa: F401  (re-exported)


def beta(theta: float, layer: int) -> float:
    return math.log(theta / layer + 1.0)


def _eff(P: Dict[str, np.ndarray], l: int, theta: float) -> np.ndarray:
    """W'_l of layer l = 1 .. L."""
    W = np.asarray(P[f"convs.{l - 1}.weight"], np.float64)
    b = beta(theta, l)
    return (1.0 - b) * np.eye(W.shape[0]) + b * W


def _forward(props, x, P, L, alpha, theta):
    """props[l](rows) = A rows for layer l's rows (a closure, so that the distributed form can exchange first)."""
    q0 = np.asarray(x, np.float64) @ P["lins.0.weight"] + P["lins.0.bias"]
    h0 = np.maximum(q0, 0.0)
    h, saved = h0, []
    for l in range(1, L + 1):
        s = (1 - alpha) * props(l, h) + alpha * h0
        p = s @ _eff(P, l, theta)
        saved.append((s, p))
        h = np.maximum(p, 0.0)
    logits = h @ P["lins.1.weight"] + P["lins.1.bias"]
    return logits, {"q0": q0, "h0": h0, "hL": h, "saved": saved}


def _backward(props_t, x, P, L, alpha, theta, st, G):
    grads = {"lins.1.weight": st["hL"].T @ G, "lins.1.bias": G.sum(0)}
    dh = G @ np.asarray(P["lins.1.weight"], np.float64).T
    dh0 = np.zeros_like(st["h0"])
    for l in range(L, 0, -1):
        s, p = st["saved"][l - 1]
        dp = dh * (p > 0)
        grads[f"convs.{l - 1}.weight"] = beta(theta, l) * (s.T @ dp)
        ds = dp @ _eff(P, l, theta).T
        dh0 += alpha * ds
        dh = (1 - alpha) * props_t(l, ds)
    dq0 = (dh0 + dh) * (st["q0"] > 0)
    grads["lins.0.weight"] = np.asarray(x, np.float64).T @ dq0
    grads["lins.0.bias"] = dq0.sum(0)
    return grads


def monolithic(indptr, indices, x, P, G, L: int, alpha: float, theta: float):
    """Forward and backward on an unpartitioned graph (no halo): logits and the parameter gradients for dL/dlogits = G."""
    deg = np.diff(np.asarray(indptr, np.int64))
    A = matrix(indptr, indices, deg.size, _pow(deg, -0.5), _pow(deg, -0.5))
    logits, st = _forward(lambda l, h: A @ h, x, P, L, alpha, theta)
    grads = _backward(lambda l, g: A.T @ g, x, P, L, alpha, theta, st, G)
    return logits, grads


def dist_step(layouts, xs: Sequence[np.ndarray], P, Gs: Sequence[np.ndarray], L: int, alpha: float, theta: float):
    """Every rank's forward and backward with the protocol's exchanges.  Returns (per-rank logits, summed gradients,
    halos) where halos[key] is the per-rank list of halo rows received on `key`."""
    W = len(layouts)
    Af = [_local(Lr, True) for Lr in layouts]
    Ab = [_local(Lr, False) for Lr in layouts]
    halos: Dict[str, List[np.ndarray]] = {}
    # the ranks advance in lockstep: each layer's exchange needs every rank's rows of that layer
    q0 = [np.asarray(x, np.float64) @ P["lins.0.weight"] + P["lins.0.bias"] for x in xs]
    h0 = [np.maximum(q, 0.0) for q in q0]
    hs, saved = list(h0), [[] for _ in range(W)]
    for l in range(1, L + 1):
        halo = exchange(hs, layouts)
        halos[f"forward{l - 1}"] = halo
        for r in range(W):
            s = (1 - alpha) * (Af[r] @ np.concatenate([hs[r], halo[r]])) + alpha * h0[r]
            p = s @ _eff(P, l, theta)
            saved[r].append((s, p))
            hs[r] = np.maximum(p, 0.0)
    logits = [h @ P["lins.1.weight"] + P["lins.1.bias"] for h in hs]
    grads: Dict[str, np.ndarray] = {"lins.1.weight": sum(h.T @ G for h, G in zip(hs, Gs)),
                                    "lins.1.bias": sum(G.sum(0) for G in Gs)}
    dh = [G @ np.asarray(P["lins.1.weight"], np.float64).T for G in Gs]
    dh0 = [np.zeros_like(h) for h in h0]
    for l in range(L, 0, -1):
        dss = []
        grads[f"convs.{l - 1}.weight"] = 0.0
        for r in range(W):
            s, p = saved[r][l - 1]
            dp = dh[r] * (p > 0)
            grads[f"convs.{l - 1}.weight"] = grads[f"convs.{l - 1}.weight"] + beta(theta, l) * (s.T @ dp)
            ds = dp @ _eff(P, l, theta).T
            dh0[r] += alpha * ds
            dss.append(ds)
        halo = exchange(dss, layouts)
        halos[f"backward{l - 1}"] = halo
        dh = [(1 - alpha) * (Ab[r] @ np.concatenate([dss[r], halo[r]])) for r in range(W)]
    dq0 = [(dh0[r] + dh[r]) * (q0[r] > 0) for r in range(W)]
    grads["lins.0.weight"] = sum(np.asarray(x, np.float64).T @ d for x, d in zip(xs, dq0))
    grads["lins.0.bias"] = sum(d.sum(0) for d in dq0)
    return logits, grads, halos


# ---------------------------------------------------------------- float64 torch reference (edge list, autograd)
def torch_gcnii(src, dst, x, P, L: int, alpha: float, theta: float):
    """Plain edge-list GCNII in torch (float64 autograd reference, dropout off), GCN norms from the edge list.
    P maps the state_dict names to tensors."""
    import torch
    n = x.shape[0]
    ones = torch.ones_like(dst, dtype=x.dtype)
    deg_in = torch.zeros(n, dtype=x.dtype).index_add(0, dst, ones)
    deg_out = torch.zeros(n, dtype=x.dtype).index_add(0, src, ones)
    w = (deg_out.clamp(min=1).pow(-0.5)[src] * deg_in.clamp(min=1).pow(-0.5)[dst]).unsqueeze(1)
    h0 = torch.relu(x @ P["lins.0.weight"] + P["lins.0.bias"])
    h = h0
    for l in range(1, L + 1):
        s = (1 - alpha) * torch.zeros_like(h).index_add(0, dst, w * h[src]) + alpha * h0
        b = beta(theta, l)
        Wc = P[f"convs.{l - 1}.weight"]
        h = torch.relu(s @ ((1 - b) * torch.eye(Wc.shape[0], dtype=x.dtype) + b * Wc))
    return h @ P["lins.1.weight"] + P["lins.1.bias"]


def init_params(rng, F: int, H: int, C: int, L: int) -> Dict[str, np.ndarray]:
    """Random parameters with the model's names and shapes (xavier-like scale, small biases)."""
    P = {"lins.0.weight": rng.randn(F, H) * math.sqrt(2.0 / (F + H)), "lins.0.bias": rng.randn(H) * 0.1,
         "lins.1.weight": rng.randn(H, C) * math.sqrt(2.0 / (H + C)), "lins.1.bias": rng.randn(C) * 0.1}
    for l in range(L):
        P[f"convs.{l}.weight"] = rng.randn(H, H) * math.sqrt(1.0 / H)
    return P

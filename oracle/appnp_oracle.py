"""float64 numpy restatement of APPNP's propagation (DESIGN.md §13) and of its distributed exchange protocol.

    A = D^-1/2 A D^-1/2  (per edge u -> v: pre[u] * post[v], pre = out_deg^-1/2, post = in_deg^-1/2)
    forward:   h_0 = z,  h_{k+1} = (1 - alpha) A h_k + alpha z,  k = 0 .. K-1;  returns h_1 .. h_K
    backward:  g_K = dL/dh_K,  g_k = (1 - alpha) A^T g_{k+1};  dz = alpha sum_{k=1..K} g_k + g_0

The graphs are symmetric, so A^T is the matrix with the norms swapped (pre = in_deg^-1/2, post = out_deg^-1/2) over
the same CSR, which is how a rank computes it for its own rows.  `dist_forward` / `dist_backward` run every rank over
prepared layouts (manager.layout) with each step's exchange simulated exactly (gat_oracle.exchange).
"""
from __future__ import annotations

from typing import List, Sequence

import numpy as np
import scipy.sparse as sp

from .gat_oracle import exchange, global_from_layouts  # noqa: F401  (re-exported for the tests)


def _pow(deg, p):
    return np.power(np.maximum(np.asarray(deg, np.float64), 1.0), p)


def matrix(indptr, indices, n_src, pre, post) -> sp.csr_matrix:
    """[n_dst, n_src] CSR with entry (v, u) = pre[u] * post[v]."""
    indptr, indices = np.asarray(indptr, np.int64), np.asarray(indices, np.int64)
    n = indptr.size - 1
    dst = np.repeat(np.arange(n), np.diff(indptr))
    vals = np.asarray(pre, np.float64)[indices] * np.asarray(post, np.float64)[dst]
    return sp.csr_matrix((vals, indices, indptr), shape=(n, n_src))


def forward(A: sp.csr_matrix, z: np.ndarray, k: int, alpha: float) -> List[np.ndarray]:
    hs, h = [], z
    for _ in range(k):
        h = (1 - alpha) * (A @ h) + alpha * z
        hs.append(h)
    return hs


def backward(A: sp.csr_matrix, g_k: np.ndarray, k: int, alpha: float):
    """(dz, [g_K, g_{K-1}, ..., g_0])."""
    gs = [g_k]
    for _ in range(k):
        gs.append((1 - alpha) * (A.T @ gs[-1]))
    dz = alpha * sum(gs[:-1]) + gs[-1]
    return dz, gs


def monolithic(indptr, indices, z, g_k, k, alpha):
    """Forward and backward on an unpartitioned graph (no halo): h_1..h_K, dz and g_K..g_0."""
    deg = np.diff(np.asarray(indptr, np.int64))
    A = matrix(indptr, indices, deg.size, _pow(deg, -0.5), _pow(deg, -0.5))
    hs = forward(A, z, k, alpha)
    dz, gs = backward(A, g_k, k, alpha)
    return {"h": hs, "dz": dz, "g": gs}


def _local(L, fwd: bool):
    ind, outd = np.asarray(L.in_degrees), np.asarray(L.out_degrees)
    pre, post = (_pow(outd, -0.5), _pow(ind, -0.5)) if fwd else (_pow(ind, -0.5), _pow(outd, -0.5))
    return matrix(L.indptr, L.indices, L.n_inner + L.n_halo, pre, post)


def dist_forward(layouts, zs: Sequence[np.ndarray], k: int, alpha: float):
    """Per rank h_1..h_K of its inner rows and, per step, the halo rows it received (h_k of the owners)."""
    As = [_local(L, True) for L in layouts]
    hs = [[np.asarray(z, np.float64)] for z in zs]
    halos = []
    for _ in range(k):
        halo = exchange([h[-1] for h in hs], layouts)
        halos.append(halo)
        for r in range(len(layouts)):
            x = np.concatenate([hs[r][-1], halo[r]])
            hs[r].append((1 - alpha) * (As[r] @ x) + alpha * zs[r])
    return [h[1:] for h in hs], halos


def dist_backward(layouts, g_ks: Sequence[np.ndarray], k: int, alpha: float):
    """Per rank dz of its inner rows and, per step (backward{K-1} first), the halo rows it received."""
    As = [_local(L, False) for L in layouts]
    gs = [[np.asarray(g, np.float64)] for g in g_ks]
    halos = []
    for _ in range(k):
        halo = exchange([g[-1] for g in gs], layouts)
        halos.append(halo)
        for r in range(len(layouts)):
            x = np.concatenate([gs[r][-1], halo[r]])
            gs[r].append((1 - alpha) * (As[r] @ x))
    dz = [alpha * sum(g[:-1]) + g[-1] for g in gs]
    return dz, halos


def masses(A_abs: sp.csr_matrix, x_abs: np.ndarray, scale: float, extra_abs: np.ndarray = None) -> np.ndarray:
    """L1 mass of one fp32 step, every term before cancellation: scale * |A| |x| (+ |extra|); rounding errors of
    the kernel are bounded by a small multiple of it."""
    m = abs(scale) * (A_abs @ x_abs)
    return m + extra_abs if extra_abs is not None else m


# ---------------------------------------------------------------- float64 torch reference (edge list, autograd)
def torch_appnp(src, dst, z, k: int, alpha: float):
    """Plain edge-list APPNP propagation in torch (float64 autograd reference), GCN norms from the edge list."""
    import torch
    n = z.shape[0]
    deg_in = torch.zeros(n, dtype=z.dtype).index_add(0, dst, torch.ones_like(dst, dtype=z.dtype))
    deg_out = torch.zeros(n, dtype=z.dtype).index_add(0, src, torch.ones_like(src, dtype=z.dtype))
    w = (deg_out.clamp(min=1).pow(-0.5)[src] * deg_in.clamp(min=1).pow(-0.5)[dst]).unsqueeze(1)
    h = z
    for _ in range(k):
        h = (1 - alpha) * torch.zeros_like(z).index_add(0, dst, w * h[src]) + alpha * z
    return h

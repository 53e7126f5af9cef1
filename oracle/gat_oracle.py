"""float64 numpy restatement of the GAT layer math (DESIGN.md, "GAT") and of its distributed exchange protocol.

Forward (H heads of width D, z = x W):
    el[i,h] = <z[i,h,:], a_l[h,:]>      er[i,h] = <z[i,h,:], a_r[h,:]>
    e[v,u,h] = LeakyReLU_0.2(el[u,h] + er[v,h])       u in CSR row v
    lse[v,h] = logsumexp_u e[v,u,h]     alpha = exp(e - lse)     out[v,h,:] = sum_u alpha[v,u,h] z[u,h,:]
Backward (g = dL/dout, s[v,h] = <g[v,h,:], out[v,h,:]>):
    t[v,u,h]  = alpha[v,u,h] (<g[v,h,:], z[u,h,:]> - s[v,h]) (1 if el[u,h] + er[v,h] > 0 else 0.2)
    dz[u]     = sum_{u->v} (alpha[v,u] g[v] + t[v,u] a_l) + (sum_{w->u} t[u,w]) a_r
    del[u,h]  = sum_{u->v} t[v,u,h]    der[v,h] = sum_{u->v} t[v,u,h]
    da_l = sum_u del[u] z[u],  da_r = sum_v der[v] z[v]  (inner rows),  dW = x^T dz,  dx = dz W^T
The graphs are symmetric, so the destinations of an inner row u are the entries of its CSR row.

`dist_gat_layer` runs one layer per rank over prepared layouts (manager.layout) with the exchanges simulated exactly:
forward rows z and scalars el, backward rows g and scalars [er | lse | s].  `global_from_layouts` rebuilds the
unpartitioned graph from the same layouts, so the monolithic layer can be compared row by row.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np
import scipy.sparse as sp

SLOPE = 0.2


def leaky(x):
    return np.where(x > 0, x, SLOPE * x)


def scores(z: np.ndarray, a_l: np.ndarray, a_r: np.ndarray, H: int):
    n = z.shape[0]
    zh = z.reshape(n, H, -1)
    return (zh * a_l.reshape(1, H, -1)).sum(-1), (zh * a_r.reshape(1, H, -1)).sum(-1)


def _rows(indptr):
    return np.repeat(np.arange(indptr.size - 1, dtype=np.int64), np.diff(indptr))


def forward(indptr, indices, z_all, el_all, er, H):
    """out [n, F], lse [n, H] of the destination rows 0..n-1 (n = len(indptr) - 1); sources index z_all / el_all."""
    indptr, indices = np.asarray(indptr, np.int64), np.asarray(indices, np.int64)
    n = indptr.size - 1
    F = z_all.shape[1]
    D = F // H
    dst = _rows(indptr)
    e = leaky(el_all[indices] + er[dst])                       # [nnz, H]
    m = np.full((n, H), -np.inf)
    np.maximum.at(m, dst, e)
    ssum = np.zeros((n, H))
    np.add.at(ssum, dst, np.exp(e - m[dst]))
    lse = m + np.log(ssum)
    alpha = np.exp(e - lse[dst])
    out = np.zeros((n, H, D))
    zh = z_all.reshape(-1, H, D)
    for h in range(H):
        A = sp.csr_matrix((alpha[:, h], indices, indptr), shape=(n, z_all.shape[0]))
        out[:, h, :] = A @ zh[:, h, :]
    return out.reshape(n, F), lse


def backward(indptr, indices, g_all, z_all, el_all, er_all, lse_all, s_all, a_l, a_r, H):
    """dz [n, F], del [n, H], der [n, H] of the local rows u = 0..n-1; every per-row array indexes sources (local rows
    first, then halo rows)."""
    indptr, indices = np.asarray(indptr, np.int64), np.asarray(indices, np.int64)
    n = indptr.size - 1
    F = z_all.shape[1]
    D = F // H
    u = _rows(indptr)
    x = indices
    gh, zh = g_all.reshape(-1, H, D), z_all.reshape(-1, H, D)
    # u as a source of destination x
    e1 = el_all[u] + er_all[x]
    a1 = np.exp(leaky(e1) - lse_all[x])
    t1 = a1 * ((gh[x] * zh[u]).sum(-1) - s_all[x]) * np.where(e1 > 0, 1.0, SLOPE)
    # x as a source of destination u
    e2 = el_all[x] + er_all[u]
    a2 = np.exp(leaky(e2) - lse_all[u])
    t2 = a2 * ((gh[u] * zh[x]).sum(-1) - s_all[u]) * np.where(e2 > 0, 1.0, SLOPE)
    dl = np.zeros((n, H))
    dr = np.zeros((n, H))
    np.add.at(dl, u, t1)
    np.add.at(dr, u, t2)
    acc = np.zeros((n, H, D))
    for h in range(H):
        A = sp.csr_matrix((a1[:, h], x, indptr), shape=(n, g_all.shape[0]))
        acc[:, h, :] = A @ gh[:, h, :]
    dz = acc + dl[:, :, None] * a_l.reshape(1, H, D) + dr[:, :, None] * a_r.reshape(1, H, D)
    return dz.reshape(n, F), dl, dr


def layer(indptr, indices, x, W, a_l, a_r, H, g):
    """One monolithic layer on a graph without halo rows: forward and backward for upstream gradient g.
    Returns a dict of every intermediate and gradient."""
    z = x @ W
    el, er = scores(z, a_l, a_r, H)
    out, lse = forward(indptr, indices, z, el, er, H)
    n, F = out.shape
    s = (g.reshape(n, H, -1) * out.reshape(n, H, -1)).sum(-1)
    dz, dl, dr = backward(indptr, indices, g, z, el, er, lse, s, a_l, a_r, H)
    zh = z.reshape(n, H, -1)
    return {"z": z, "el": el, "er": er, "out": out, "lse": lse, "s": s, "dz": dz, "del": dl, "der": dr,
            "da_l": (dl[:, :, None] * zh).sum(0), "da_r": (dr[:, :, None] * zh).sum(0), "dW": x.T @ dz,
            "dx": dz @ W.T}


# ---------------------------------------------------------------- distributed protocol
def exchange(rows: Sequence[np.ndarray], layouts) -> List[np.ndarray]:
    """halo[r][recv_idx[r][p]] = rows[p][p's send rows to r]: what the fp32 exchange delivers."""
    out = []
    for r, L in enumerate(layouts):
        h = np.zeros((L.n_halo, rows[r].shape[1]))
        for p, pos in L.recv_idx.items():
            Lp = layouts[p]
            lo, hi = Lp.send_idx[r]
            h[np.asarray(pos, np.int64)] = rows[p][np.asarray(Lp.total_send_idx[lo:hi], np.int64)]
        out.append(h)
    return out


def dist_gat_layer(layouts, xs: Sequence[np.ndarray], W, a_l, a_r, H, gs: Sequence[np.ndarray]) -> List[Dict]:
    """One GAT layer on every rank, forward then backward, with the exchanges of the protocol: forward z and el,
    backward g and [er | lse | s].  Per rank: out / lse of its inner rows, dz, del, der and its shares of dW, da_l,
    da_r (summing them over ranks gives the global gradient)."""
    zs = [np.asarray(x, np.float64) @ W for x in xs]
    sc = [scores(z, a_l, a_r, H) for z in zs]
    els, ers = [s[0] for s in sc], [s[1] for s in sc]
    z_halo, el_halo = exchange(zs, layouts), exchange(els, layouts)
    res = []
    for r, L in enumerate(layouts):
        out, lse = forward(L.indptr, L.indices, np.concatenate([zs[r], z_halo[r]]), np.concatenate([els[r], el_halo[r]]),
                           ers[r], H)
        n = out.shape[0]
        s = (gs[r].reshape(n, H, -1) * out.reshape(n, H, -1)).sum(-1)
        res.append({"z": zs[r], "out": out, "lse": lse, "s": s, "aux": np.concatenate([ers[r], lse, s], 1)})
    g_halo = exchange(gs, layouts)
    aux_halo = exchange([d["aux"] for d in res], layouts)
    for r, L in enumerate(layouts):
        d = res[r]
        aux_all = np.concatenate([d["aux"], aux_halo[r]])
        dz, dl, dr = backward(L.indptr, L.indices, np.concatenate([gs[r], g_halo[r]]), np.concatenate([zs[r], z_halo[r]]),
                              np.concatenate([els[r], el_halo[r]]), aux_all[:, :H], aux_all[:, H:2 * H],
                              aux_all[:, 2 * H:], a_l, a_r, H)
        zh = zs[r].reshape(zs[r].shape[0], H, -1)
        d.update({"dz": dz, "del": dl, "der": dr, "da_l": (dl[:, :, None] * zh).sum(0),
                  "da_r": (dr[:, :, None] * zh).sum(0), "dW": np.asarray(xs[r], np.float64).T @ dz,
                  "dx": dz @ W.T, "el_halo": el_halo[r], "aux_halo": aux_halo[r]})
    return res


def global_from_layouts(layouts):
    """The unpartitioned graph behind prepared layouts: global id of (rank r, inner row i) = base[r] + i, halo rows
    mapped to their owner's row through recv_idx / send_idx / total_send_idx.  Returns (indptr, indices, base)."""
    W = len(layouts)
    base = np.concatenate([[0], np.cumsum([L.n_inner for L in layouts])]).astype(np.int64)
    rows_ip, rows_ix = [np.zeros(1, np.int64)], []
    off = 0
    for r, L in enumerate(layouts):
        gid = np.empty(L.n_inner + L.n_halo, np.int64)
        gid[:L.n_inner] = base[r] + np.arange(L.n_inner)
        for p, pos in L.recv_idx.items():
            Lp = layouts[p]
            lo, hi = Lp.send_idx[r]
            gid[L.n_inner + np.asarray(pos, np.int64)] = base[p] + np.asarray(Lp.total_send_idx[lo:hi], np.int64)
        ip = np.asarray(L.indptr, np.int64)
        rows_ip.append(ip[1:] + off)
        off += int(ip[-1])
        rows_ix.append(gid[np.asarray(L.indices, np.int64)])
    indptr = np.concatenate(rows_ip)
    indices = np.concatenate(rows_ix) if rows_ix else np.zeros(0, np.int64)
    # sort the columns of every row (scipy keeps the values aligned)
    A = sp.csr_matrix((np.ones(indices.size), indices, indptr), shape=(int(base[W]), int(base[W])))
    A.sort_indices()
    return A.indptr.astype(np.int64), A.indices.astype(np.int64), base


# ---------------------------------------------------------------- float64 torch reference (edge list, autograd)
def torch_gat_layer(src, dst, x, W, a_l, a_r, b, H):
    """Plain edge-list GAT layer in torch (float64 autograd reference): y = out + b."""
    import torch
    z = x @ W
    n = x.shape[0]
    zh = z.view(n, H, -1)
    el = (zh * a_l.view(1, H, -1)).sum(-1)
    er = (zh * a_r.view(1, H, -1)).sum(-1)
    e = torch.nn.functional.leaky_relu(el[src] + er[dst], SLOPE)
    m = torch.full((n, H), -float("inf"), dtype=z.dtype).scatter_reduce(0, dst.view(-1, 1).expand(-1, H), e, "amax")
    p = torch.exp(e - m[dst].detach())
    ssum = torch.zeros((n, H), dtype=z.dtype).index_add(0, dst, p)
    alpha = p / ssum[dst]
    out = torch.zeros_like(zh).index_add(0, dst, alpha.unsqueeze(-1) * zh[src])
    return out.reshape(n, -1) + b


def masses(indptr, indices, g_all, z_all, el_all, er_all, lse_all, s_all, a_l, a_r, H):
    """Per-row L1 masses that bound the rounding error of an fp32 evaluation, every term taken before cancellation:
    forward sum_u alpha |z[u]| [n, F]; t-masses alpha (1 + |e| + |lse|) (sum_d |g z| + |s|) summed into m1 (del) and
    m2 (der) [n, H] (the exponent's magnitude bounds the relative error of alpha); backward
    sum_v alpha (1 + |e| + |lse|) |g[v]| + |a_l| m1 + |a_r| m2 [n, F]."""
    indptr, indices = np.asarray(indptr, np.int64), np.asarray(indices, np.int64)
    n = indptr.size - 1
    F = z_all.shape[1]
    D = F // H
    u, x = _rows(indptr), indices
    gh, zh = np.abs(g_all).reshape(-1, H, D), np.abs(z_all).reshape(-1, H, D)
    e0 = leaky(el_all[x] + er_all[u])
    a0 = np.exp(e0 - lse_all[u])                                     # alpha[u, x]
    e1 = leaky(el_all[u] + er_all[x])
    a1 = np.exp(e1 - lse_all[x])                                     # alpha[x, u]
    w1 = a1 * (1 + np.abs(e1) + np.abs(lse_all[x]))
    w0 = a0 * (1 + np.abs(e0) + np.abs(lse_all[u]))
    t1 = w1 * ((gh[x] * zh[u]).sum(-1) + np.abs(s_all[x]))
    t2 = w0 * ((gh[u] * zh[x]).sum(-1) + np.abs(s_all[u]))
    fm, bm = np.zeros((n, H, D)), np.zeros((n, H, D))
    for h in range(H):
        fm[:, h, :] = sp.csr_matrix((a0[:, h], x, indptr), shape=(n, z_all.shape[0])) @ zh[:, h, :]
        bm[:, h, :] = sp.csr_matrix((w1[:, h], x, indptr), shape=(n, g_all.shape[0])) @ gh[:, h, :]
    m1, m2 = np.zeros((n, H)), np.zeros((n, H))
    np.add.at(m1, u, t1)
    np.add.at(m2, u, t2)
    bm += m1[:, :, None] * np.abs(a_l).reshape(1, H, D) + m2[:, :, None] * np.abs(a_r).reshape(1, H, D)
    return fm.reshape(n, F), bm.reshape(n, F), m1, m2

"""float64 numpy restatement of the GATv2 layer math (DESIGN.md, "GATv2") and of its distributed protocol.

Forward (H heads of width D, zs = x W_s + b_s, zd = x W_d + b_d):
    s[v,u] = zs[u] + zd[v]       e[v,u,h] = sum_{c in head h} a[h,c] LeakyReLU_0.2(s[v,u,h,c])      u in CSR row v
    lse[v,h] = logsumexp_u e[v,u,h]     alpha = exp(e - lse)     out[v,h,:] = sum_u alpha[v,u,h] zs[u,h,:]
Backward (g = dL/dout, S[v,h] = <g[v,h,:], out[v,h,:]>), for every edge u -> v:
    t[v,u,h] = alpha[v,u,h] (<g[v,h,:], zs[u,h,:]> - S[v,h])
    dzs[u] += alpha[v,u] g[v] + t[v,u] a . LeakyReLU'(s[v,u])        (the source side)
    dzd[v] += t[v,u] a . LeakyReLU'(s[v,u])                           (the destination side)
    da     += t[v,u] LeakyReLU(s[v,u])                                (da_rows[v]: the share of destination v)

`backward` splits the source side as the kernels do: inner sources (dzs of the local rows) and halo sources (the
rows a rank pushes back to their owners); `fold` adds the pushed rows.  `dist_gatv2_layer` runs one layer per rank
over prepared layouts with the forward exchange of zs and the push simulated exactly.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np

from .gat_oracle import SLOPE, _rows, exchange, global_from_layouts, leaky  # noqa: F401


def _edges(indptr, indices, zs_all, zd, attn, H):
    indptr, indices = np.asarray(indptr, np.int64), np.asarray(indices, np.int64)
    v, u = _rows(indptr), indices
    D = zs_all.shape[1] // H
    s = zs_all.reshape(-1, H, D)[u] + zd.reshape(-1, H, D)[v]                 # [E, H, D]
    e = (attn.reshape(1, H, D) * leaky(s)).sum(-1)                             # [E, H]
    return v, u, s, e


def forward(indptr, indices, zs_all, zd, attn, H):
    """out [n, F], lse [n, H] of the destination rows 0..n-1 (n = len(indptr) - 1); sources index zs_all."""
    n = len(indptr) - 1
    F = zs_all.shape[1]
    v, u, s, e = _edges(indptr, indices, zs_all, zd, attn, H)
    m = np.full((n, H), -np.inf)
    np.maximum.at(m, v, e)
    ssum = np.zeros((n, H))
    np.add.at(ssum, v, np.exp(e - m[v]))
    lse = m + np.log(ssum)
    alpha = np.exp(e - lse[v])
    out = np.zeros((n, H, F // H))
    np.add.at(out, v, alpha[:, :, None] * zs_all.reshape(-1, H, F // H)[u])
    return out.reshape(n, F), lse


def backward(indptr, indices, zs_all, zd, g, lse, S, attn, H):
    """Backward of the destination rows 0..n-1 whose sources index zs_all (n local rows first, then halo rows).
    Returns dzs [n, F] (the source side of the edges with a local source, nothing pushed), dzs_halo [rows of
    zs_all - n, F] (the source side of the edges with a halo source), dzd [n, F] and da_rows [n, F]."""
    n = len(indptr) - 1
    F = zs_all.shape[1]
    D = F // H
    v, u, s, e = _edges(indptr, indices, zs_all, zd, attn, H)
    alpha = np.exp(e - lse[v])
    gh, zh = g.reshape(-1, H, D), zs_all.reshape(-1, H, D)
    t = alpha * ((gh[v] * zh[u]).sum(-1) - S[v])
    ta = t[:, :, None] * attn.reshape(1, H, D) * np.where(s > 0, 1.0, SLOPE)
    src = alpha[:, :, None] * gh[v] + ta
    dzs_all = np.zeros((zs_all.shape[0], H, D))
    np.add.at(dzs_all, u, src)
    dzd, da = np.zeros((n, H, D)), np.zeros((n, H, D))
    np.add.at(dzd, v, ta)
    np.add.at(da, v, t[:, :, None] * leaky(s))
    dzs_all = dzs_all.reshape(-1, F)
    return dzs_all[:n], dzs_all[n:], dzd.reshape(n, F), da.reshape(n, F)


def fold(dzs, push, fold_indptr, fold_pos):
    """dzs[u] + the pushed rows push[fold_pos[fold_indptr[u] .. fold_indptr[u+1])]."""
    out = np.array(dzs, np.float64, copy=True)
    fold_indptr = np.asarray(fold_indptr, np.int64)
    rows = _rows(fold_indptr)
    np.add.at(out, rows, np.asarray(push, np.float64)[np.asarray(fold_pos, np.int64)])
    return out


def layer(indptr, indices, x, Ws, bs, Wd, bd, attn, H, g):
    """One monolithic layer on a graph without halo rows: forward and backward for upstream gradient g."""
    zs, zd = x @ Ws + bs, x @ Wd + bd
    out, lse = forward(indptr, indices, zs, zd, attn, H)
    n, F = out.shape
    S = (g.reshape(n, H, -1) * out.reshape(n, H, -1)).sum(-1)
    dzs, _, dzd, da_rows = backward(indptr, indices, zs, zd, g, lse, S, attn, H)
    return {"zs": zs, "zd": zd, "out": out, "lse": lse, "S": S, "dzs": dzs, "dzd": dzd,
            "da": da_rows.sum(0).reshape(H, -1), "dWs": x.T @ dzs, "dWd": x.T @ dzd, "dbs": dzs.sum(0),
            "dbd": dzd.sum(0), "dx": dzs @ Ws.T + dzd @ Wd.T}


# ---------------------------------------------------------------- distributed protocol
def push(rows: Sequence[np.ndarray], layouts) -> List[np.ndarray]:
    """region[r][i] = the row that the holder p of r's send position i (lo <= i < hi for (lo, hi) = send_idx[p])
    pushes back: rows[p][recv_idx_p[r][i - lo]].  What the push delivers to every owner."""
    out = []
    for r, L in enumerate(layouts):
        reg = np.zeros((len(L.total_send_idx), rows[r].shape[1]))
        for p, (lo, hi) in L.send_idx.items():
            reg[lo:hi] = rows[p][np.asarray(layouts[p].recv_idx[r], np.int64)]
        out.append(reg)
    return out


def fold_table(L):
    """Fold table of a layout, built directly: for each inner row, its positions in total_send_idx, in send-peer
    order."""
    per_row: List[List[int]] = [[] for _ in range(L.n_inner)]
    for p, (lo, hi) in L.send_idx.items():
        for i in range(lo, hi):
            per_row[int(L.total_send_idx[i])].append(i)
    indptr = np.concatenate([[0], np.cumsum([len(x) for x in per_row])]).astype(np.int64)
    pos = np.asarray([i for x in per_row for i in x], np.int64)
    return indptr, pos


def dist_gatv2_layer(layouts, xs: Sequence[np.ndarray], Ws, bs, Wd, bd, attn, H, gs: Sequence[np.ndarray],
                     zs_halo: Optional[Sequence[np.ndarray]] = None) -> List[Dict]:
    """One GATv2 layer on every rank, forward then backward, with the exchanges of the protocol: forward zs, then
    the push of every halo row's source-side gradient to its owner.  `zs_halo` replaces the exchanged halo rows
    (the dequantised rows a rank actually received).  Per rank: out / lse of its inner rows, dzs (pushed rows
    folded in), dzd, da_rows, the pushed rows it sent (dzs_halo) and its shares of dW_s, dW_d, db_s, db_d and da
    (summing them over ranks gives the global gradient)."""
    xs = [np.asarray(x, np.float64) for x in xs]
    zss = [x @ Ws + bs for x in xs]
    zds = [x @ Wd + bd for x in xs]
    halo = exchange(zss, layouts) if zs_halo is None else [np.asarray(h, np.float64) for h in zs_halo]
    res = []
    for r, L in enumerate(layouts):
        zs_all = np.concatenate([zss[r], halo[r]])
        out, lse = forward(L.indptr, L.indices, zs_all, zds[r], attn, H)
        n = out.shape[0]
        S = (gs[r].reshape(n, H, -1) * out.reshape(n, H, -1)).sum(-1)
        dzs, dzs_halo, dzd, da_rows = backward(L.indptr, L.indices, zs_all, zds[r], gs[r], lse, S, attn, H)
        res.append({"zs": zss[r], "zd": zds[r], "zs_halo": halo[r], "out": out, "lse": lse, "S": S, "dzs_inner": dzs,
                    "dzs_halo": dzs_halo, "dzd": dzd, "da_rows": da_rows})
    regions = push([d["dzs_halo"] for d in res], layouts)
    for r, L in enumerate(layouts):
        d = res[r]
        fi, fp = fold_table(L)
        dzs = fold(d["dzs_inner"], regions[r], fi, fp)
        x = xs[r]
        d.update({"push": regions[r], "dzs": dzs, "dWs": x.T @ dzs, "dWd": x.T @ d["dzd"], "dbs": dzs.sum(0),
                  "dbd": d["dzd"].sum(0), "da": d["da_rows"].sum(0).reshape(H, -1), "dx": dzs @ Ws.T + d["dzd"] @ Wd.T})
    return res


# ---------------------------------------------------------------- float64 torch reference (edge list, autograd)
def torch_gatv2_layer(src, dst, x, Ws, bs, Wd, bd, attn, H):
    """Plain edge-list GATv2 layer in torch (float64 autograd reference)."""
    import torch
    n = x.shape[0]
    zs, zd = (x @ Ws + bs).view(n, H, -1), (x @ Wd + bd).view(n, H, -1)
    e = (attn.view(1, H, -1) * torch.nn.functional.leaky_relu(zs[src] + zd[dst], SLOPE)).sum(-1)
    m = torch.full((n, H), -float("inf"), dtype=x.dtype).scatter_reduce(0, dst.view(-1, 1).expand(-1, H), e, "amax")
    p = torch.exp(e - m[dst].detach())
    ssum = torch.zeros((n, H), dtype=x.dtype).index_add(0, dst, p)
    alpha = p / ssum[dst]
    out = torch.zeros_like(zs).index_add(0, dst, alpha.unsqueeze(-1) * zs[src])
    return out.reshape(n, -1)


def masses(indptr, indices, zs_all, zd, g, lse, S, attn, H):
    """Per-row L1 masses that bound the rounding error of an fp32 evaluation, every term taken before cancellation
    (each alpha weighted by 1 + the magnitude of its exponent): forward sum_u alpha |zs[u]| [n, F]; backward the
    absolute source-side terms of dzs (inner sources [n, F], halo sources [rows - n, F]), of dzd [n, F] and of
    da_rows [n, F]."""
    n = len(indptr) - 1
    F = zs_all.shape[1]
    D = F // H
    v, u, s, e = _edges(indptr, indices, zs_all, zd, attn, H)
    alpha = np.exp(e - lse[v])
    ex = 1 + (np.abs(attn).reshape(1, H, D) * np.abs(s)).sum(-1) + np.abs(lse[v])
    w = alpha * ex
    gh, zh = np.abs(g).reshape(-1, H, D), np.abs(zs_all).reshape(-1, H, D)
    tm = w * ((gh[v] * zh[u]).sum(-1) + np.abs(S[v]))
    ta = tm[:, :, None] * np.abs(attn).reshape(1, H, D)
    fm = np.zeros((n, H, D))
    np.add.at(fm, v, alpha[:, :, None] * zh[u])
    sm = np.zeros((zs_all.shape[0], H, D))
    np.add.at(sm, u, w[:, :, None] * gh[v] + ta)
    dm, am = np.zeros((n, H, D)), np.zeros((n, H, D))
    np.add.at(dm, v, ta)
    np.add.at(am, v, tm[:, :, None] * np.abs(s))
    sm = sm.reshape(-1, F)
    return fm.reshape(n, F), sm[:n], sm[n:], dm.reshape(n, F), am.reshape(n, F)

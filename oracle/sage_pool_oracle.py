"""float64 numpy restatement of the GraphSAGE max-pool layer (DESIGN.md, "GraphSAGE max-pool") and of its distributed
exchange protocol.

Layer (DGL SAGEConv, aggregator_type='pool'), x of width F:
    p        = relu(x W_pool^T + b_pool)
    m[v,c]   = max_{u in N_in(v)} p[u,c]        arg[v,c] = the first u in CSR order attaining it
    rst      = x W_self^T + m W_neigh^T + b
Backward (g = dL/drst, gm = g W_neigh):
    dp[u,c]  = sum_{v : u in N_in(v)} gm[v,c] [arg[v,c] = u]      dpre = dp (p > 0)
    dW_pool = dpre^T x,  db_pool = sum dpre,  dW_self = g^T x,  dW_neigh = g^T m,  db = sum g,
    dx = g W_self + dpre W_pool
arg is stored as (source id - n_split), the encoding the rows travel in: a halo position (>= 0) for halo sources, a
negative value for local ones, NO_ARG for a row without sources (whose m is 0).  The graphs are symmetric, so the
destinations of an inner row u are the entries of its CSR row, and want[e] is row u in the encoding of the owner of
the entry's column.

`dist_pool_layer` runs one layer per rank over prepared layouts (manager.layout) with the exchanges simulated exactly:
forward rows p, backward rows gm and the arg rows; `pool_want_bruteforce` builds each rank's match table from global
ids.  Received halo rows can be given instead of the simulated fp32 exchange (quantised modes).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import numpy as np

from .gat_oracle import exchange, global_from_layouts  # noqa: F401  (global_from_layouts re-exported for tests)

NO_ARG = -2 ** 31
COLS = 32          # column block: bounds the [nnz, COLS] temporaries of hub rows


def _rows(indptr):
    return np.repeat(np.arange(indptr.size - 1, dtype=np.int64), np.diff(indptr))


def forward(indptr, indices, x_all, n_split):
    """m [n, F] (float64) and arg [n, F] (int64, encoded) of the destination rows 0..n-1 (n = len(indptr) - 1)."""
    indptr, indices = np.asarray(indptr, np.int64), np.asarray(indices, np.int64)
    n, F = indptr.size - 1, x_all.shape[1]
    m = np.zeros((n, F))
    arg = np.full((n, F), NO_ARG, np.int64)
    rows = np.nonzero(np.diff(indptr) > 0)[0]
    if rows.size == 0:
        return m, arg
    starts = indptr[rows]
    pos = np.arange(indices.size, dtype=np.int64)[:, None]
    for c0 in range(0, F, COLS):
        v = np.asarray(x_all[indices, c0:c0 + COLS], np.float64)
        mx = np.maximum.reduceat(v, starts, axis=0)
        dst = _rows(indptr)
        first = np.where(v == mx[np.searchsorted(rows, dst)], pos, indices.size)    # first maximum in CSR order
        e = np.minimum.reduceat(first, starts, axis=0)
        m[rows, c0:c0 + COLS] = mx
        arg[rows, c0:c0 + COLS] = indices[e] - n_split
    return m, arg


def backward(indptr, indices, want, g_all, arg_all):
    """dp [n, F] of the local rows u = 0..n-1: sum over the entries e = (u, x) of g_all[x] where arg_all[x] == want[e].
    g_all / arg_all index sources (local rows first, then halo rows)."""
    indptr, indices = np.asarray(indptr, np.int64), np.asarray(indices, np.int64)
    want = np.asarray(want, np.int64)
    n, F = indptr.size - 1, g_all.shape[1]
    dp = np.zeros((n, F))
    rows = np.nonzero(np.diff(indptr) > 0)[0]
    if rows.size == 0:
        return dp
    for c0 in range(0, F, COLS):
        hit = np.asarray(arg_all[indices, c0:c0 + COLS], np.int64) == want[:, None]
        v = np.where(hit, np.asarray(g_all[indices, c0:c0 + COLS], np.float64), 0.0)
        dp[rows, c0:c0 + COLS] = np.add.reduceat(v, indptr[rows], axis=0)
    return dp


def _finish(x, p, m, arg, g, dp, Wp, Ws, Wn, b):
    dpre = dp * (p > 0)
    return {"p": p, "m": m, "arg": arg, "rst": x @ Ws.T + m @ Wn.T + b, "gm": g @ Wn, "dp": dp,
            "dW_pool": dpre.T @ x, "db_pool": dpre.sum(0), "dW_self": g.T @ x, "dW_neigh": g.T @ m, "db": g.sum(0),
            "dx": g @ Ws + dpre @ Wp}


def layer(indptr, indices, x, Wp, bp, Ws, Wn, b, g):
    """One monolithic layer on a graph without halo rows: forward and backward for upstream gradient g.
    Returns a dict of every intermediate and gradient."""
    x = np.asarray(x, np.float64)
    n = x.shape[0]
    p = np.maximum(x @ Wp.T + bp, 0.0)
    m, arg = forward(indptr, indices, p, n)
    want = _rows(np.asarray(indptr, np.int64)) - n
    dp = backward(indptr, indices, want, g @ Wn, arg)
    return _finish(x, p, m, arg, g, dp, Wp, Ws, Wn, b)


# ---------------------------------------------------------------- distributed protocol
def _gids(layouts) -> List[np.ndarray]:
    """Global id of every (inner + halo) row of every rank: base[r] + i for inner rows, the owner's row for halo rows."""
    base = np.concatenate([[0], np.cumsum([L.n_inner for L in layouts])]).astype(np.int64)
    out = []
    for r, L in enumerate(layouts):
        gid = np.empty(L.n_inner + L.n_halo, np.int64)
        gid[:L.n_inner] = base[r] + np.arange(L.n_inner)
        for p, pos in L.recv_idx.items():
            Lp = layouts[p]
            lo, hi = Lp.send_idx[r]
            gid[L.n_inner + np.asarray(pos, np.int64)] = base[p] + np.asarray(Lp.total_send_idx[lo:hi], np.int64)
        out.append(gid)
    return out


def pool_want_bruteforce(layouts, r: int) -> np.ndarray:
    """want[e] for every CSR entry e = (u, x) of rank r, looked up entry by entry in global ids: u - n_inner for a
    local x; for a halo x owned by P, the position j with P's halo row n_inner_P + j == u."""
    gids = _gids(layouts)
    base = np.concatenate([[0], np.cumsum([L.n_inner for L in layouts])]).astype(np.int64)
    halo_pos = [{int(g): j for j, g in enumerate(gids[p][Lp.n_inner:])} for p, Lp in enumerate(layouts)]
    L = layouts[r]
    indptr, indices = np.asarray(L.indptr, np.int64), np.asarray(L.indices, np.int64)
    want = np.empty(indices.size, np.int64)
    for u in range(L.n_inner):
        for e in range(indptr[u], indptr[u + 1]):
            x = int(indices[e])
            if x < L.n_inner:
                want[e] = u - L.n_inner
            else:
                owner = int(np.searchsorted(base, gids[r][x], side="right") - 1)
                want[e] = halo_pos[owner][int(base[r] + u)]
    return want


def dist_pool_layer(layouts, xs: Sequence[np.ndarray], Wp, bp, Ws, Wn, b, gs: Sequence[np.ndarray],
                    p_halos: Optional[Sequence[np.ndarray]] = None,
                    g_halos: Optional[Sequence[np.ndarray]] = None) -> List[Dict]:
    """One max-pool layer on every rank, forward then backward, with the exchanges of the protocol: forward p,
    backward gm = g W_neigh and the encoded arg rows.  p_halos / g_halos replace the simulated fp32 exchange of p / gm
    (the rows a quantised exchange delivered).  Per rank: p, m, arg, rst, dp of its inner rows, the received
    arg_halo, want, and its shares of every weight gradient (summing them over ranks gives the global gradient)."""
    xs = [np.asarray(x, np.float64) for x in xs]
    ps = [np.maximum(x @ Wp.T + bp, 0.0) for x in xs]
    p_halo = exchange(ps, layouts) if p_halos is None else [np.asarray(h, np.float64) for h in p_halos]
    fw = [forward(L.indptr, L.indices, np.concatenate([ps[r], p_halo[r]]), L.n_inner) for r, L in enumerate(layouts)]
    gms = [np.asarray(g, np.float64) @ Wn for g in gs]
    g_halo = exchange(gms, layouts) if g_halos is None else [np.asarray(h, np.float64) for h in g_halos]
    arg_halo = [h.astype(np.int64) for h in exchange([a for _, a in fw], layouts)]
    res = []
    for r, L in enumerate(layouts):
        m, arg = fw[r]
        want = pool_want_bruteforce(layouts, r)
        dp = backward(L.indptr, L.indices, want, np.concatenate([gms[r], g_halo[r]]), np.concatenate([arg, arg_halo[r]]))
        d = _finish(xs[r], ps[r], m, arg, np.asarray(gs[r], np.float64), dp, Wp, Ws, Wn, b)
        d.update({"arg_halo": arg_halo[r], "want": want})
        res.append(d)
    return res


# ---------------------------------------------------------------- float64 torch reference (edge list, autograd)
def torch_pool_layer(src, dst, x, Wp, bp, Ws, Wn, b):
    """Plain edge-list max-pool SAGE layer in torch (float64 autograd reference).  Ties split the gradient evenly in
    torch's amax, so compare on inputs whose only ties are at 0 (masked by the ReLU)."""
    import torch
    n = x.shape[0]
    p = torch.relu(x @ Wp.T + bp)
    idx = dst.view(-1, 1).expand(-1, p.shape[1])
    m = torch.zeros((n, p.shape[1]), dtype=p.dtype).scatter_reduce(0, idx, p[src], "amax", include_self=False)
    return x @ Ws.T + m @ Wn.T + b

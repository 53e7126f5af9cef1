"""GraphSAGE max-pool aggregation (host mirror of csrc/sage_pool.cu).

`forward` computes the column-wise neighbourhood max m and its argmax of a destination row range, `backward` the
argmax-routed gradient dp of local rows, and `pool_want` the per-entry match table the backward pass compares the
received arg rows with (DESIGN.md, "GraphSAGE max-pool").  Like spmm(), the source rows come from the local matrix
(ids < n_inner) and the received halo matrix without concatenation, and `part='local'` / `part='halo'` split each row
into its local-source and halo-source segments, the halo part continuing from what the local part wrote.  fp32 CUDA
tensors only; there is no torch fall-back: an unsupported shape is an error from the library.

arg entries are (source id - n_inner) in the numbering of the rank that computed them: a halo position (>= 0) for a
halo source, a negative value for a local one, NO_ARG for a row without sources.
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib
from .manager.graph import part_segments

NO_ARG = -2 ** 31
LAUNCHES = {"sage_pool_fwd_kernel": 0, "sage_pool_bwd_kernel": 0}


def _rows(t: Optional[Tensor], F: int, dtype=torch.float32) -> Optional[Tensor]:
    if t is None or t.shape[0] == 0:
        return None
    assert t.dtype == dtype and t.dim() == 2 and t.shape[1] == F and t.stride(1) == 1, (t.dtype, t.shape, t.stride())
    return t


def forward(graph, x: Tensor, x_halo: Optional[Tensor], row_begin: int = 0, row_end: Optional[int] = None,
            out: Optional[Tensor] = None, arg: Optional[Tensor] = None, part: Optional[str] = None,
            stream=None) -> Tuple[Tensor, Tensor]:
    """Rows [row_begin, row_end) of m = column-wise max of x over each CSR row, and arg (int32, encoded as above).
    `graph` is a LocalGraph (indptr, indices, halo_split, n_inner); `out` / `arg` are written at row - row_begin."""
    row_end = graph.n_inner if row_end is None else int(row_end)
    F = int(x.shape[1])
    assert x.dtype == torch.float32 and x.stride(1) == 1
    x_halo = _rows(x_halo, F)
    n = row_end - row_begin
    if part == "halo":
        assert out is not None and arg is not None, "the halo part continues from the output of the local part"
    if out is None:
        out = torch.empty((n, F), dtype=torch.float32, device=x.device)
    if arg is None:
        arg = torch.empty((n, F), dtype=torch.int32, device=x.device)
    assert out.stride(1) == 1 and arg.stride(1) == 1 and arg.dtype == torch.int32
    seg_start, seg_end, acc = part_segments(graph, part)
    rc = _lib.load().adaqp_sage_pool_fwd_f32(
        graph.indptr.data_ptr(), seg_start, seg_end, graph.indices.data_ptr(), graph.n_inner, x.data_ptr(),
        x.stride(0), x_halo.data_ptr() if x_halo is not None else None, x_halo.stride(0) if x_halo is not None else 0,
        F, int(row_begin), row_end, acc, out.data_ptr(), out.stride(0), arg.data_ptr(), arg.stride(0),
        _lib.stream_ptr(stream))
    _lib.check(rc, "adaqp_sage_pool_fwd_f32")
    LAUNCHES["sage_pool_fwd_kernel"] += 1
    return out, arg


def backward(graph, want: Tensor, g: Tensor, g_halo: Optional[Tensor], arg: Tensor, arg_halo: Optional[Tensor],
             row_begin: int = 0, row_end: Optional[int] = None, dp: Optional[Tensor] = None,
             part: Optional[str] = None, stream=None) -> Tensor:
    """dp of the local rows [row_begin, row_end) (written at row - row_begin): the gradient g[x] of every
    destination x of row u, routed to u in the columns where arg[x] == want[e]."""
    row_end = graph.n_inner if row_end is None else int(row_end)
    F = int(g.shape[1])
    g_halo, arg_halo = _rows(g_halo, F), _rows(arg_halo, F, torch.int32)
    if g_halo is None or arg_halo is None:
        g_halo = arg_halo = None
    assert g.dtype == torch.float32 and g.stride(1) == 1 and arg.dtype == torch.int32 and arg.stride(1) == 1
    assert want.dtype == torch.int32 and want.numel() == graph.nnz
    if part == "halo":
        assert dp is not None, "the halo part continues from the output of the local part"
    if dp is None:
        dp = torch.empty((row_end - row_begin, F), dtype=torch.float32, device=g.device)
    assert dp.stride(1) == 1
    seg_start, seg_end, acc = part_segments(graph, part)
    rc = _lib.load().adaqp_sage_pool_bwd_f32(
        graph.indptr.data_ptr(), seg_start, seg_end, graph.indices.data_ptr(), want.data_ptr(), graph.n_inner,
        g.data_ptr(), g.stride(0), g_halo.data_ptr() if g_halo is not None else None,
        g_halo.stride(0) if g_halo is not None else 0, arg.data_ptr(), arg.stride(0),
        arg_halo.data_ptr() if arg_halo is not None else None, arg_halo.stride(0) if arg_halo is not None else 0, F,
        int(row_begin), row_end, acc, dp.data_ptr(), dp.stride(0), _lib.stream_ptr(stream))
    _lib.check(rc, "adaqp_sage_pool_bwd_f32")
    LAUNCHES["sage_pool_bwd_kernel"] += 1
    return dp


def pool_want(indptr: np.ndarray, indices: np.ndarray, n_inner: int, recv_idx: Dict[int, np.ndarray],
              send_idx: Dict[int, Tuple[int, int]], total_send_idx: np.ndarray,
              peer_recv_idx: Dict[int, np.ndarray]) -> np.ndarray:
    """int32[nnz] aligned with `indices`: for entry e = (u, x) of row u, the arg value x's owner stores when u
    attains the max of x -- u - n_inner when x is local; u's position in the halo block of x's owner P otherwise.
    recv_idx[P] = my halo positions of the rows P sends me; peer_recv_idx[P] = P's recv_idx[me], aligned with my
    send rows total_send_idx[send_idx[P]]."""
    indptr = np.asarray(indptr, np.int64)
    indices = np.asarray(indices, np.int64)
    rows = np.repeat(np.arange(indptr.size - 1, dtype=np.int64), np.diff(indptr))
    want = np.empty(indices.size, np.int64)
    local = indices < n_inner
    want[local] = rows[local] - n_inner
    halo = np.nonzero(~local)[0]
    if halo.size:
        n_halo = int(indices[halo].max()) - n_inner + 1
        owner = np.full(n_halo, -1, np.int64)
        for p, pos in recv_idx.items():
            owner[np.asarray(pos, np.int64)] = p
        own = owner[indices[halo] - n_inner]
        if (own < 0).any():
            raise ValueError("a halo column is not received from any peer")
        for p in np.unique(own):
            lo, hi = send_idx[int(p)]
            pos_at = np.full(n_inner, -1, np.int64)
            pos_at[np.asarray(total_send_idx[lo:hi], np.int64)] = np.asarray(peer_recv_idx[int(p)], np.int64)
            sel = halo[own == p]
            want[sel] = pos_at[rows[sel]]
        if (want[halo] < 0).any():
            raise ValueError("an inner row adjacent to a halo row is not sent to its owner: the graph is not symmetric")
    return want.astype(np.int32)

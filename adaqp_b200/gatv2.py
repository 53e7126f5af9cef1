"""GATv2 attention aggregation (host mirror of csrc/gatv2.cu).

`forward(graph, zs, zs_halo, zd, attn, H)` computes the softmax-weighted aggregation of a destination row range (out
and the per-head log-sum-exp), `backward_halo` the source-side gradient of every received halo row (the rows a
holder pushes back to their owners), and `backward_inner` dzs, dzd and the per-row shares of da of the inner rows,
with the pushed rows folded into dzs (DESIGN.md, "GATv2").  `halo_table` and `fold_table` are the two set-up tables
of the backward pass.  Like spmm(), the source rows come from the local matrix (ids < n_inner) and the received halo
matrix without concatenation.  fp32 CUDA tensors only; there is no torch fall-back: an unsupported shape is an
error from the library.
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor

from . import _lib

LAUNCHES = {"gatv2_fwd_kernel": 0, "gatv2_bwd_inner_kernel": 0, "gatv2_bwd_halo_kernel": 0}


def _ptr(t: Optional[Tensor]):
    return t.data_ptr() if t is not None else None


def _rows(t: Optional[Tensor], F: int) -> Optional[Tensor]:
    if t is None or t.shape[0] == 0:
        return None
    assert t.dtype == torch.float32 and t.dim() == 2 and t.shape[1] == F and t.stride(1) == 1, (t.shape, t.stride())
    return t


def halo_table(indptr: np.ndarray, indices: np.ndarray, n_inner: int, num_remote: int) -> Tuple[np.ndarray, np.ndarray]:
    """The halo-transposed CSR: for halo row h, its inner destinations (the inner rows whose CSR row holds
    n_inner + h), ascending.  Returns (halo_indptr int64 [num_remote + 1], halo_dst int32)."""
    indptr, indices = np.asarray(indptr, np.int64), np.asarray(indices, np.int64)
    dst = np.repeat(np.arange(n_inner, dtype=np.int64), np.diff(indptr[:n_inner + 1]))
    src = indices[:indptr[n_inner]]
    sel = src >= n_inner
    h, v = src[sel] - n_inner, dst[sel]
    order = np.argsort(h, kind="stable")                 # v ascending inside each h: CSR rows are visited in order
    counts = np.bincount(h, minlength=num_remote)
    return np.concatenate([[0], np.cumsum(counts)]).astype(np.int64), v[order].astype(np.int32)


def fold_table(n_inner: int, send_peers: Sequence[int], send_idx: Dict[int, Tuple[int, int]],
               total_send_idx: np.ndarray) -> Tuple[np.ndarray, np.ndarray]:
    """For each inner row, its positions in total_send_idx (the rows of the push region), in send-peer order.
    Returns (fold_indptr int64 [n_inner + 1], fold_pos int32)."""
    total_send_idx = np.asarray(total_send_idx, np.int64)
    pos = np.concatenate([np.arange(*send_idx[p], dtype=np.int64) for p in send_peers] or [np.zeros(0, np.int64)])
    rows = total_send_idx[pos]
    order = np.argsort(rows, kind="stable")
    counts = np.bincount(rows, minlength=n_inner)
    return np.concatenate([[0], np.cumsum(counts)]).astype(np.int64), pos[order].astype(np.int32)


def forward(graph, zs: Tensor, zs_halo: Optional[Tensor], zd: Tensor, attn: Tensor, heads: int, row_begin: int = 0,
            row_end: Optional[int] = None, out: Optional[Tensor] = None, lse: Optional[Tensor] = None,
            stream=None) -> Tuple[Tensor, Tensor]:
    """Rows [row_begin, row_end) of out = softmax-weighted sum of zs over each CSR row, and lse [rows, H].
    `graph` is a LocalGraph (indptr, indices, n_inner); `out` / `lse` are written at row - row_begin."""
    row_end = graph.n_inner if row_end is None else int(row_end)
    F = int(zs.shape[1])
    zs_halo = _rows(zs_halo, F)
    n = row_end - row_begin
    if out is None:
        out = torch.empty((n, F), dtype=torch.float32, device=zs.device)
    if lse is None:
        lse = torch.empty((n, heads), dtype=torch.float32, device=zs.device)
    attn = attn.contiguous()
    assert zs.stride(1) == 1 and zd.stride(1) == 1 and out.stride(1) == 1 and lse.is_contiguous()
    rc = _lib.load().adaqp_gatv2_fwd_f32(
        graph.indptr.data_ptr(), graph.indices.data_ptr(), graph.n_inner, zs.data_ptr(), zs.stride(0), _ptr(zs_halo),
        zs_halo.stride(0) if zs_halo is not None else 0, zd.data_ptr(), zd.stride(0), attn.data_ptr(), heads, F,
        int(row_begin), row_end, out.data_ptr(), out.stride(0), lse.data_ptr(), _lib.stream_ptr(stream))
    _lib.check(rc, "adaqp_gatv2_fwd_f32")
    LAUNCHES["gatv2_fwd_kernel"] += 1
    return out, lse


def backward_halo(halo_indptr: Tensor, halo_dst: Tensor, zs_halo: Tensor, zd: Tensor, g: Tensor, lse: Tensor,
                  S: Tensor, attn: Tensor, heads: int, row_begin: int = 0, row_end: Optional[int] = None,
                  out: Optional[Tensor] = None, stream=None) -> Tensor:
    """Rows [row_begin, row_end) of dzs_halo[h] = sum over the inner destinations v of halo row h of
    alpha[v,h] g[v] + t[v,h] a . LeakyReLU'(zs_halo[h] + zd[v]); lse / S are [n_inner, H]."""
    F = int(zd.shape[1])
    row_end = int(zs_halo.shape[0]) if row_end is None else int(row_end)
    n = row_end - row_begin
    if out is None:
        out = torch.empty((n, F), dtype=torch.float32, device=zd.device)
    if n == 0:
        return out
    attn = attn.contiguous()
    assert zs_halo.stride(1) == 1 and zd.stride(1) == 1 and g.stride(1) == 1 and out.stride(1) == 1
    assert lse.is_contiguous() and S.is_contiguous()
    rc = _lib.load().adaqp_gatv2_bwd_halo_f32(
        halo_indptr.data_ptr(), halo_dst.data_ptr(), zs_halo.data_ptr(), zs_halo.stride(0), zd.data_ptr(),
        zd.stride(0), g.data_ptr(), g.stride(0), lse.data_ptr(), S.data_ptr(), attn.data_ptr(), heads, F,
        int(row_begin), row_end, out.data_ptr(), out.stride(0), _lib.stream_ptr(stream))
    _lib.check(rc, "adaqp_gatv2_bwd_halo_f32")
    LAUNCHES["gatv2_bwd_halo_kernel"] += 1
    return out


def backward_inner(graph, zs: Tensor, zs_halo: Optional[Tensor], zd: Tensor, g: Tensor, lse: Tensor, S: Tensor,
                   attn: Tensor, heads: int, push: Optional[Tensor] = None, fold: Optional[Tuple[Tensor, Tensor]] = None,
                   row_begin: int = 0, row_end: Optional[int] = None, dzs: Optional[Tensor] = None,
                   dzd: Optional[Tensor] = None, da: Optional[Tensor] = None,
                   stream=None) -> Tuple[Tensor, Tensor, Tensor]:
    """dzs, dzd and the per-row shares of da [rows, F] of the local rows [row_begin, row_end) (written at
    row - row_begin).  With `push` (the push region, one row per position of total_send_idx) and `fold` =
    (fold_indptr, fold_pos), the pushed rows of each row are added to its dzs."""
    row_end = graph.n_inner if row_end is None else int(row_end)
    F = int(zs.shape[1])
    zs_halo = _rows(zs_halo, F)
    push = _rows(push, F)
    fi, fp = fold if (fold is not None and push is not None) else (None, None)
    if fi is None:
        push = None
    n = row_end - row_begin
    dzs = torch.empty((n, F), dtype=torch.float32, device=zs.device) if dzs is None else dzs
    dzd = torch.empty((n, F), dtype=torch.float32, device=zs.device) if dzd is None else dzd
    da = torch.empty((n, F), dtype=torch.float32, device=zs.device) if da is None else da
    attn = attn.contiguous()
    assert zs.stride(1) == 1 and zd.stride(1) == 1 and g.stride(1) == 1 and lse.is_contiguous() and S.is_contiguous()
    assert dzs.stride(1) == 1 and dzd.stride(1) == 1 and da.stride(1) == 1
    rc = _lib.load().adaqp_gatv2_bwd_inner_f32(
        graph.indptr.data_ptr(), graph.indices.data_ptr(), graph.n_inner, zs.data_ptr(), zs.stride(0), _ptr(zs_halo),
        zs_halo.stride(0) if zs_halo is not None else 0, zd.data_ptr(), zd.stride(0), g.data_ptr(), g.stride(0),
        lse.data_ptr(), S.data_ptr(), attn.data_ptr(), _ptr(push), push.stride(0) if push is not None else 0,
        _ptr(fi), _ptr(fp), heads, F, int(row_begin), row_end, dzs.data_ptr(), dzs.stride(0), dzd.data_ptr(),
        dzd.stride(0), da.data_ptr(), da.stride(0), _lib.stream_ptr(stream))
    _lib.check(rc, "adaqp_gatv2_bwd_inner_f32")
    LAUNCHES["gatv2_bwd_inner_kernel"] += 1
    return dzs, dzd, da

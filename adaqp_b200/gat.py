"""Graph attention aggregation (host mirror of csrc/gat.cu).

`scores(z, a_l, a_r, H)` computes the per-head attention logits el / er of every row, `forward` the softmax-weighted
aggregation of a destination row range (out and the per-head log-sum-exp), `backward` the gradient of z together with
the per-row attention-logit gradients del / der (DESIGN.md, "GAT").  Like spmm(), the source rows come from the local
matrix (ids < n_inner) and the received halo matrix without concatenation.  fp32 CUDA tensors only; there is no
torch fall-back: an unsupported shape is an error from the library.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
from torch import Tensor

from . import _lib

LAUNCHES = {"gat_scores_kernel": 0, "gat_fwd_kernel": 0, "gat_bwd_kernel": 0}


def _ptr(t: Optional[Tensor]):
    return t.data_ptr() if t is not None else None


def _rows(t: Optional[Tensor], F: int) -> Optional[Tensor]:
    if t is None or t.shape[0] == 0:
        return None
    assert t.dtype == torch.float32 and t.dim() == 2 and t.shape[1] == F and t.stride(1) == 1, (t.shape, t.stride())
    return t


def scores(z: Tensor, a_l: Tensor, a_r: Tensor, heads: int, stream=None) -> Tuple[Tensor, Tensor]:
    """el[i,h] = <z[i,h,:], a_l[h,:]>, er[i,h] = <z[i,h,:], a_r[h,:]>; a_l / a_r of shape [H, D] or [H * D]."""
    n, F = z.shape
    assert z.stride(1) == 1 and z.dtype == torch.float32
    a_l, a_r = a_l.contiguous(), a_r.contiguous()
    el = torch.empty((n, heads), dtype=torch.float32, device=z.device)
    er = torch.empty((n, heads), dtype=torch.float32, device=z.device)
    rc = _lib.load().adaqp_gat_scores_f32(z.data_ptr(), z.stride(0), n, heads, F, a_l.data_ptr(), a_r.data_ptr(),
                                          el.data_ptr(), er.data_ptr(), _lib.stream_ptr(stream))
    _lib.check(rc, "adaqp_gat_scores_f32")
    LAUNCHES["gat_scores_kernel"] += 1
    return el, er


def forward(graph, z: Tensor, z_halo: Optional[Tensor], el: Tensor, el_halo: Optional[Tensor], er: Tensor, heads: int,
            row_begin: int = 0, row_end: Optional[int] = None, out: Optional[Tensor] = None,
            lse: Optional[Tensor] = None, stream=None) -> Tuple[Tensor, Tensor]:
    """Rows [row_begin, row_end) of out = softmax-weighted sum of z over each CSR row, and lse [rows, H].
    `graph` is a LocalGraph (indptr, indices, n_inner); `out` / `lse` are written at row - row_begin."""
    row_end = graph.n_inner if row_end is None else int(row_end)
    F = int(z.shape[1])
    z_halo, el_halo = _rows(z_halo, F), _rows(el_halo, heads)
    if z_halo is None or el_halo is None:
        z_halo = el_halo = None
    n = row_end - row_begin
    if out is None:
        out = torch.empty((n, F), dtype=torch.float32, device=z.device)
    if lse is None:
        lse = torch.empty((n, heads), dtype=torch.float32, device=z.device)
    assert out.stride(1) == 1 and lse.is_contiguous() and er.is_contiguous() and el.is_contiguous()
    rc = _lib.load().adaqp_gat_fwd_f32(
        graph.indptr.data_ptr(), graph.indices.data_ptr(), graph.n_inner, z.data_ptr(), z.stride(0), _ptr(z_halo),
        z_halo.stride(0) if z_halo is not None else 0, el.data_ptr(), _ptr(el_halo), er.data_ptr(), heads, F,
        int(row_begin), row_end, out.data_ptr(), out.stride(0), lse.data_ptr(), _lib.stream_ptr(stream))
    _lib.check(rc, "adaqp_gat_fwd_f32")
    LAUNCHES["gat_fwd_kernel"] += 1
    return out, lse


def backward(graph, g: Tensor, g_halo: Optional[Tensor], z: Tensor, z_halo: Optional[Tensor], el: Tensor,
             el_halo: Optional[Tensor], aux: Tensor, aux_halo: Optional[Tensor], a_l: Tensor, a_r: Tensor, heads: int,
             row_begin: int = 0, row_end: Optional[int] = None, dz: Optional[Tensor] = None,
             dl: Optional[Tensor] = None, dr: Optional[Tensor] = None, stream=None) -> Tuple[Tensor, Tensor, Tensor]:
    """dz, del, der of the local rows [row_begin, row_end) (written at row - row_begin).  aux / aux_halo rows are
    [er | lse | s] with s[v,h] = <g[v,h,:], out[v,h,:]>."""
    row_end = graph.n_inner if row_end is None else int(row_end)
    F = int(z.shape[1])
    halo = [_rows(g_halo, F), _rows(z_halo, F), _rows(el_halo, heads), _rows(aux_halo, 3 * heads)]
    if any(t is None for t in halo):
        halo = [None] * 4
    g_halo, z_halo, el_halo, aux_halo = halo
    n = row_end - row_begin
    if dz is None:
        dz = torch.empty((n, F), dtype=torch.float32, device=z.device)
    if dl is None:
        dl = torch.empty((n, heads), dtype=torch.float32, device=z.device)
    if dr is None:
        dr = torch.empty((n, heads), dtype=torch.float32, device=z.device)
    a_l, a_r = a_l.contiguous(), a_r.contiguous()
    assert g.stride(1) == 1 and aux.is_contiguous() and el.is_contiguous() and dz.stride(1) == 1
    rc = _lib.load().adaqp_gat_bwd_f32(
        graph.indptr.data_ptr(), graph.indices.data_ptr(), graph.n_inner, g.data_ptr(), g.stride(0), _ptr(g_halo),
        g_halo.stride(0) if g_halo is not None else 0, z.data_ptr(), z.stride(0), _ptr(z_halo),
        z_halo.stride(0) if z_halo is not None else 0, el.data_ptr(), _ptr(el_halo), aux.data_ptr(), _ptr(aux_halo),
        a_l.data_ptr(), a_r.data_ptr(), heads, F, int(row_begin), row_end, dz.data_ptr(), dz.stride(0), dl.data_ptr(),
        dr.data_ptr(), _lib.stream_ptr(stream))
    _lib.check(rc, "adaqp_gat_bwd_f32")
    LAUNCHES["gat_bwd_kernel"] += 1
    return dz, dl, dr

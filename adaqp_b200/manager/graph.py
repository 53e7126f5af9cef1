"""Device-resident partition graph for the aggregation kernels.

Stands in for the DGL graph objects the reference keeps on the GPU
(AdaQP/manager/graphEngine.py:62-63,149-161): dst-major CSR of all in-edges of the inner
nodes, global degrees in `ndata`, and the degree norms of AdaQP/model/ops.py:21-25,49-57
precomputed once with the same torch expressions (deg.float().clamp(min=1).pow(p)).
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch

from .. import _lib


class LocalGraph(object):
    def __init__(self, indptr: np.ndarray, indices: np.ndarray, in_degrees: np.ndarray,
                 out_degrees: np.ndarray, n_inner: int, n_halo: int, device: torch.device):
        self.device = torch.device(device)
        self.n_inner, self.n_halo = int(n_inner), int(n_halo)
        self.indptr = torch.from_numpy(np.ascontiguousarray(indptr, np.int64)).to(self.device)
        self.indices = torch.from_numpy(np.ascontiguousarray(indices, np.int32)).to(self.device)
        self.nnz = int(self.indices.numel())
        # first halo column of every row (columns are sorted, halo ids >= n_inner): lets the
        # aggregation of a row be split into its local-source and halo-source segments
        ip = np.ascontiguousarray(indptr, np.int64)
        is_local = (np.asarray(indices) < self.n_inner)
        csum = np.concatenate([[0], np.cumsum(is_local, dtype=np.int64)])
        self.halo_split = torch.from_numpy(ip[:-1] + (csum[ip[1:]] - csum[ip[:-1]])).to(self.device)
        self.ndata: Dict[str, torch.Tensor] = {
            "in_degrees": torch.from_numpy(np.ascontiguousarray(in_degrees)).to(self.device),
            "out_degrees": torch.from_numpy(np.ascontiguousarray(out_degrees)).to(self.device),
        }
        ind = self.ndata["in_degrees"].float().clamp(min=1)
        outd = self.ndata["out_degrees"].float().clamp(min=1)
        self.norm = {
            "in_-0.5": ind.pow(-0.5).contiguous(), "out_-0.5": outd.pow(-0.5).contiguous(),
            "out_-1": torch.pow(outd, -1).contiguous(), "in_+1_-1": torch.pow(ind + 1, -1).contiguous(),
            "out_+1_-1": torch.pow(outd + 1, -1).contiguous(),
        }

    def num_nodes(self) -> int:
        return self.n_inner + self.n_halo

    def num_edges(self) -> int:
        return self.nnz

    def to(self, device):
        return self if torch.device(device) == self.device else NotImplemented


class RowList(object):
    """A device list of destination rows for spmm(..., rows=): int32 CSR row ids, ascending and unique, with their
    bounds kept on the host (`first`, `last`; None when empty), so a launch can check its range without reading
    the device.  Built by row_list(); `below(n)` / `from_(n)` are the views of the ids < n and >= n."""

    def __init__(self, ids: torch.Tensor, host: np.ndarray):
        assert ids.dtype == torch.int32 and ids.dim() == 1 and ids.is_contiguous() and ids.numel() == host.size
        self.ids, self._host = ids, host
        self.n = int(host.size)
        self.first = int(host[0]) if self.n else None
        self.last = int(host[-1]) if self.n else None

    def _cut(self, k: int) -> int:
        return int(np.searchsorted(self._host, k, side="left"))

    def below(self, n: int) -> "RowList":
        k = self._cut(n)
        return RowList(self.ids[:k], self._host[:k])

    def from_(self, n: int) -> "RowList":
        k = self._cut(n)
        return RowList(self.ids[k:], self._host[k:])

    def __len__(self) -> int:
        return self.n


def row_list(mask: torch.Tensor, n_rows: int, device) -> RowList:
    """The rows a mask selects among [0, n_rows) as a RowList on `device`: a bool mask of n_rows entries, or an
    index tensor (any integer type, duplicates and order allowed).  Built on the host once; ids outside
    [0, n_rows) are refused."""
    m = mask.detach().cpu()
    if m.dtype == torch.bool:
        if m.dim() != 1 or m.numel() != n_rows:
            raise ValueError(f"bool row mask of shape {tuple(m.shape)} for {n_rows} rows")
        host = torch.nonzero(m).flatten().numpy().astype(np.int64)
    else:
        if m.is_floating_point() or m.is_complex():
            raise ValueError(f"row mask of dtype {m.dtype}: a bool mask or integer row ids")
        host = np.unique(m.flatten().to(torch.int64).numpy())
    if host.size and (host[0] < 0 or host[-1] >= n_rows):
        raise ValueError(f"row ids [{int(host[0])}, {int(host[-1])}] outside [0, {n_rows})")
    host = host.astype(np.int32)
    return RowList(torch.from_numpy(host).to(device), host)


def part_segments(graph: LocalGraph, part: Optional[str]):
    """(seg_start, seg_end, accumulate) of one launch over CSR rows, by how the launch splits each row for the
    two-pass marginal schedule: part=None reads whole rows; 'local' reads each row's local-source segment only (up to
    halo_split), which needs no halo; 'halo' reads its halo-source segment (from halo_split) and accumulates into
    what the local part wrote."""
    if part is None:
        return None, None, 0
    if part == "local":
        return None, graph.halo_split.data_ptr(), 0
    if part == "halo":
        return graph.halo_split.data_ptr(), None, 1
    raise ValueError(part)


def spmm(graph: LocalGraph, x_local: torch.Tensor, x_halo: Optional[torch.Tensor],
         pre: Optional[torch.Tensor], post: Optional[torch.Tensor], mean: bool = False,
         add_self: bool = False, row_begin: int = 0, row_end: Optional[int] = None,
         out: Optional[torch.Tensor] = None, stream=None, part: Optional[str] = None,
         live: Optional[torch.Tensor] = None, rows: Optional[RowList] = None) -> torch.Tensor:
    """out[v - row_begin] = post[v] * sum_u pre[u] x[u]  over the CSR rows [row_begin, row_end).
    part='local': only the local-source neighbours of each row (no halo needed);
    part='halo' : only the halo-source neighbours, ACCUMULATED into `out`.
    live: uint8 per row of x_local from row_live(x_local): the gather skips the all-zero local rows, which add
    exactly nothing, so the result is the same (None: every source row is read).
    rows: a RowList inside [row_begin, row_end): only those rows of `out` are computed (each exactly as without
    the list), the others are left as they are; an empty list launches nothing."""
    L = _lib.load()
    row_end = graph.n_inner if row_end is None else int(row_end)
    F = int(x_local.shape[1])
    assert x_local.dtype == torch.float32 and x_local.stride(1) == 1
    if out is None:
        out = torch.empty((row_end - row_begin, F), dtype=torch.float32, device=x_local.device)
    n_list = 0
    if rows is not None:
        assert live is None, "a row list and row liveness are not combined"
        assert rows.ids.dtype == torch.int32 and rows.ids.is_contiguous() and rows.ids.device == x_local.device
        if rows.n == 0:
            return out
        assert row_begin <= rows.first and rows.last < row_end, (rows.first, rows.last, row_begin, row_end)
        n_list = rows.n
    if x_halo is not None and x_halo.shape[0] == 0:
        x_halo = None
    seg_start, seg_end, accumulate = part_segments(graph, part)
    if part == "halo":
        assert out is not None, "the halo part accumulates into the output of the local part"
        add_self = False
    if live is not None:
        assert live.dtype == torch.uint8 and live.is_contiguous() and live.numel() >= graph.n_inner
    rc = L.adaqp_spmm_csr_seg_f32(
        graph.indptr.data_ptr(), seg_start, seg_end, graph.indices.data_ptr(), x_local.data_ptr(),
        x_local.stride(0), graph.n_inner, x_halo.data_ptr() if x_halo is not None else None,
        x_halo.stride(0) if x_halo is not None else 0,
        pre.data_ptr() if pre is not None else None, post.data_ptr() if post is not None else None,
        1 if mean else 0, 1 if add_self else 0, accumulate, int(row_begin), row_end, F, out.data_ptr(),
        out.stride(0), live.data_ptr() if live is not None else None,
        rows.ids.data_ptr() if rows is not None else None, n_list, _lib.stream_ptr(stream))
    _lib.check(rc, "adaqp_spmm_csr_seg_f32")
    return out


def row_live(x: torch.Tensor, out: Optional[torch.Tensor] = None, stream=None) -> torch.Tensor:
    """live[r] = any(x[r, :] != 0) as uint8 (a NaN row is live), one read of x on the current (or given) stream:
    the `live` argument of spmm()."""
    assert x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
    rows, F = int(x.shape[0]), int(x.shape[1])
    if out is None:
        out = torch.empty(rows, dtype=torch.uint8, device=x.device)
    assert out.dtype == torch.uint8 and out.is_contiguous() and out.numel() >= rows
    if rows == 0:
        return out
    rc = _lib.load().adaqp_row_live_f32(x.data_ptr(), x.stride(0), rows, F, out.data_ptr(), _lib.stream_ptr(stream))
    _lib.check(rc, "adaqp_row_live_f32")
    return out


# acc_mode bits of appnp_prop (include/adaqp_b200.h): the acc term is on / continue from acc / fold it into out
ACC_ON, ACC_READ, ACC_FOLD = 1, 2, 4


def appnp_prop(graph: LocalGraph, x_local: torch.Tensor, x_halo: Optional[torch.Tensor],
               pre: Optional[torch.Tensor], post: Optional[torch.Tensor], scale: float, alpha: float,
               row_begin: int = 0, row_end: Optional[int] = None, out: Optional[torch.Tensor] = None,
               tele: Optional[torch.Tensor] = None, acc: Optional[torch.Tensor] = None, acc_mode: int = 0,
               stream=None, part: Optional[str] = None) -> torch.Tensor:
    """One APPNP propagation step over CSR rows [row_begin, row_end) (csrc/spmm.cu appnp_prop_kernel):
        out[v - row_begin] = scale * post[v] * sum_u pre[u] x[u]  (+ alpha * tele[v - row_begin])
    and, with acc_mode (backward), acc[v - row_begin] = alpha * x[v] (+ acc[..] with ACC_READ), or with ACC_FOLD
    the acc term added to out instead.  `tele`, `acc` and `out` are indexed like out.  part='local' / 'halo' as in
    spmm(): the halo part accumulates its segment's share into `out` and adds no tele / acc term.  16-byte rows whose
    width is a multiple of 128 above 128 run column-sliced (appnp_prop_sliced_kernel, bitwise the same result); option
    spmm_slice_cols forces a slice width as for spmm()."""
    L = _lib.load()
    row_end = graph.n_inner if row_end is None else int(row_end)
    F = int(x_local.shape[1])
    assert x_local.dtype == torch.float32 and x_local.stride(1) == 1
    if out is None:
        out = torch.empty((row_end - row_begin, F), dtype=torch.float32, device=x_local.device)
    if x_halo is not None and x_halo.shape[0] == 0:
        x_halo = None
    seg_start, seg_end, accumulate = part_segments(graph, part)
    for t in (tele, acc):
        assert t is None or (t.dtype == torch.float32 and t.stride(1) == 1 and t.shape[0] >= row_end - row_begin)
    rc = L.adaqp_appnp_prop_f32(
        graph.indptr.data_ptr(), seg_start, seg_end, graph.indices.data_ptr(), x_local.data_ptr(), x_local.stride(0),
        graph.n_inner, x_halo.data_ptr() if x_halo is not None else None,
        x_halo.stride(0) if x_halo is not None else 0,
        pre.data_ptr() if pre is not None else None, post.data_ptr() if post is not None else None,
        float(scale), float(alpha), tele.data_ptr() if tele is not None else None,
        tele.stride(0) if tele is not None else 0, acc.data_ptr() if acc is not None else None,
        acc.stride(0) if acc is not None else 0, int(acc_mode), accumulate, int(row_begin), row_end, F,
        out.data_ptr(), out.stride(0), _lib.stream_ptr(stream))
    _lib.check(rc, "adaqp_appnp_prop_f32")
    return out

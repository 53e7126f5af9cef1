"""Partition -> hot-path layout, DGL-free (numpy CSR).

Restates the data-layout contract the reference's Manager hands to the exchange and
aggregation code (SURVEY.md 3.6):

  halo requests / send_idx / recv_idx / aggregation scores   AdaQP/manager/processing.py:40-107
  node reorder [central | marginal | halo]                   AdaQP/manager/conversion.py:56-90
  send_idx -> (lo, hi) offsets into total_send_idx           AdaQP/manager/conversion.py:92-106
  central / marginal decomposition                           AdaQP/manager/conversion.py:114-172

All functions are pure (no process group): the all_gather steps of the reference are the
caller's job (GraphEngine does them over the control plane; tests do them in-process).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Tuple

import numpy as np

from ..helper import DistGNNType
from .partition_synth import RawPartition


def _clamped_pow(deg: np.ndarray, p: float) -> np.ndarray:
    return np.power(np.maximum(deg.astype(np.float32), np.float32(1.0)), np.float32(p)).astype(np.float32)


def halo_requests(raw: RawPartition, model_type: DistGNNType):
    """Receiver side of processing.py:40-60.

    Returns (recv_idx, requests): recv_idx[p] = positions inside the halo block of the
    halo nodes owned by p (ascending); requests[p] = (ids local to p's inner block in the
    same order, (forward score, backward score)) -- what p must send and how much the
    receiver's aggregation weighs each row."""
    n_in = raw.n_inner
    nnz_dst = np.repeat(np.arange(n_in, dtype=np.int64), np.diff(raw.indptr))
    src = raw.indices.astype(np.int64)
    from_halo = src >= n_in
    h = src[from_halo] - n_in
    v = nnz_dst[from_halo]
    if model_type in (DistGNNType.DistGCN, DistGNNType.DistAPPNP, DistGNNType.DistGCNII):
        # processing.py:90-98: sum_v in_deg[v]^-1/2 * out_deg[h]^-1/2 over halo h -> inner v edges (APPNP and GCNII
        # weigh their halo rows by the same norms, scaled by the constant 1 - alpha)
        w_f = _clamped_pow(raw.in_degrees[v], -0.5).astype(np.float64)
        fp = np.bincount(h, weights=w_f, minlength=raw.n_halo) * _clamped_pow(raw.out_degrees[n_in:], -0.5)
        w_b = _clamped_pow(raw.out_degrees[v], -0.5).astype(np.float64)
        bp = np.bincount(h, weights=w_b, minlength=raw.n_halo) * _clamped_pow(raw.in_degrees[n_in:], -0.5)
    elif model_type is DistGNNType.DistSAGE:
        fp = np.bincount(h, weights=_clamped_pow(raw.in_degrees[v], -1).astype(np.float64), minlength=raw.n_halo)
        bp = np.bincount(h, weights=_clamped_pow(raw.out_degrees[v], -1).astype(np.float64), minlength=raw.n_halo)
    elif model_type in (DistGNNType.DistGAT, DistGNNType.DistGATv2):
        # static proxy: the attention weights are data-dependent and change every step, so a halo row is scored by
        # the weight it would get under uniform attention, sum_v 1/indeg[v] (the SAGE-mean score); forward rows (z)
        # and backward rows (dL/dout) are both weighed by it
        fp = np.bincount(h, weights=_clamped_pow(raw.in_degrees[v], -1).astype(np.float64), minlength=raw.n_halo)
        bp = fp.copy()
    else:
        raise NotImplementedError(f"{model_type} is not implemented yet.")
    fp = fp.astype(np.float32)
    bp = bp.astype(np.float32)
    recv_idx: Dict[int, np.ndarray] = {}
    requests: Dict[int, Tuple[np.ndarray, Tuple[np.ndarray, np.ndarray]]] = {}
    for p in range(raw.num_parts):
        if p == raw.rank:
            continue
        pos = np.nonzero(raw.halo_part == p)[0].astype(np.int64)
        if pos.size == 0:
            continue
        recv_idx[p] = pos
        requests[p] = (raw.halo_gid[pos] - int(raw.starts[p]), (fp[pos], bp[pos]))
    return recv_idx, requests


def send_side(rank: int, requests_of_all: List[Dict[int, tuple]]):
    """processing.py:62-71: rows this rank must send to each peer, in the peer's halo order."""
    send_idx: Dict[int, np.ndarray] = {}
    scores: Dict[int, Tuple[np.ndarray, np.ndarray]] = {}
    for p, req in enumerate(requests_of_all):
        if p == rank or req is None:
            continue
        if rank in req:
            send_idx[p] = np.asarray(req[rank][0], np.int64)
            scores[p] = req[rank][1]
    return send_idx, scores


@dataclass
class Reordered:
    n_central: int
    n_marginal: int
    n_inner: int
    n_halo: int
    new_id: np.ndarray        # old inner id -> new inner id
    indptr: np.ndarray        # CSR rows in new inner order (dst), cols new local ids
    indices: np.ndarray
    in_degrees: np.ndarray    # new order, inner + halo
    out_degrees: np.ndarray
    feat: np.ndarray
    label: np.ndarray
    train_mask: np.ndarray
    val_mask: np.ndarray
    test_mask: np.ndarray
    send_idx: Dict[int, np.ndarray]   # reordered local ids per peer


def reorder_partition(raw: RawPartition, send_idx: Dict[int, np.ndarray]) -> Reordered:
    """conversion.py:56-90: inner nodes -> [central | marginal], halo untouched.
    marginal = inner destinations of at least one halo -> inner edge."""
    n_in, n_h = raw.n_inner, raw.n_halo
    deg = np.diff(raw.indptr)
    dst = np.repeat(np.arange(n_in, dtype=np.int64), deg)
    marginal = np.zeros(n_in, bool)
    marginal[np.unique(dst[raw.indices >= n_in])] = True
    n_m = int(marginal.sum())
    n_c = n_in - n_m
    new_id = np.empty(n_in, np.int64)
    new_id[~marginal] = np.arange(n_c)
    new_id[marginal] = np.arange(n_c, n_in)
    old_of_new = np.empty(n_in, np.int64)
    old_of_new[new_id] = np.arange(n_in)
    # permute CSR rows, remap inner columns; rows keep ascending column order
    new_deg = deg[old_of_new]
    indptr = np.concatenate([[0], np.cumsum(new_deg)]).astype(np.int64)
    gather = _row_gather_index(raw.indptr, old_of_new, new_deg)
    cols = raw.indices[gather].astype(np.int64)
    inner_col = cols < n_in
    cols[inner_col] = new_id[cols[inner_col]]
    cols = _sort_within_rows(indptr, cols)

    def perm_nodes(a):
        out = a.copy()
        out[new_id] = a[:n_in]
        return out

    in_deg = raw.in_degrees.copy()
    in_deg[:n_in][new_id] = raw.in_degrees[:n_in]
    out_deg = raw.out_degrees.copy()
    out_deg[:n_in][new_id] = raw.out_degrees[:n_in]
    return Reordered(n_central=n_c, n_marginal=n_m, n_inner=n_in, n_halo=n_h, new_id=new_id,
                     indptr=indptr, indices=cols.astype(np.int32), in_degrees=in_deg,
                     out_degrees=out_deg, feat=perm_nodes(raw.feat), label=perm_nodes(raw.label),
                     train_mask=perm_nodes(raw.train_mask), val_mask=perm_nodes(raw.val_mask),
                     test_mask=perm_nodes(raw.test_mask),
                     send_idx={p: new_id[ids] for p, ids in send_idx.items()})


def _row_gather_index(indptr: np.ndarray, rows: np.ndarray, row_len: np.ndarray) -> np.ndarray:
    """Flat positions of the entries of `rows` (in that order) in a CSR."""
    total = int(row_len.sum())
    if total == 0:
        return np.zeros(0, np.int64)
    starts = indptr[rows]
    out_ptr = np.concatenate([[0], np.cumsum(row_len)])[:-1]
    idx = np.arange(total, dtype=np.int64)
    return idx - np.repeat(out_ptr, row_len) + np.repeat(starts, row_len)


def _sort_within_rows(indptr: np.ndarray, cols: np.ndarray) -> np.ndarray:
    import scipy.sparse as sp
    n = indptr.size - 1
    width = int(cols.max()) + 1 if cols.size else 1
    A = sp.csr_matrix((np.ones(cols.size, np.int8), cols, indptr), shape=(n, width))
    A.sort_indices()
    return A.indices.astype(np.int64)


def convert_send_idx(send_idx: Dict[int, np.ndarray]):
    """conversion.py:92-106: per-peer (lo, hi) offsets into the concatenation (dict order =
    ascending peer rank)."""
    offset = 0
    converted: Dict[int, Tuple[int, int]] = {}
    parts = []
    for p, ids in send_idx.items():
        converted[p] = (offset, offset + len(ids))
        offset += len(ids)
        parts.append(np.asarray(ids, np.int64))
    total = np.concatenate(parts) if parts else np.zeros(0, np.int64)
    return converted, total


def decomposition_indices(indptr: np.ndarray, indices: np.ndarray, n_central: int, n_inner: int):
    """src_marginal_idx / src_central_idx of conversion.py:133-172 (API parity; the SpMM
    kernel addresses rows of the full matrix directly and does not need them):
      src_marginal_idx = marginal nodes that feed central destinations (ascending),
      src_central_idx  = central nodes that feed marginal destinations (ascending)."""
    cols_c = indices[indptr[0]:indptr[n_central]]
    src_marginal = np.unique(cols_c[(cols_c >= n_central) & (cols_c < n_inner)]).astype(np.int64)
    cols_m = indices[indptr[n_central]:indptr[n_inner]]
    src_central = np.unique(cols_m[cols_m < n_central]).astype(np.int64)
    return src_marginal, src_central

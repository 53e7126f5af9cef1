"""Per-rank hot-path layout assembled from a raw partition (host side, one-off).

Pipeline of the reference's GraphEngine.__init__ (AdaQP/manager/graphEngine.py:54-76):
convert_partition -> get_send_recv_idx_scores -> reorder_graph -> convert_send_idx
(-> decompose_graph), restated DGL-free on numpy CSR.  `prepare_rank` is the multi-process
form (collectives supplied by the caller), `layouts_from_raw` wires W ranks inside one process
(synthetic partitions for tests, smoke() and the single-GPU loopback bench; real partitions from
`raw_partitions` or tools/convert_dgl_partition.py).
"""
from __future__ import annotations

import json
import os
from dataclasses import dataclass
from typing import Callable, Dict, List, Optional, Tuple

import numpy as np
import scipy.sparse as sp

from ..helper import DistGNNType
from . import conversion as cv
from .partition_synth import RawPartition, SynthSpec, attach_global_degrees, block_starts, build_raw_partition


@dataclass
class RankLayout:
    rank: int
    world_size: int
    n_central: int
    n_marginal: int
    n_inner: int
    n_halo: int
    indptr: np.ndarray                      # int64 [n_inner + 1], rows = inner nodes [central | marginal]
    indices: np.ndarray                     # int32, source local ids (>= n_inner: halo)
    in_degrees: np.ndarray                  # global, all local nodes
    out_degrees: np.ndarray
    feat: np.ndarray
    label: np.ndarray
    train_mask: np.ndarray
    val_mask: np.ndarray
    test_mask: np.ndarray
    send_idx: Dict[int, Tuple[int, int]]    # peer -> (lo, hi) into total_send_idx
    total_send_idx: np.ndarray              # int64 local inner row ids
    recv_idx: Dict[int, np.ndarray]         # peer -> positions inside the halo block
    scores: Dict[int, Tuple[np.ndarray, np.ndarray]]   # peer -> (forward, backward) aggregation scores
    src_marginal_idx: np.ndarray
    src_central_idx: np.ndarray
    is_bidirected: bool = True
    # int64 [n_inner], rows in [central | marginal] order: each inner node's id in the dataset's original
    # numbering (what predictions are keyed by); None in files written before the field existed
    inner_gid: Optional[np.ndarray] = None


def _finish(raw: RawPartition, recv_idx, send_ids, scores) -> RankLayout:
    ro = cv.reorder_partition(raw, send_ids)
    send_idx, total = cv.convert_send_idx(ro.send_idx)
    sm, sc = cv.decomposition_indices(ro.indptr, ro.indices, ro.n_central, ro.n_inner)
    inner_gid = None
    if raw.inner_gid is not None:
        inner_gid = np.empty(ro.n_inner, np.int64)
        inner_gid[ro.new_id] = raw.inner_gid
    return RankLayout(rank=raw.rank, world_size=raw.num_parts, n_central=ro.n_central,
                      n_marginal=ro.n_marginal, n_inner=ro.n_inner, n_halo=ro.n_halo,
                      indptr=ro.indptr, indices=ro.indices, in_degrees=ro.in_degrees,
                      out_degrees=ro.out_degrees, feat=ro.feat, label=ro.label,
                      train_mask=ro.train_mask, val_mask=ro.val_mask, test_mask=ro.test_mask,
                      send_idx=send_idx, total_send_idx=total, recv_idx=recv_idx, scores=scores,
                      src_marginal_idx=sm, src_central_idx=sc,
                      is_bidirected=bool(np.array_equal(ro.in_degrees, ro.out_degrees)), inner_gid=inner_gid)


def prepare_rank(spec: SynthSpec, rank: int, model_type: DistGNNType,
                 all_gather: Callable[[object], List[object]]) -> RankLayout:
    """Multi-process form: `all_gather(obj)` returns every rank's obj in rank order."""
    raw = build_raw_partition(spec, rank)
    degs = all_gather(raw.inner_degrees)
    attach_global_degrees(raw, degs, block_starts(spec))
    recv_idx, requests = cv.halo_requests(raw, model_type)
    all_requests = all_gather(requests)
    send_ids, scores = cv.send_side(rank, all_requests)
    return _finish(raw, recv_idx, send_ids, scores)


def layouts_from_raw(raws: List[RawPartition], model_type: DistGNNType) -> List[RankLayout]:
    """halo_requests -> send_side -> reorder / convert_send_idx / decompose for all ranks in one process (the
    reference does the two exchanges with all_gather_object, processing.py:65-71).  `raws` carry global degrees."""
    rr = [cv.halo_requests(r, model_type) for r in raws]
    all_requests = [x[1] for x in rr]
    out = []
    for r in range(len(raws)):
        send_ids, scores = cv.send_side(r, all_requests)
        out.append(_finish(raws[r], rr[r][0], send_ids, scores))
    return out


def prepare_all_in_process(spec: SynthSpec, model_type: DistGNNType = DistGNNType.DistGCN) -> List[RankLayout]:
    W = spec.num_parts
    raws = [build_raw_partition(spec, r) for r in range(W)]
    degs = [r.inner_degrees for r in raws]
    starts = block_starts(spec)
    for r in raws:
        attach_global_degrees(r, degs, starts)
    return layouts_from_raw(raws, model_type)


def raw_partitions(graph, part: np.ndarray) -> List[RawPartition]:
    """Cut a global graph (helper.dataset.GlobalGraph: symmetric CSR, node data) along `part`.

    Nodes are relabelled so that block p owns a contiguous range of global ids, ascending original id within
    the block (DGL's reshuffle).  Rank p keeps the in-edges of its inner nodes, the ids and owners of its halo
    nodes, its slices of features / labels / masks and the global degrees (CSR row lengths) of all its nodes."""
    part = np.asarray(part, np.int64)
    n = graph.indptr.size - 1
    assert part.shape == (n,), (part.shape, n)
    W = int(part.max()) + 1
    old_of_new = np.argsort(part, kind="stable")
    new_of_old = np.empty(n, np.int64)
    new_of_old[old_of_new] = np.arange(n)
    starts = np.concatenate([[0], np.cumsum(np.bincount(part, minlength=W))]).astype(np.int64)
    deg = np.diff(graph.indptr).astype(np.int64)
    A = sp.csr_matrix((np.ones(graph.indices.size, np.int8), graph.indices, graph.indptr), shape=(n, n))
    raws = []
    for p in range(W):
        g0, g1 = int(starts[p]), int(starts[p + 1])
        ids = old_of_new[g0:g1]
        rows = A[ids]
        src = new_of_old[rows.indices]
        inner = (src >= g0) & (src < g1)
        halo_gid = np.unique(src[~inner])
        local = np.empty(src.size, np.int64)
        local[inner] = src[inner] - g0
        local[~inner] = (g1 - g0) + np.searchsorted(halo_gid, src[~inner])
        B = sp.csr_matrix((np.ones(src.size, np.int8), local, rows.indptr), shape=(g1 - g0, g1 - g0 + halo_gid.size))
        B.sort_indices()
        d = deg[np.concatenate([ids, old_of_new[halo_gid]])]
        raws.append(RawPartition(
            rank=p, num_parts=W, n_inner=g1 - g0, inner_start=g0, starts=starts, indptr=B.indptr.astype(np.int64),
            indices=B.indices.astype(np.int32), halo_gid=halo_gid.astype(np.int64),
            halo_part=(np.searchsorted(starts, halo_gid, side="right") - 1).astype(np.int32),
            feat=graph.feat[ids], label=graph.label[ids], train_mask=graph.train_mask[ids],
            val_mask=graph.val_mask[ids], test_mask=graph.test_mask[ids], in_degrees=d, out_degrees=d.copy(),
            inner_gid=ids.astype(np.int64)))
    return raws


def save_partition_book(part: np.ndarray, part_dir: str, dataset: str, header: dict) -> str:
    """`<part_dir>/<dataset>/<W>part/partition_book.npz`: the block of every original node id plus a JSON header
    (seed, k, edge cut, block sizes, halo rows ...); plain arrays, nothing is unpickled on load."""
    d = f"{part_dir}/{dataset}/{int(header['k'])}part"
    os.makedirs(d, exist_ok=True)
    path = f"{d}/partition_book.npz"
    np.savez_compressed(path, part=np.ascontiguousarray(part, np.int32),
                        header_json=np.frombuffer(json.dumps(header).encode("utf-8"), dtype=np.uint8))
    return path


def read_partition_book(path: str):
    z = np.load(path, allow_pickle=False)
    return z["part"], json.loads(bytes(z["header_json"]).decode("utf-8"))

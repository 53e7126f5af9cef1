"""GPU multilevel k-way graph partitioning (label propagation throughout, KaMinPar / Jet style).

Host mirror of csrc/partition.cu, as dense.py and fused.py are for theirs: it replaces
dgl.distributed.partition_graph(graph, ..., num_hops=1, balance_edges=False) -- METIS -- at
AdaQP/helper/partition.py:71-72 with the same objective and constraint:

* minimise the edge cut (undirected non-self edges whose ends lie in different blocks), unit vertex weights;
* every block holds at most ceil(1.03 * N / k) nodes (METIS's default imbalance) and at least one.

Levels: (1) coarsen by size-constrained LP clustering (cluster weight cap 0.03 * N / k, the balance slack)
and contraction until about 2000 * k vertices remain or a level shrinks by less than 5 %; (2) greedy
graph-growing recursive bisection of the coarsest graph on the host (numpy), best of a few seeds, then
balanced; (3) project down level by level with a few rounds of k-way LP refinement each, and finish with a
deterministic rebalancing pass and a fill of empty blocks.  The CUDA kernels rate and apply moves and remap
edges; torch sorts proposals and contraction keys and holds every buffer.  Same input and seed give the same
`part` on every run (the move rule is in DESIGN.md, "Graph partitioning").  There is no CPU path.
"""
from __future__ import annotations

import time
from dataclasses import dataclass
from typing import Dict, Optional

import numpy as np
import scipy.sparse as sp
import torch

from . import _lib

CLUSTER_ROUNDS = 5
REFINE_ROUNDS = 6
COARSEST_PER_BLOCK = 2000
MIN_SHRINK = 0.95
INITIAL_SEEDS = 4
INT64_MAX = (1 << 63) - 1
HUB_SCRATCH_BYTES = 1 << 30


def max_block_weight(n: int, k: int) -> int:
    """ceil(1.03 * N / k), in exact integer arithmetic."""
    return -(-103 * n // (100 * k))


def check_k(n: int, k: int):
    if not 1 <= k <= _lib.MAX_PARTS:
        raise ValueError(f"k={k}: supported 1 <= k <= {_lib.MAX_PARTS} (the exchange's channel limit)")
    if n < k:
        raise ValueError(f"cannot cut {n} nodes into {k} non-empty blocks")


def edge_cut(indptr: np.ndarray, indices: np.ndarray, part: np.ndarray) -> int:
    """Undirected non-self edges of a symmetric CSR whose two ends are in different blocks."""
    rows = np.repeat(np.arange(indptr.size - 1), np.diff(indptr))
    return int(np.count_nonzero(part[rows] != part[indices])) // 2


@dataclass
class Graph:
    """One level on the device: symmetric CSR without self-loops, integer edge and vertex weights."""
    indptr: torch.Tensor      # int64 [n + 1]
    indices: torch.Tensor     # int32
    ew: torch.Tensor          # int32, one per edge
    vw: torch.Tensor          # int32 [n]

    @property
    def n(self) -> int:
        return self.vw.numel()

    @staticmethod
    def from_csr(indptr, indices, device, ew=None, vw=None) -> "Graph":
        """Upload a CSR and drop its self-loops (they never change the cut)."""
        ip = torch.as_tensor(np.asarray(indptr, np.int64)).to(device)
        ix = torch.as_tensor(np.asarray(indices, np.int32)).to(device)
        n = ip.numel() - 1
        rows = torch.repeat_interleave(torch.arange(n, device=device, dtype=torch.int32), ip.diff())
        keep = ix != rows
        csum = torch.zeros(ix.numel() + 1, dtype=torch.int64, device=device)
        torch.cumsum(keep.long(), 0, out=csum[1:])
        ew_t = torch.ones(ix.numel(), dtype=torch.int32, device=device) if ew is None else \
            torch.as_tensor(np.asarray(ew, np.int32)).to(device)
        vw_t = torch.ones(n, dtype=torch.int32, device=device) if vw is None else \
            torch.as_tensor(np.asarray(vw, np.int32)).to(device)
        return Graph(csum[ip], ix[keep], ew_t[keep], vw_t)

    def hub_tables(self):
        """Hub list of the clustering rating and its zeroed dense counter rows (at most HUB_SCRATCH_BYTES)."""
        hubs = torch.nonzero(self.indptr.diff() > _lib.LP_HUB_DEGREE).squeeze(1).int()
        if hubs.numel() == 0:
            return None
        ctas = int(max(1, min(hubs.numel(), 1024, HUB_SCRATCH_BYTES // (4 * self.n))))
        return hubs, torch.zeros(ctas * self.n, dtype=torch.int32, device=hubs.device), ctas


def _p(t: Optional[torch.Tensor]) -> int:
    return 0 if t is None else t.data_ptr()


def _sorted_proposals(tgt, gain, hkey, group) -> torch.Tensor:
    """Proposing vertices ordered by (group asc, gain desc, hkey asc, v asc): stable sorts, last key first."""
    o = torch.nonzero(tgt >= 0).squeeze(1)
    o = o[torch.sort(hkey[o], stable=True).indices]
    o = o[torch.sort(-gain[o], stable=True).indices]
    o = o[torch.sort(group[o], stable=True).indices]
    return o


def _apply(g: Graph, tgt, gain, hkey, label, lw, cap: int) -> int:
    o = _sorted_proposals(tgt, gain, hkey, tgt)
    if o.numel() == 0:
        return 0
    csum = torch.cumsum(g.vw[o].long(), 0)
    dlw = torch.zeros_like(lw)
    _lib.check(_lib.load().adaqp_lp_apply(_p(o.int()), o.numel(), _p(csum), _p(tgt), _p(g.vw), _p(label), _p(lw),
                                          int(cap), _p(dlw), _lib.stream_ptr()), "lp_apply")
    lw += dlw
    return o.numel()


def _scratch(g: Graph):
    dev = g.vw.device
    return (torch.empty(g.n, dtype=torch.int32, device=dev), torch.empty(g.n, dtype=torch.int64, device=dev),
            torch.empty(g.n, dtype=torch.int64, device=dev))


def cluster_subround(g: Graph, label, lw, cap: int, seed: int, r: int, s: int, hubs=None, scratch=None) -> int:
    """One clustering sub-round (r, s): rate, order, apply.  `label` int32 [n], `lw` int64 [n] updated in place."""
    tgt, gain, hkey = scratch or _scratch(g)
    h = hubs if hubs is not None else g.hub_tables()
    hv, hscratch, hctas = h if h is not None else (None, None, 0)
    _lib.check(_lib.load().adaqp_lp_rate_clusters(
        _p(g.indptr), _p(g.indices), _p(g.ew), _p(g.vw), g.n, _p(label), _p(lw), int(cap), _p(hv),
        0 if hv is None else hv.numel(), _p(hscratch), hctas, seed, r, s, _p(tgt), _p(gain), _p(hkey),
        _lib.stream_ptr()), "lp_rate_clusters")
    return _apply(g, tgt, gain, hkey, label, lw, cap)


def refine_subround(g: Graph, part, bw, k: int, cap: int, seed: int, r: int, s: int, scratch=None) -> int:
    """One k-way refinement sub-round (r, s).  `part` int32 [n], `bw` int64 [k] updated in place."""
    tgt, gain, hkey = scratch or _scratch(g)
    _lib.check(_lib.load().adaqp_lp_rate_blocks(
        _p(g.indptr), _p(g.indices), _p(g.ew), _p(g.vw), g.n, _p(part), _p(bw), k, int(cap), seed, r, s, 0,
        _p(tgt), _p(gain), _p(hkey), _lib.stream_ptr()), "lp_rate_blocks")
    return _apply(g, tgt, gain, hkey, part, bw, cap)


def rebalance(g: Graph, part, bw, k: int, cap: int, seed: int, max_rounds: int = 256) -> int:
    """Move vertices out of blocks over `cap` into blocks with room, least cut increase first.  Returns rounds."""
    tgt, gain, hkey = _scratch(g)
    lib = _lib.load()
    for r in range(max_rounds):
        if int(bw.max()) <= cap:
            return r
        _lib.check(lib.adaqp_lp_rate_blocks(
            _p(g.indptr), _p(g.indices), _p(g.ew), _p(g.vw), g.n, _p(part), _p(bw), k, int(cap), seed,
            (1 << 31) + r, 0, 1, _p(tgt), _p(gain), _p(hkey), _lib.stream_ptr()), "lp_rate_blocks (rebalance)")
        o = _sorted_proposals(tgt, gain, hkey, part)
        if o.numel() == 0:
            break
        csum = torch.cumsum(g.vw[o].long(), 0)
        _lib.check(lib.adaqp_lp_rebalance_select(_p(o.int()), o.numel(), _p(csum), _p(part), _p(g.vw), _p(bw),
                                                 int(cap), _p(tgt), _lib.stream_ptr()), "lp_rebalance_select")
        _apply(g, tgt, gain, hkey, part, bw, cap)
    if int(bw.max()) > cap:
        raise RuntimeError(f"rebalancing did not bring every block under {cap}: {bw.tolist()}")
    return max_rounds


def contract(g: Graph, label) -> tuple:
    """Coarse graph of the clusters `label` and the map fine vertex -> coarse vertex."""
    uniq, cid = torch.unique(label, return_inverse=True)
    cid = cid.int()
    nc = uniq.numel()
    dev = g.vw.device
    cvw = torch.zeros(nc, dtype=torch.int64, device=dev).index_add_(0, cid.long(), g.vw.long()).int()
    key = torch.empty(g.indices.numel(), dtype=torch.int64, device=dev)
    _lib.check(_lib.load().adaqp_contract_edges(_p(g.indptr), _p(g.indices), g.n, _p(cid), _p(key),
                                                _lib.stream_ptr()), "contract_edges")
    skey, perm = torch.sort(key)
    m = int(torch.searchsorted(skey, torch.tensor([INT64_MAX], device=dev)))
    skey = skey[:m]
    w = torch.cumsum(g.ew[perm[:m]].long(), 0)
    ukey, counts = torch.unique_consecutive(skey, return_counts=True)
    ends = torch.cumsum(counts, 0) - 1
    cw = w[ends]
    cw[1:] -= w[ends[:-1]]
    rows = ukey >> 32
    indptr = torch.zeros(nc + 1, dtype=torch.int64, device=dev)
    torch.cumsum(torch.bincount(rows, minlength=nc), 0, out=indptr[1:])
    return Graph(indptr, (ukey & 0xFFFFFFFF).int(), cw.int(), cvw), cid


# ------------------------------------------------------------------- host initial partition
def _grow(A: sp.csr_matrix, vw: np.ndarray, dw: np.ndarray, target: int, rng: np.random.Generator) -> np.ndarray:
    """Greedy graph growing: from a random seed, repeatedly add the 1/32 of the frontier with the largest share of
    their edge weight going into the region (ties by a random priority) while it fits under `target`.  The share,
    unlike the absolute gain, does not favour light vertices of a coarse graph.  Returns the region mask."""
    n = vw.size
    rank = np.empty(n, np.int64)
    rank[rng.permutation(n)] = np.arange(n)
    deg = np.diff(A.indptr)
    inr = np.zeros(n, bool)
    conn = np.zeros(n, np.float64)
    w = 0
    while w < target:
        room = target - w
        cand = np.nonzero(~inr & (conn > 0))[0]
        if cand.size == 0:                       # new component: a batch of isolated vertices or one seed
            rest = np.nonzero(~inr & (vw <= room))[0]
            if rest.size == 0:
                break
            rest = rest[np.argsort(rank[rest], kind="stable")]
            iso = rest[deg[rest] == 0]
            if iso.size:
                fit = iso[np.cumsum(vw[iso]) <= room]
            else:
                fit = rest[:1]
        else:
            order = cand[np.lexsort((rank[cand], -conn[cand] / np.maximum(dw[cand], 1e-300)))]
            take = order[:max(1, order.size // 32)]
            fit = take[np.cumsum(vw[take]) <= room]
            if fit.size == 0:
                ok = order[vw[order] <= room]
                if ok.size == 0:
                    break
                fit = ok[:1]
        inr[fit] = True
        w += int(vw[fit].sum())
        conn += np.asarray(A[fit].sum(axis=0)).ravel()
    return inr


def _refine_bisection(A: sp.csr_matrix, vw: np.ndarray, dw: np.ndarray, side: np.ndarray, caps, rng,
                      passes: int = 12) -> np.ndarray:
    """Two-way label propagation: move the vertices with a positive gain to the other side, best gain first, while
    that side stays under its cap; alternate directions; keep the best cut seen."""
    rank = rng.permutation(side.size)
    best, best_cut = side.copy(), None
    for p in range(passes):
        c1 = A @ side.astype(np.float64)
        own = np.where(side, c1, dw - c1)
        gain = dw - 2 * own
        cut = float((dw - own).sum()) / 2
        if best_cut is None or cut < best_cut:
            best, best_cut = side.copy(), cut
        src = bool(p % 2)
        cand = np.nonzero((side == src) & (gain > 0))[0]
        if cand.size == 0:
            if p > 0 and not np.any((side != src) & (gain > 0)):
                break
            continue
        cand = cand[np.lexsort((rank[cand], -gain[cand]))]
        room = caps[int(not src)] - int(vw[side != src].sum())
        take = cand[np.cumsum(vw[cand]) <= room]
        side = side.copy()
        side[take] = not src
    c1 = A @ side.astype(np.float64)
    cut = float((dw - np.where(side, c1, dw - c1)).sum()) / 2
    return side if cut < best_cut else best


def _bisect(A: sp.csr_matrix, vw: np.ndarray, k0: int, k: int, rng, n_seeds: int) -> np.ndarray:
    total = int(vw.sum())
    target = int(round(total * k0 / k))
    caps = (int(total * k0 / k * 1.01) + 1, int(total * (k - k0) / k * 1.01) + 1)
    dw = np.asarray(A.sum(axis=1)).ravel()
    best, best_cut = None, None
    for _ in range(n_seeds):
        side = _refine_bisection(A, vw, dw, _grow(A, vw, dw, target, rng), caps, rng)
        c1 = A @ side.astype(np.float64)
        cut = float((dw - np.where(side, c1, dw - c1)).sum())
        if best is None or cut < best_cut:
            best, best_cut = side, cut
    return best


def _recursive_bisection(A, vw, ids, k, first, part, rng, n_seeds):
    if k == 1:
        part[ids] = first
        return
    k0 = k // 2
    side = _bisect(A, vw, k0, k, rng, n_seeds)
    for mask, kk, f in ((side, k0, first), (~side, k - k0, first + k0)):
        sub = np.nonzero(mask)[0]
        _recursive_bisection(A[sub][:, sub].tocsr(), vw[sub], ids[sub], kk, f, part, rng, n_seeds)


def _host_balance(A: sp.csr_matrix, vw: np.ndarray, part: np.ndarray, k: int, cap: int):
    """Move single vertices from the heaviest to the lightest block (least cut increase) until no block is over
    `cap` or no vertex fits; the finest level's rebalancing pass handles what remains."""
    bw = np.bincount(part, weights=vw, minlength=k).astype(np.int64)
    for _ in range(A.shape[0]):
        hi = int(np.argmax(bw))
        if bw[hi] <= cap:
            return
        lo = int(np.argmin(bw))
        cand = np.nonzero((part == hi) & (vw <= cap - bw[lo]))[0]
        if cand.size == 0:
            return
        sub = A[cand]
        v = cand[int(np.argmax(sub @ (part == lo).astype(np.float64) - sub @ (part == hi).astype(np.float64)))]
        part[v] = lo
        bw[hi] -= vw[v]
        bw[lo] += vw[v]


def initial_partition(indptr, indices, ew, vw, k: int, seed: int = 0, n_seeds: int = INITIAL_SEEDS,
                      total_weight: Optional[int] = None) -> np.ndarray:
    """Host k-way partition of a (coarse) symmetric CSR graph: greedy graph-growing recursive bisection, the best
    of `n_seeds` seeds per bisection, then balanced against ceil(1.03 * total_weight / k)."""
    n = len(indptr) - 1
    vw = np.asarray(vw, np.int64)
    A = sp.csr_matrix((np.asarray(ew, np.float64), np.asarray(indices, np.int64), np.asarray(indptr, np.int64)),
                      shape=(n, n))
    part = np.zeros(n, np.int32)
    rng = np.random.default_rng(seed)
    _recursive_bisection(A, vw, np.arange(n), k, 0, part, rng, n_seeds)
    total = int(vw.sum()) if total_weight is None else int(total_weight)
    _host_balance(A, vw, part, k, max_block_weight(total, k))
    return part


# ------------------------------------------------------------------- driver
def _sync_time(t0: float) -> float:
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def partition(indptr, indices, k: int, seed: int = 0, device=None, info: Optional[Dict] = None) -> np.ndarray:
    """k-way partition `part int32[N]` of a symmetric CSR graph (self-loops allowed, ignored).

    `info`, when given, receives the levels, per-phase times (host clock around device-synchronised work)
    and the final edge cut."""
    indptr = np.asarray(indptr, np.int64)
    n = indptr.size - 1
    check_k(n, k)
    if not torch.cuda.is_available():
        raise RuntimeError("graph partitioning runs on the GPU and no CUDA device is visible")
    _lib.load()
    dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
    info = {} if info is None else info
    times = info.setdefault("times", {})
    t0 = time.perf_counter()
    g = Graph.from_csr(indptr, indices, dev)
    times["upload"] = _sync_time(t0)
    cap = max_block_weight(n, k)
    if k == 1:
        info.update(levels=[n], edge_cut=0)
        return np.zeros(n, np.int32)

    t0 = time.perf_counter()
    levels, maps = [g], []
    ccap = max(1, int(0.03 * n / k))
    while levels[-1].n > COARSEST_PER_BLOCK * k and len(levels) < 40:
        cur = levels[-1]
        label = torch.arange(cur.n, dtype=torch.int32, device=dev)
        lw = cur.vw.long().clone()
        hubs, scratch = cur.hub_tables(), _scratch(cur)
        for r in range(CLUSTER_ROUNDS):
            moved = sum(cluster_subround(cur, label, lw, ccap, seed, r, s, hubs, scratch) for s in (0, 1))
            if moved == 0:
                break
        coarse, cid = contract(cur, label)
        if coarse.n >= cur.n:
            break
        levels.append(coarse)
        maps.append(cid)
        if coarse.n > MIN_SHRINK * cur.n:
            break
    times["coarsen"] = _sync_time(t0)

    t0 = time.perf_counter()
    top = levels[-1]
    part_h = initial_partition(top.indptr.cpu().numpy(), top.indices.cpu().numpy(), top.ew.cpu().numpy(),
                               top.vw.cpu().numpy(), k, seed, total_weight=n)
    part = torch.from_numpy(part_h).to(dev)
    times["initial"] = _sync_time(t0)

    t0 = time.perf_counter()
    for lvl in range(len(levels) - 1, -1, -1):
        cur = levels[lvl]
        if lvl < len(levels) - 1:
            part = part[maps[lvl].long()]
        bw = torch.zeros(k, dtype=torch.int64, device=dev).index_add_(0, part.long(), cur.vw.long())
        scratch = _scratch(cur)
        for r in range(REFINE_ROUNDS):
            moved = sum(refine_subround(cur, part, bw, k, cap, seed, r, s, scratch) for s in (0, 1))
            if moved == 0:
                break
    times["refine"] = _sync_time(t0)

    t0 = time.perf_counter()
    rounds = rebalance(g, part, bw, k, cap, seed)
    _fill_empty_blocks(part, bw, k)
    times["rebalance"] = _sync_time(t0)
    info["rebalance_rounds"] = rounds
    info["levels"] = [lv.n for lv in levels]
    rows = torch.repeat_interleave(torch.arange(g.n, device=dev, dtype=torch.int32), g.indptr.diff())
    info["edge_cut"] = int((part[rows] != part[g.indices]).sum()) // 2
    out = part.cpu().numpy().astype(np.int32)
    assert int(bw.min()) >= 1 and int(bw.max()) <= cap, bw.tolist()
    return out


def _fill_empty_blocks(part, bw, k: int):
    """Give every empty block one node: the smallest id of the currently largest block (smallest block id on ties)."""
    for b in range(k):
        if int(bw[b]) > 0:
            continue
        src = int(np.argmax(bw.cpu().numpy()))
        v = int(torch.nonzero(part == src)[0, 0])
        part[v] = b
        bw[src] -= 1
        bw[b] += 1

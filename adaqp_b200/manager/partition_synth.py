"""DGL-free synthetic graph partitions with the reference's per-rank layout.

The reference loads METIS partitions written by dgl.distributed.partition_graph
(AdaQP/helper/partition.py:32-72, AdaQP/manager/conversion.py:17-54).  Neither DGL, the
datasets nor the network are available here, so measurements and tests run on a seeded
generator that produces, per rank, exactly what `convert_partition` hands to the rest of
the Manager: a 1-hop-halo partition graph (all in-edges of the inner nodes), node
features / labels / masks, the partition id of every halo node and GLOBAL degrees.

Model: W blocks (= partitions) of contiguous global ids; inside a block, contiguous
communities (label = community id mod classes, features = class centroid + noise) with a
`homophily` share of the intra-block edges inside communities; truncated power-law node
weights (Chung-Lu style endpoint sampling, closed-form inverse CDF); every undirected
edge leaves its block with probability `cross_fraction` towards a uniformly random other
block, ending on the `boundary_fraction` heaviest nodes of either side (a cut touches only
part of a partition); the graph is symmetrised, de-duplicated and given self-loops like
AdaQP/helper/partition.py:58-60.  Every block / block pair has its own seeded stream, so
rank p builds its partition without materialising the whole graph and both ends of a
cross edge agree.
"""
from __future__ import annotations

import os
from dataclasses import dataclass, asdict
from typing import List, Optional, Tuple

import numpy as np
import scipy.sparse as sp


@dataclass
class SynthSpec:
    name: str
    num_nodes: int
    num_edges: int                 # directed, self-loops included
    num_parts: int
    num_feats: int
    num_classes: int
    is_multilabel: bool = False
    cross_fraction: float = 0.15
    boundary_fraction: float = 0.5   # share of a block's nodes that may carry cross-partition edges
    degree_exponent: float = 2.3
    community_size: int = 4096
    homophily: float = 0.6
    feature_signal: float = 0.5
    label_noise: float = 0.05
    train_fraction: float = 0.5
    val_fraction: float = 0.1
    seed: int = 0

    def scaled(self, scale: float) -> "SynthSpec":
        """Same shape statistics (mean degree, halo ratio) on `scale` x the nodes."""
        d = asdict(self)
        mean_deg = self.num_edges / self.num_nodes
        d["num_nodes"] = max(int(self.num_nodes * scale), 8 * self.num_parts)
        d["num_edges"] = int(d["num_nodes"] * mean_deg)
        d["community_size"] = max(16, min(self.community_size, d["num_nodes"] // (4 * self.num_parts) or 16))
        return SynthSpec(**d)


def spec_from_config(config: dict, num_parts: int, scale: float = 1.0) -> SynthSpec:
    """Build a spec from adaqp_b200/config/<dataset>.yaml (sections data + synthetic)."""
    d, s = config["data"], config["synthetic"]
    spec = SynthSpec(name=d["name"], num_nodes=int(s["num_nodes"]), num_edges=int(s["num_edges"]),
                     num_parts=num_parts, num_feats=int(d["num_feats"]),
                     num_classes=int(d["num_classes"]), is_multilabel=bool(d["is_multilabel"]),
                     cross_fraction=float(s["cross_fraction"]),
                     boundary_fraction=float(s.get("boundary_fraction", 0.5)),
                     degree_exponent=float(s.get("degree_exponent", 2.3)),
                     community_size=int(s.get("community_size", 4096)),
                     homophily=float(s.get("homophily", 0.6)),
                     feature_signal=float(os.environ.get("ADAQP_SYNTH_SIGNAL", s.get("feature_signal", 0.5))),
                     label_noise=float(os.environ.get("ADAQP_SYNTH_LABEL_NOISE", s.get("label_noise", 0.05))),
                     train_fraction=float(s["train_fraction"]), val_fraction=float(s["val_fraction"]),
                     seed=int(s.get("seed", 0)))
    return spec.scaled(scale) if scale != 1.0 else spec


@dataclass
class RawPartition:
    """What convert_partition (conversion.py:17-54) yields, as numpy arrays.

    Local node ids: [0, n_inner) inner nodes in global-id order, then halo nodes in
    ascending global id (hence grouped by owner).  `indptr/indices` is the dst-major CSR
    of all edges whose destination is an inner node (source ids are local ids)."""
    rank: int
    num_parts: int
    n_inner: int
    inner_start: int               # global id of local node 0
    starts: np.ndarray             # int64 [W + 1] global id range of every block
    indptr: np.ndarray             # int64 [n_inner + 1]
    indices: np.ndarray            # int32 [nnz]
    halo_gid: np.ndarray           # int64 [n_halo]
    halo_part: np.ndarray          # int32 [n_halo]
    feat: np.ndarray               # float32 [n_inner, F]
    label: np.ndarray              # int64 [n_inner] or float32 [n_inner, C] (multilabel)
    train_mask: np.ndarray
    val_mask: np.ndarray
    test_mask: np.ndarray
    in_degrees: Optional[np.ndarray] = None   # global degrees of all local nodes (inner + halo)
    out_degrees: Optional[np.ndarray] = None
    inner_gid: Optional[np.ndarray] = None    # int64 [n_inner]: each inner node's id in the dataset's own numbering

    @property
    def n_halo(self) -> int:
        return int(self.halo_gid.size)

    @property
    def inner_degrees(self) -> np.ndarray:
        """Global in-degree (= out-degree, symmetric graph) of the inner nodes: every
        in-edge of an inner node is in the partition."""
        return np.diff(self.indptr).astype(np.int64)


# ----------------------------------------------------------------------------- pieces
def block_starts(spec: SynthSpec) -> np.ndarray:
    W = spec.num_parts
    base, rem = divmod(spec.num_nodes, W)
    sizes = np.full(W, base, np.int64)
    sizes[:rem] += 1
    return np.concatenate([[0], np.cumsum(sizes)])


def _rng(spec: SynthSpec, *key) -> np.random.Generator:
    return np.random.default_rng(np.random.SeedSequence([spec.seed, *[int(k) for k in key]]))


def _perm(spec: SynthSpec, p: int, n: int) -> np.ndarray:
    return _rng(spec, 11, p).permutation(n)


class _PowerLaw:
    """Closed-form sampler of ranks i in [0, n) with P(i) ~ (i + i0)^(-alpha)."""

    def __init__(self, n: int, degree_exponent: float):
        self.n = n
        self.alpha = min(0.95, 1.0 / max(degree_exponent - 1.0, 1.05))
        self.i0 = max(4.0, 0.002 * n)
        e = 1.0 - self.alpha
        self.a0 = self.i0 ** e
        self.a1 = (n + self.i0) ** e
        self.inv = 1.0 / e

    def sample(self, rng: np.random.Generator, m: int) -> np.ndarray:
        u = rng.random(m)
        i = (u * (self.a1 - self.a0) + self.a0) ** self.inv - self.i0
        return np.minimum(i.astype(np.int64), self.n - 1)


def _edge_budget(spec: SynthSpec) -> Tuple[int, int]:
    """(intra undirected edges per block, cross undirected edges per block pair)."""
    W = spec.num_parts
    m_total = max((spec.num_edges - spec.num_nodes) // 2, 0)
    chi = spec.cross_fraction if W > 1 else 0.0
    m_cross = int(m_total * chi)
    m_intra = m_total - m_cross
    pairs = W * (W - 1) // 2
    return m_intra // W, (m_cross // pairs if pairs else 0)


def _intra_edges(spec: SynthSpec, p: int, n: int) -> Tuple[np.ndarray, np.ndarray]:
    m, _ = _edge_budget(spec)
    rng = _rng(spec, 21, p)
    pl = _PowerLaw(n, spec.degree_exponent)
    perm = _perm(spec, p, n)
    u = perm[pl.sample(rng, m)]
    v = perm[pl.sample(rng, m)]
    # homophily: re-draw v inside u's community for a share of the edges
    cs = max(int(spec.community_size), 1)
    if spec.homophily > 0 and n > cs:
        pick = rng.random(m) < spec.homophily
        k = int(pick.sum())
        base = (u[pick] // cs) * cs
        width = np.minimum(base + cs, n) - base
        v[pick] = base + (rng.random(k) * width).astype(np.int64)
    return u, v


def _cross_edges(spec: SynthSpec, p: int, q: int, n_p: int, n_q: int) -> Tuple[np.ndarray, np.ndarray]:
    """Undirected edges between blocks p < q as (local id in p, local id in q)."""
    assert p < q
    _, m = _edge_budget(spec)
    rng = _rng(spec, 31, p, q)
    # a METIS cut touches only part of a partition: cross edges end on the block's
    # `boundary_fraction` highest-weight nodes, the rest stay central (no halo in-neighbour)
    nb_p = max(1, int(n_p * spec.boundary_fraction))
    nb_q = max(1, int(n_q * spec.boundary_fraction))
    a = _perm(spec, p, n_p)[_PowerLaw(nb_p, spec.degree_exponent).sample(rng, m)]
    b = _perm(spec, q, n_q)[_PowerLaw(nb_q, spec.degree_exponent).sample(rng, m)]
    return a, b


def _node_data(spec: SynthSpec, p: int, n: int):
    rng = _rng(spec, 41, p)
    cs = max(int(spec.community_size), 1)
    C, F = spec.num_classes, spec.num_feats
    comm = np.arange(n) // cs
    cls = ((comm + 7 * p) % C).astype(np.int64)
    flip = rng.random(n) < spec.label_noise          # label noise
    cls[flip] = rng.integers(0, C, int(flip.sum()))
    cent = np.random.default_rng(spec.seed + 977).standard_normal((C, F)).astype(np.float32)
    feat = rng.standard_normal((n, F), dtype=np.float32)
    feat += np.float32(spec.feature_signal) * cent[cls]
    if spec.is_multilabel:
        label = np.zeros((n, C), np.float32)
        label[np.arange(n), cls] = 1.0
        extra = (cls + 1 + comm % 3) % C             # a second, correlated label
        label[np.arange(n), extra] = 1.0
    else:
        label = cls
    r = rng.random(n)
    train = r < spec.train_fraction
    val = (~train) & (r < spec.train_fraction + spec.val_fraction)
    test = ~(train | val)
    return feat, label, train, val, test


def build_raw_partition(spec: SynthSpec, rank: int) -> RawPartition:
    W = spec.num_parts
    starts = block_starts(spec)
    n = int(starts[rank + 1] - starts[rank])
    src_parts: List[np.ndarray] = []   # global src ids
    dst_parts: List[np.ndarray] = []   # local dst ids (inner)
    u, v = _intra_edges(spec, rank, n)
    g0 = int(starts[rank])
    src_parts += [u + g0, v + g0, np.arange(n, dtype=np.int64) + g0]     # both directions + self-loops
    dst_parts += [v, u, np.arange(n, dtype=np.int64)]
    for q in range(W):
        if q == rank:
            continue
        n_q = int(starts[q + 1] - starts[q])
        if rank < q:
            a, b = _cross_edges(spec, rank, q, n, n_q)
            mine, theirs = a, b
        else:
            a, b = _cross_edges(spec, q, rank, n_q, n)
            mine, theirs = b, a
        src_parts.append(theirs + int(starts[q]))    # halo -> inner (the inner -> halo twin lives on q)
        dst_parts.append(mine)
    src = np.concatenate(src_parts)
    dst = np.concatenate(dst_parts)
    inner = (src >= g0) & (src < g0 + n)
    halo_gid = np.unique(src[~inner])
    local_src = np.empty(src.size, np.int64)
    local_src[inner] = src[inner] - g0
    local_src[~inner] = n + np.searchsorted(halo_gid, src[~inner])
    n_all = n + halo_gid.size
    A = sp.coo_matrix((np.ones(src.size, np.int8), (dst, local_src)), shape=(n, n_all)).tocsr()
    A.sum_duplicates()                                # multi-edges collapse like a simple graph
    A.sort_indices()
    halo_part = (np.searchsorted(starts, halo_gid, side="right") - 1).astype(np.int32)
    feat, label, tr, va, te = _node_data(spec, rank, n)
    return RawPartition(rank=rank, num_parts=W, n_inner=n, inner_start=g0, starts=starts,
                        indptr=A.indptr.astype(np.int64), indices=A.indices.astype(np.int32),
                        halo_gid=halo_gid.astype(np.int64), halo_part=halo_part, feat=feat,
                        label=label, train_mask=tr, val_mask=va, test_mask=te,
                        inner_gid=g0 + np.arange(n, dtype=np.int64))


def attach_global_degrees(raw: RawPartition, inner_degrees_of_all: List[np.ndarray], starts: np.ndarray):
    """conversion.py:24-27: in/out degrees of the WHOLE graph for inner + halo nodes.
    `inner_degrees_of_all[q]` = RawPartition.inner_degrees of rank q (all-gathered)."""
    deg = np.empty(raw.n_inner + raw.n_halo, np.int64)
    deg[:raw.n_inner] = inner_degrees_of_all[raw.rank]
    for q in range(raw.num_parts):
        m = raw.halo_part == q
        if m.any():
            deg[raw.n_inner:][m] = inner_degrees_of_all[q][raw.halo_gid[m] - int(starts[q])]
    raw.in_degrees = deg
    raw.out_degrees = deg.copy()                      # symmetric graph (is_bidirected)
    return raw


def build_all_partitions(spec: SynthSpec) -> List[RawPartition]:
    """All ranks in one process (tests / single-process simulation)."""
    raws = [build_raw_partition(spec, r) for r in range(spec.num_parts)]
    degs = [r.inner_degrees for r in raws]
    starts = block_starts(spec)
    for r in raws:
        attach_global_degrees(r, degs, starts)
    return raws


def global_graph(spec: SynthSpec):
    """The generator's whole graph as one helper.dataset.GlobalGraph (symmetric CSR with self-loops, node data)
    and its planted blocks `part` -- the input graph_partition.py would see for a dataset of this shape."""
    from ..helper.dataset import GlobalGraph
    raws = build_all_partitions(spec)
    rows, cols = [], []
    for r in raws:
        rows.append(r.inner_start + np.repeat(np.arange(r.n_inner, dtype=np.int64), np.diff(r.indptr)))
        loc = r.indices.astype(np.int64)
        halo = r.halo_gid[np.maximum(loc - r.n_inner, 0)] if r.n_halo else loc
        cols.append(np.where(loc < r.n_inner, loc + r.inner_start, halo))
    n = spec.num_nodes
    row = np.concatenate(rows)
    A = sp.csr_matrix((np.ones(row.size, np.int8), (row, np.concatenate(cols))), shape=(n, n))
    A.sort_indices()
    cat = lambda f: np.concatenate([getattr(r, f) for r in raws])  # noqa: E731
    g = GlobalGraph(name=spec.name, indptr=A.indptr.astype(np.int64), indices=A.indices.astype(np.int32),
                    feat=cat("feat"), label=cat("label"), train_mask=cat("train_mask"), val_mask=cat("val_mask"),
                    test_mask=cat("test_mask"))
    return g, np.concatenate([np.full(r.n_inner, r.rank, np.int32) for r in raws])

"""GraphEngine ("Manager") and DecompGraph: per-rank graph state the hot path reads.

Public surface of AdaQP/manager/graphEngine.py:14-224 kept (constructor signature, `ctx`,
properties incl. the historical `num_remove` spelling, DecompGraph's copy-buffer API).
DGL is replaced by a CSR `LocalGraph`; partitions come from `<part_dir>/<dataset>/<W>part/
part<rank>.npz` when present, else from the seeded synthetic generator described by
config/<dataset>.yaml (manager/partition_synth.py).

GPU specifics: the central / marginal sub-graphs are row ranges of one CSR
([0, n_central) and [n_central, n_inner)), so the reference's copy buffers and
`torch.cat`s disappear from the data path (they stay available through the API); overlap
uses one side stream and CUDA events only -- no helper thread, no host synchronisation.
"""
from __future__ import annotations

import logging
import json
import os
from multiprocessing import Event
from multiprocessing.pool import ThreadPool
from typing import List, Optional, Tuple

import numpy as np
import torch
import yaml
from torch import Tensor

from ..communicator import Communicator as comm
from ..helper import BitType, DistGNNType
from ..util import Recorder, Timer
from .graph import LocalGraph
from .layout import RankLayout, prepare_rank
from .partition_synth import spec_from_config

logger = logging.getLogger("trainer")


class RowRange(object):
    """A destination-row window of a LocalGraph (what the reference builds as a separate
    central / marginal DGL graph, conversion.py:133-172)."""

    def __init__(self, graph: LocalGraph, begin: int, end: int):
        self.graph, self.begin, self.end = graph, int(begin), int(end)

    def num_nodes(self):
        return self.end - self.begin


class DecompGraph(object):
    def __init__(self, central_graph, marginal_geaph, src_marginal_idx: Tensor, src_central_idx: Tensor):
        self.central_graph = central_graph
        self.marginal_graph = marginal_geaph
        self._src_marginal_idx = src_marginal_idx
        self._src_central_idx = src_central_idx
        self.copy_buffers: List[Tuple[Tensor, Tensor]] = []

    @property
    def src_marginal_idx(self):
        return self._src_marginal_idx

    @property
    def src_central_idx(self):
        return self._src_central_idx

    @property
    def full(self) -> LocalGraph:
        return self.central_graph.graph

    def to(self, device: torch.device):
        self._src_central_idx = self._src_central_idx.to(device)
        self._src_marginal_idx = self._src_marginal_idx.to(device)

    def init_copy_buffers(self, feats_dim: int, hidden_dim: int, num_layers: int, device: torch.device):
        """graphEngine.py:39-44.  Not used by the fused path (rows are read in place);
        allocated lazily on first get_copy_buffers() to keep HBM free."""
        self._copy_spec = (feats_dim, hidden_dim, num_layers, device)

    def get_copy_buffers(self, layer: int) -> Tuple[Tensor, Tensor]:
        if not self.copy_buffers:
            f, h, n, dev = self._copy_spec
            m, c = self.src_marginal_idx.size(0), self.src_central_idx.size(0)
            for i in range(n):
                d = f if i == 0 else h
                self.copy_buffers.append((torch.zeros((m, d), device=dev), torch.zeros((c, d), device=dev)))
        return self.copy_buffers[layer]


def _load_config(dataset: str) -> dict:
    path = os.path.join(os.path.dirname(os.path.dirname(__file__)), "config", f"{dataset}.yaml")
    with open(path, "r") as f:
        return yaml.load(f, Loader=yaml.FullLoader)


_ARRAY_FIELDS = ("indptr", "indices", "in_degrees", "out_degrees", "feat", "label", "train_mask", "val_mask",
                 "test_mask", "total_send_idx", "src_marginal_idx", "src_central_idx")
_SCALAR_FIELDS = ("rank", "world_size", "n_central", "n_marginal", "n_inner", "n_halo", "is_bidirected")


def save_rank_layout(layout: RankLayout, part_dir: str, dataset: str) -> str:
    """Write one rank's prepared layout where load_rank_layout looks for it
    (`<part_dir>/<dataset>/<W>part/part<rank>.npz`): the ingest point for real partitions, e.g. the
    output of tools/convert_dgl_partition.py run where DGL is installed.  Plain ndarrays plus a JSON
    header only -- nothing in the file is unpickled on load."""
    d = f"{part_dir}/{dataset}/{layout.world_size}part"
    os.makedirs(d, exist_ok=True)
    path = f"{d}/part{layout.rank}.npz"
    arrays = {k: np.ascontiguousarray(getattr(layout, k)) for k in _ARRAY_FIELDS}
    if layout.inner_gid is not None:
        arrays["inner_gid"] = np.ascontiguousarray(layout.inner_gid, np.int64)
    header = {k: (bool(getattr(layout, k)) if k == "is_bidirected" else int(getattr(layout, k))) for k in _SCALAR_FIELDS}
    header["send_idx"] = {str(p): [int(lo), int(hi)] for p, (lo, hi) in layout.send_idx.items()}
    header["recv_peers"] = [int(p) for p in layout.recv_idx]
    header["score_peers"] = [int(p) for p in layout.scores]
    for p, v in layout.recv_idx.items():
        arrays[f"recv_idx_{int(p)}"] = np.ascontiguousarray(v)
    for p, (fw, bw) in layout.scores.items():
        arrays[f"score_fwd_{int(p)}"] = np.ascontiguousarray(fw)
        arrays[f"score_bwd_{int(p)}"] = np.ascontiguousarray(bw)
    arrays["header_json"] = np.frombuffer(json.dumps(header).encode("utf-8"), dtype=np.uint8)
    np.savez_compressed(path, **arrays)
    return path


def read_rank_layout(path: str) -> RankLayout:
    z = np.load(path, allow_pickle=False)
    h = json.loads(bytes(z["header_json"]).decode("utf-8"))
    kw = {k: z[k] for k in _ARRAY_FIELDS}
    kw.update({k: h[k] for k in _SCALAR_FIELDS})
    kw["send_idx"] = {int(p): (int(v[0]), int(v[1])) for p, v in h["send_idx"].items()}
    kw["recv_idx"] = {int(p): z[f"recv_idx_{int(p)}"] for p in h["recv_peers"]}
    kw["scores"] = {int(p): (z[f"score_fwd_{int(p)}"], z[f"score_bwd_{int(p)}"]) for p in h["score_peers"]}
    kw["inner_gid"] = z["inner_gid"] if "inner_gid" in z.files else None      # optional: older files lack it
    return RankLayout(**kw)


def load_rank_layout(part_dir: str, dataset: str, model_type: DistGNNType) -> RankLayout:
    rank, W = comm.get_rank(), comm.get_world_size()
    path = f"{part_dir}/{dataset}/{W}part/part{rank}.npz"
    if os.path.exists(path):
        return read_rank_layout(path)
    # No partition files: the DGL-free synthetic generator is an explicit opt-in, so that a mistyped
    # partition path cannot silently train on random data under the real dataset's name.
    if os.environ.get("ADAQP_SYNTHETIC", "0") != "1":
        raise FileNotFoundError(
            f"no partition file {path}. Partition a dataset with graph_partition.py, convert DGL partitions with "
            f"tools/convert_dgl_partition.py, or set "
            f"ADAQP_SYNTHETIC=1 to train on synthetic partitions of the dataset's shape (config `synthetic:`).")
    scale = float(os.environ.get("ADAQP_SYNTH_SCALE", "1.0"))
    spec = spec_from_config(_load_config(dataset), W, scale)
    if rank == 0:
        logger.warning(f"<no partition files under {part_dir}/{dataset}/{W}part: SYNTHETIC partitions "
                       f"N={spec.num_nodes} E={spec.num_edges} W={W} seed={spec.seed} (ADAQP_SYNTHETIC=1)>")
    return prepare_rank(spec, rank, model_type, comm.gather_all)


class GraphEngine(object):
    ctx: "GraphEngine" = None

    def __init__(self, epoches: int, part_dir, dataset, msg_precision_type: str, model_type: DistGNNType,
                 use_parallel=False, layout: RankLayout = None):
        L = layout if layout is not None else load_rank_layout(part_dir, dataset, model_type)
        self.layout = L
        self._is_bidirected = L.is_bidirected
        if not L.is_bidirected:
            # The reference builds bwd_graph = dgl.reverse(graph, copy_ndata=False) (graphEngine.py:135-147): the reversed
            # graph carries no 'in_degrees' / 'out_degrees', which its backward aggregation reads (ops.py:23-24,50), and the
            # reverse of the LOCAL graph has no edge back to the owners of halo sources, so their gradient share would be
            # dropped.  Its four datasets are symmetrised (helper/partition.py:58-60); directed input is refused up front.
            raise NotImplementedError("directed (non-symmetrised) partitions are not supported: in_degrees != out_degrees; "
                                      "symmetrise the graph before partitioning as the reference's helper/partition.py does")
        self._use_parallel = use_parallel
        if msg_precision_type == "full":
            self._bit_type = BitType.FULL
        elif msg_precision_type == "quant":
            self._bit_type = BitType.QUANT
        else:
            raise NotImplementedError(f"only full and quant are supported now, {msg_precision_type} is undifined.")
        self._num_remove, self._num_inner = L.n_halo, L.n_inner
        self._num_marginal, self._num_central = L.n_marginal, L.n_central
        self._device = comm.ctx.device
        dev = self._device
        self._send_idx = dict(L.send_idx)
        self._recv_idx = {p: torch.from_numpy(v) for p, v in L.recv_idx.items()}
        self._scores = {p: (torch.from_numpy(s[0]), torch.from_numpy(s[1])) for p, s in L.scores.items()}
        self._total_send_idx = torch.from_numpy(L.total_send_idx).to(dev)
        self.feats = torch.from_numpy(L.feat).to(dev)
        self.labels = torch.from_numpy(L.label).to(dev)
        self.train_mask = torch.nonzero(torch.from_numpy(L.train_mask)).squeeze(1).to(dev)
        self.val_mask = torch.nonzero(torch.from_numpy(L.val_mask)).squeeze(1).to(dev)
        self.test_mask = torch.nonzero(torch.from_numpy(L.test_mask)).squeeze(1).to(dev)
        if dev.type == "cuda":
            self.local_graph = LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, dev)
        else:
            from .graph_cpu import CpuGraph          # gloo plumbing mode only
            self.local_graph = CpuGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo)
        if use_parallel:
            self.graph = DecompGraph(RowRange(self.local_graph, 0, L.n_central),
                                     RowRange(self.local_graph, L.n_central, L.n_inner),
                                     torch.from_numpy(L.src_marginal_idx).to(dev),
                                     torch.from_numpy(L.src_central_idx).to(dev))
            self._init_stream_ctx()
        else:
            self.graph = self.local_graph
        self.bwd_graph = self.graph          # graphEngine.py:141-147 (bidirected)
        self.timer = Timer(device=dev)
        self.recorder = Recorder(epoches)
        self._agg_type: str = None
        # index of the model's output layer (num_layers - 1), set by the Trainer: the backward aggregation of that
        # layer skips the all-zero gradient rows of the nodes outside the train mask (ops._live_rows); None = off
        self.top_layer: Optional[int] = None
        GraphEngine.ctx = self

    def __repr__(self):
        return (f"<GraphEngine(rank: {comm.get_rank()}, remote nodes: {self.num_remove} central nodes: "
                f"{self.num_central}, marginal nodes: {self.num_marginal})>")

    def _init_stream_ctx(self):
        """graphEngine.py:122-132.  The exchange kernels run on `marginal_stream`; ordering with
        the default stream is by CUDA events only.  The CPU events exist for API parity."""
        if self._device.type == "cuda":
            self.marginal_stream = torch.cuda.Stream(device=self._device)
            self.quant_cuda_event = torch.cuda.Event()
            self.comp_cuda_event = torch.cuda.Event()
        else:
            self.marginal_stream = self.quant_cuda_event = self.comp_cuda_event = None
        self.quant_cpu_event = Event()
        self.comp_cpu_event = Event()
        # helper thread of the reference (graphEngine.py:131); only the gloo plumbing transport uses it -- on p2p the
        # exchange is a kernel on marginal_stream and needs no thread
        self.marginal_pool = ThreadPool(processes=1) if self._device.type != "cuda" else None
        self.marginal_pool = None

    # ---- read-only accessors of the reference (graphEngine.py:169-224), generated below ------------------
    @property
    def agg_type(self):
        assert self._agg_type is not None, "please set the aggregator type first."
        return self._agg_type

    @agg_type.setter
    def agg_type(self, agg_type: str):
        self._agg_type = agg_type


def _readonly(attr: str):
    return property(lambda self: getattr(self, attr))


# public name -> private field; `num_remove` is the reference's (historical) spelling of num_remote and is
# what op_util.py:147 reads, so it is kept verbatim, with `num_remote` as an alias
for _public, _private in {"device": "_device", "is_bidirected": "_is_bidirected", "use_parallel": "_use_parallel",
                          "bit_type": "_bit_type", "num_remove": "_num_remove", "num_remote": "_num_remove",
                          "num_inner": "_num_inner", "num_marginal": "_num_marginal", "num_central": "_num_central",
                          "send_idx": "_send_idx", "recv_idx": "_recv_idx", "scores": "_scores",
                          "total_send_idx": "_total_send_idx"}.items():
    setattr(GraphEngine, _public, _readonly(_private))

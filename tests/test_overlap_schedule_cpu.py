"""What the distributed aggregations enqueue, in order, on the CPU.

The autograd Functions of model/ops.py are driven through their static forward / backward on small CPU tensors
while everything below ops.py records what it is asked to do:

  * the library (`_lib.load()`): each entry point with its destination rows, its part of the two-pass marginal
    schedule (read from the segment pointers), whether it was given the halo rows, row liveness or a row list, and
    its stream;
  * the p2p exchange (`comm.ctx.comm_buffer.p2p`): posts, receives and releases per key and stream;
  * the streams and events (`torch.cuda.current_stream`, `torch.cuda.Event`, `Tensor.record_stream`);
  * the timer on `engine.ctx`: region begin / end with its stream, and each exposed-wait record.

The expected traces are literals.  They pin the exchange-and-overlap schedule (which rows run before the wait for
the halo and which after, on which stream, inside which timer region) so a change to how ops.py is organised can be
checked to enqueue exactly the same work.  The exchanges are fp32: the quantised exchange draws its Philox offsets
from the CUDA generators, which a CPU run does not have; its schedule is the same, only the region of the exchange is
named `{name}_quantization` instead.
"""
import os
import sys
from contextlib import contextmanager
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adaqp_b200 import _lib  # noqa: E402
from adaqp_b200.assigner import Assigner  # noqa: E402
from adaqp_b200.communicator import Communicator  # noqa: E402
from adaqp_b200.helper import BitType  # noqa: E402
from adaqp_b200.manager import GraphEngine  # noqa: E402
from adaqp_b200.manager.graph import LocalGraph  # noqa: E402
from adaqp_b200.manager.graphEngine import DecompGraph, RowRange  # noqa: E402
from adaqp_b200.model import ops  # noqa: E402

# argument positions of the traced entry points: (row_begin, row_end, seg_start, seg_end, halo, live, n_list);
# None where the entry point has no such argument
ARGS = {
    "adaqp_spmm_csr_seg_f32": (14, 15, 1, 2, 7, 19, 21),
    "adaqp_row_live_f32": (None, None, None, None, None, None, None),
    "adaqp_appnp_prop_f32": (19, 20, 1, 2, 7, None, None),
    "adaqp_gat_scores_f32": (None, None, None, None, None, None, None),
    "adaqp_gat_fwd_f32": (12, 13, None, None, 5, None, None),
    "adaqp_gat_bwd_f32": (19, 20, None, None, 5, None, None),
    "adaqp_gatv2_fwd_f32": (12, 13, None, None, 5, None, None),
    "adaqp_gatv2_bwd_inner_f32": (20, 21, None, None, 14, None, None),
    "adaqp_gatv2_bwd_halo_f32": (13, 14, None, None, None, None, None),
    "adaqp_sage_pool_fwd_f32": (10, 11, 1, 2, 7, None, None),
    "adaqp_sage_pool_bwd_f32": (15, 16, 1, 2, 8, None, None),
}

N_INNER, N_CENTRAL, N_HALO, F, HEADS = 6, 3, 3, 8, 2
# rows 0-2 read local rows only (central), rows 3-5 read halo rows 6-8 too (marginal); columns ascending
INDPTR = np.array([0, 2, 3, 5, 7, 10, 12])
INDICES = np.array([1, 2, 0, 0, 1, 2, 6, 3, 7, 8, 4, 6])


class Harness:
    def __init__(self, use_parallel: bool, n_central: int = N_CENTRAL):
        self.trace = []
        self.n_events = 0
        self.main = self.stream("main", 1)
        self.side = self.stream("side", 2) if use_parallel else None
        self.names = {1: "main", 2: "side"}
        self.width = {}
        lg = LocalGraph(INDPTR, INDICES, np.full(N_INNER + N_HALO, 2), np.full(N_INNER + N_HALO, 2), N_INNER, N_HALO,
                        "cpu")
        self.graph = (DecompGraph(RowRange(lg, 0, n_central), RowRange(lg, n_central, N_INNER),
                                  torch.arange(n_central, N_INNER), torch.arange(n_central)) if use_parallel else lg)
        self.eng = SimpleNamespace(
            use_parallel=use_parallel, num_inner=N_INNER, num_central=n_central, marginal_stream=self.side,
            timer=self.timer(), bit_type=BitType.FULL, top_layer=1, agg_type="mean", _agg_type="mean",
            feats=torch.zeros(N_INNER, F), graph=self.graph, bwd_graph=self.graph,
            pool_want=torch.zeros(len(INDICES), dtype=torch.int32),
            gatv2_halo=(torch.tensor([0, 2, 3, 4]), torch.tensor([3, 5, 4, 4], dtype=torch.int32)),
            gatv2_fold=(torch.tensor([0, 0, 0, 1, 2, 3, 3]), torch.tensor([0, 1, 2], dtype=torch.int32)))
        self.comm = SimpleNamespace(transport="p2p", comm_buffer=SimpleNamespace(p2p=self.exchange()))

    def log(self, *words):
        self.trace.append(" ".join(str(w) for w in words))

    def at(self, stream):
        return (stream if stream is not None else self.main).name

    def stream(self, name, handle):
        h = self

        class Stream:
            def __init__(self):
                self.name, self.cuda_stream = name, handle

            def wait_event(self, ev):
                h.log("wait", self.name, ev.label)
        return Stream()

    def event_class(self):
        h = self

        class Event:
            def __init__(self, enable_timing=False, **_):
                self.label = f"e{h.n_events}" + (" timing" if enable_timing else "")
                h.n_events += 1

            def record(self, stream=None):
                h.log("event", self.label, "@" + h.at(stream))
        return Event

    def timer(self):
        h = self

        class Timer:
            @contextmanager
            def record_events(self, name, stream=None):
                h.log("begin", name, "@" + h.at(stream))
                yield
                h.log("end", name, "@" + h.at(stream))

            def record_exposed(self, name, compute_done, data_ready):
                h.log("exposed", name, compute_done.label, data_ready.label)
        return Timer()

    def exchange(self):
        h = self

        class Exchange:
            transport = "p2p"

            def post_send_fp(self, key, x, gathered=False, stream=None):
                h.width[key] = int(x.shape[1])
                h.log("post", key, tuple(x.shape), "@" + h.at(stream))
                return 1

            def complete_recv_fp(self, key, stream=None):
                h.log("recv", key, "@" + h.at(stream))
                return torch.zeros(N_HALO, h.width[key])

            def release_fp(self, key, stream=None):
                h.log("release", key, "@" + h.at(stream))
        return Exchange()

    def library(self):
        h = self

        class Library:
            def __getattr__(self, name):
                assert name in ARGS, f"untraced library entry point {name}"

                def call(*a):
                    assert len(a) == len(_lib.SYMBOLS[name][1]), (name, len(a))
                    rb, re, s0, s1, halo, live, n_list = (a[i] if i is not None else None for i in ARGS[name])
                    words = [name[len("adaqp_"):]]
                    if rb is not None:
                        words.append(f"[{rb},{re})")
                    if s0 is not None or s1 is not None:
                        words.append("part=" + ("halo" if s0 is not None else "local"))
                    if halo is not None:
                        words.append("halo")
                    if live is not None:
                        words.append("live")
                    if n_list:
                        words.append(f"rows={n_list}")
                    h.log("lib", *words, "@" + h.names[a[-1]])
                    return 0
                return call
        return Library()

    @contextmanager
    def installed(self, monkeypatch, split: bool):
        h = self
        monkeypatch.setattr(_lib, "load", self.library)
        monkeypatch.setattr(torch.cuda, "current_stream", lambda device=None: h.main)
        monkeypatch.setattr(torch.cuda, "Event", self.event_class())
        monkeypatch.setattr(torch.Tensor, "record_stream", lambda t, s: h.log("record_stream", tuple(t.shape), s.name),
                            raising=False)
        new_zeros = torch.Tensor.new_zeros

        def zeros(t, *a, **k):               # the zero-fill of the rows a row list leaves out
            out = new_zeros(t, *a, **k)
            h.log("zeros", tuple(out.shape), "@main")
            return out
        monkeypatch.setattr(torch.Tensor, "new_zeros", zeros)
        # the liveness and row-list paths are device-path features; the tensors here stand in for device tensors
        monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda t: True), raising=False)
        monkeypatch.setattr(Communicator, "ctx", self.comm)
        monkeypatch.setattr(GraphEngine, "ctx", self.eng)
        monkeypatch.setattr(Assigner, "ctx", None)
        monkeypatch.setenv("ADAQP_MARGINAL_SPLIT", "1" if split else "0")
        monkeypatch.setenv("ADAQP_SKIP_ZERO_ROWS", "1")
        monkeypatch.setattr(ops, "_SPLIT", None)
        monkeypatch.setattr(ops, "_SKIP", None)
        yield


class Ctx:
    """Stands in for the autograd context of a Function."""

    def save_for_backward(self, *t):
        self.saved_tensors = t


def x(rows=N_INNER, cols=F):
    return torch.arange(rows * cols, dtype=torch.float32).reshape(rows, cols) / 7.0


# ---------------------------------------------------------------- scenarios: each returns nothing, the trace is the result
def conv_step(cls):
    def run(h):
        ctx = Ctx()
        cls.forward(ctx, x(), h.graph, 1, True)
        h.log("--")
        cls.backward(ctx, x())                    # layer 1 is the top layer: row liveness
        h.log("--")
        ctx = Ctx()
        cls.forward(ctx, x(), h.graph, 0, False)  # evaluation: test0, every row
        h.log("--")
        cls.backward(ctx, x())                    # a lower layer: no liveness
    return run


def conv_loss_rows(cls, rows):
    def run(h):
        with ops.loss_rows(torch.tensor(rows)):
            cls.forward(Ctx(), x(), h.graph, 1, True)
            h.log("--")
            cls.forward(Ctx(), x(), h.graph, 0, True)   # not the top layer: every row
    return run


def gat_step(h):
    ctx = Ctx()
    a = torch.ones(HEADS, F // HEADS)
    ops.DistAggGAT.forward(ctx, x(), a, a, h.graph, 0, True, HEADS)
    h.log("--")
    ops.DistAggGAT.backward(ctx, x())


def gatv2_step(h):
    ctx = Ctx()
    ops.DistAggGATv2.forward(ctx, x(), x(), torch.ones(HEADS, F // HEADS), h.graph, 1, True, HEADS)
    h.log("--")
    ops.DistAggGATv2.backward(ctx, x())


def sage_pool_step(h):
    ctx = Ctx()
    ops.DistAggSAGEPool.forward(ctx, x(), h.graph, 0, True)
    h.log("--")
    ops.DistAggSAGEPool.backward(ctx, x())


def appnp_step(h):
    ctx = Ctx()
    ops.DistAPPNPProp.forward(ctx, x(), h.graph, 2, 0.1, True)
    h.log("--")
    ops.DistAPPNPProp.backward(ctx, x())


def gcnii_step(h):
    ctx = Ctx()
    ops.DistGCNIIProp.forward(ctx, x(), x(), h.graph, 0.1, True, 1)
    h.log("--")
    ops.DistGCNIIProp.backward(ctx, x())


SCENARIOS = {
    "gcn": conv_step(ops.DistAggConv),
    "sage": conv_step(ops.DistAggSAGE),
    "gcn_loss_rows": conv_loss_rows(ops.DistAggConv, [1, 4, 5]),
    "gcn_loss_rows_marginal_only": conv_loss_rows(ops.DistAggConv, [3, 5]),
    "gcn_loss_rows_central_only": conv_loss_rows(ops.DistAggConv, [0, 2]),
    "sage_loss_rows": conv_loss_rows(ops.DistAggSAGE, [1, 4, 5]),
    "gat": gat_step,
    "gatv2": gatv2_step,
    "sage_pool": sage_pool_step,
    "appnp": appnp_step,
    "gcnii": gcnii_step,
}
# GraphSAGE enqueues what GCN does: only the norms the kernel reads differ
SAME_AS = {"sage": "gcn", "sage_loss_rows": "gcn_loss_rows"}
MODES = {"serial": (False, True), "overlap": (True, True), "overlap_nosplit": (True, False)}


def run_scenario(monkeypatch, scenario: str, mode: str, n_central: int = N_CENTRAL):
    use_parallel, split = MODES[mode]
    h = Harness(use_parallel, n_central)
    with h.installed(monkeypatch, split):
        SCENARIOS[scenario](h)
    return h.trace


EXPECTED = {
    ("appnp", "overlap"): """
        event e0 @main
        wait side e0
        begin forward0_communication @side
        post forward0 (6, 8) @side
        recv forward0 @side
        end forward0_communication @side
        event e1 timing @side
        begin forward0_central_aggregation @main
        lib appnp_prop_f32 [0,3) @main
        end forward0_central_aggregation @main
        begin forward0_marginal_aggregation_local @main
        lib appnp_prop_f32 [3,6) part=local @main
        end forward0_marginal_aggregation_local @main
        event e2 timing @main
        exposed forward0 e2 timing e1 timing
        wait main e1 timing
        begin forward0_marginal_aggregation_halo @main
        lib appnp_prop_f32 [3,6) part=halo halo @main
        end forward0_marginal_aggregation_halo @main
        release forward0 @main
        record_stream (6, 8) side
        event e3 @main
        wait side e3
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e4 timing @side
        begin forward1_central_aggregation @main
        lib appnp_prop_f32 [0,3) @main
        end forward1_central_aggregation @main
        begin forward1_marginal_aggregation_local @main
        lib appnp_prop_f32 [3,6) part=local @main
        end forward1_marginal_aggregation_local @main
        event e5 timing @main
        exposed forward1 e5 timing e4 timing
        wait main e4 timing
        begin forward1_marginal_aggregation_halo @main
        lib appnp_prop_f32 [3,6) part=halo halo @main
        end forward1_marginal_aggregation_halo @main
        release forward1 @main
        record_stream (6, 8) side
        --
        event e6 @main
        wait side e6
        begin backward1_communication @side
        post backward1 (6, 8) @side
        recv backward1 @side
        end backward1_communication @side
        event e7 timing @side
        begin backward1_central_aggregation @main
        lib appnp_prop_f32 [0,3) @main
        end backward1_central_aggregation @main
        begin backward1_marginal_aggregation_local @main
        lib appnp_prop_f32 [3,6) part=local @main
        end backward1_marginal_aggregation_local @main
        event e8 timing @main
        exposed backward1 e8 timing e7 timing
        wait main e7 timing
        begin backward1_marginal_aggregation_halo @main
        lib appnp_prop_f32 [3,6) part=halo halo @main
        end backward1_marginal_aggregation_halo @main
        release backward1 @main
        record_stream (6, 8) side
        event e9 @main
        wait side e9
        begin backward0_communication @side
        post backward0 (6, 8) @side
        recv backward0 @side
        end backward0_communication @side
        event e10 timing @side
        begin backward0_central_aggregation @main
        lib appnp_prop_f32 [0,3) @main
        end backward0_central_aggregation @main
        begin backward0_marginal_aggregation_local @main
        lib appnp_prop_f32 [3,6) part=local @main
        end backward0_marginal_aggregation_local @main
        event e11 timing @main
        exposed backward0 e11 timing e10 timing
        wait main e10 timing
        begin backward0_marginal_aggregation_halo @main
        lib appnp_prop_f32 [3,6) part=halo halo @main
        end backward0_marginal_aggregation_halo @main
        release backward0 @main
        record_stream (6, 8) side
    """,
    ("appnp", "overlap_nosplit"): """
        event e0 @main
        wait side e0
        begin forward0_communication @side
        post forward0 (6, 8) @side
        recv forward0 @side
        end forward0_communication @side
        event e1 timing @side
        begin forward0_central_aggregation @main
        lib appnp_prop_f32 [0,3) @main
        end forward0_central_aggregation @main
        event e2 timing @main
        exposed forward0 e2 timing e1 timing
        wait main e1 timing
        begin forward0_marginal_aggregation @main
        lib appnp_prop_f32 [3,6) halo @main
        end forward0_marginal_aggregation @main
        release forward0 @main
        record_stream (6, 8) side
        event e3 @main
        wait side e3
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e4 timing @side
        begin forward1_central_aggregation @main
        lib appnp_prop_f32 [0,3) @main
        end forward1_central_aggregation @main
        event e5 timing @main
        exposed forward1 e5 timing e4 timing
        wait main e4 timing
        begin forward1_marginal_aggregation @main
        lib appnp_prop_f32 [3,6) halo @main
        end forward1_marginal_aggregation @main
        release forward1 @main
        record_stream (6, 8) side
        --
        event e6 @main
        wait side e6
        begin backward1_communication @side
        post backward1 (6, 8) @side
        recv backward1 @side
        end backward1_communication @side
        event e7 timing @side
        begin backward1_central_aggregation @main
        lib appnp_prop_f32 [0,3) @main
        end backward1_central_aggregation @main
        event e8 timing @main
        exposed backward1 e8 timing e7 timing
        wait main e7 timing
        begin backward1_marginal_aggregation @main
        lib appnp_prop_f32 [3,6) halo @main
        end backward1_marginal_aggregation @main
        release backward1 @main
        record_stream (6, 8) side
        event e9 @main
        wait side e9
        begin backward0_communication @side
        post backward0 (6, 8) @side
        recv backward0 @side
        end backward0_communication @side
        event e10 timing @side
        begin backward0_central_aggregation @main
        lib appnp_prop_f32 [0,3) @main
        end backward0_central_aggregation @main
        event e11 timing @main
        exposed backward0 e11 timing e10 timing
        wait main e10 timing
        begin backward0_marginal_aggregation @main
        lib appnp_prop_f32 [3,6) halo @main
        end backward0_marginal_aggregation @main
        release backward0 @main
        record_stream (6, 8) side
    """,
    ("appnp", "serial"): """
        begin forward0_communication @main
        post forward0 (6, 8) @main
        recv forward0 @main
        end forward0_communication @main
        begin forward0_full_aggregation @main
        lib appnp_prop_f32 [0,6) halo @main
        end forward0_full_aggregation @main
        release forward0 @main
        begin forward1_communication @main
        post forward1 (6, 8) @main
        recv forward1 @main
        end forward1_communication @main
        begin forward1_full_aggregation @main
        lib appnp_prop_f32 [0,6) halo @main
        end forward1_full_aggregation @main
        release forward1 @main
        --
        begin backward1_communication @main
        post backward1 (6, 8) @main
        recv backward1 @main
        end backward1_communication @main
        begin backward1_full_aggregation @main
        lib appnp_prop_f32 [0,6) halo @main
        end backward1_full_aggregation @main
        release backward1 @main
        begin backward0_communication @main
        post backward0 (6, 8) @main
        recv backward0 @main
        end backward0_communication @main
        begin backward0_full_aggregation @main
        lib appnp_prop_f32 [0,6) halo @main
        end backward0_full_aggregation @main
        release backward0 @main
    """,
    ("gat", "overlap"): """
        lib gat_scores_f32 @main
        event e0 @main
        wait side e0
        begin forward0_communication @side
        post attn_fwd0 (6, 2) @side
        post forward0 (6, 8) @side
        recv forward0 @side
        recv attn_fwd0 @side
        end forward0_communication @side
        event e1 timing @side
        begin forward0_central_aggregation @main
        lib gat_fwd_f32 [0,3) @main
        end forward0_central_aggregation @main
        event e2 timing @main
        exposed forward0 e2 timing e1 timing
        wait main e1 timing
        begin forward0_marginal_aggregation @main
        lib gat_fwd_f32 [3,6) halo @main
        end forward0_marginal_aggregation @main
        release forward0 @main
        release attn_fwd0 @main
        record_stream (6, 8) side
        record_stream (6, 2) side
        --
        event e3 @main
        wait side e3
        begin backward0_communication @side
        post attn_bwd0 (6, 6) @side
        post backward0 (6, 8) @side
        recv backward0 @side
        recv attn_bwd0 @side
        end backward0_communication @side
        event e4 timing @side
        begin backward0_central_aggregation @main
        lib gat_bwd_f32 [0,3) @main
        end backward0_central_aggregation @main
        event e5 timing @main
        exposed backward0 e5 timing e4 timing
        wait main e4 timing
        begin backward0_marginal_aggregation @main
        lib gat_bwd_f32 [3,6) halo @main
        end backward0_marginal_aggregation @main
        release backward0 @main
        release attn_bwd0 @main
        record_stream (6, 8) side
        record_stream (6, 6) side
    """,
    ("gat", "overlap_nosplit"): """
        lib gat_scores_f32 @main
        event e0 @main
        wait side e0
        begin forward0_communication @side
        post attn_fwd0 (6, 2) @side
        post forward0 (6, 8) @side
        recv forward0 @side
        recv attn_fwd0 @side
        end forward0_communication @side
        event e1 timing @side
        begin forward0_central_aggregation @main
        lib gat_fwd_f32 [0,3) @main
        end forward0_central_aggregation @main
        event e2 timing @main
        exposed forward0 e2 timing e1 timing
        wait main e1 timing
        begin forward0_marginal_aggregation @main
        lib gat_fwd_f32 [3,6) halo @main
        end forward0_marginal_aggregation @main
        release forward0 @main
        release attn_fwd0 @main
        record_stream (6, 8) side
        record_stream (6, 2) side
        --
        event e3 @main
        wait side e3
        begin backward0_communication @side
        post attn_bwd0 (6, 6) @side
        post backward0 (6, 8) @side
        recv backward0 @side
        recv attn_bwd0 @side
        end backward0_communication @side
        event e4 timing @side
        begin backward0_central_aggregation @main
        lib gat_bwd_f32 [0,3) @main
        end backward0_central_aggregation @main
        event e5 timing @main
        exposed backward0 e5 timing e4 timing
        wait main e4 timing
        begin backward0_marginal_aggregation @main
        lib gat_bwd_f32 [3,6) halo @main
        end backward0_marginal_aggregation @main
        release backward0 @main
        release attn_bwd0 @main
        record_stream (6, 8) side
        record_stream (6, 6) side
    """,
    ("gat", "serial"): """
        lib gat_scores_f32 @main
        begin forward0_communication @main
        post attn_fwd0 (6, 2) @main
        post forward0 (6, 8) @main
        recv forward0 @main
        recv attn_fwd0 @main
        end forward0_communication @main
        begin forward0_full_aggregation @main
        lib gat_fwd_f32 [0,6) halo @main
        end forward0_full_aggregation @main
        release forward0 @main
        release attn_fwd0 @main
        --
        begin backward0_communication @main
        post attn_bwd0 (6, 6) @main
        post backward0 (6, 8) @main
        recv backward0 @main
        recv attn_bwd0 @main
        end backward0_communication @main
        begin backward0_full_aggregation @main
        lib gat_bwd_f32 [0,6) halo @main
        end backward0_full_aggregation @main
        release backward0 @main
        release attn_bwd0 @main
    """,
    ("gatv2", "overlap"): """
        event e0 @main
        wait side e0
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e1 timing @side
        begin forward1_central_aggregation @main
        lib gatv2_fwd_f32 [0,3) @main
        end forward1_central_aggregation @main
        event e2 timing @main
        exposed forward1 e2 timing e1 timing
        wait main e1 timing
        begin forward1_marginal_aggregation @main
        lib gatv2_fwd_f32 [3,6) halo @main
        end forward1_marginal_aggregation @main
        release forward1 @main
        record_stream (6, 8) side
        --
        lib gatv2_bwd_halo_f32 [0,3) @main
        event e3 @main
        wait side e3
        begin backward1_communication @side
        post push1 (3, 8) @side
        recv push1 @side
        end backward1_communication @side
        event e4 timing @side
        begin backward1_central_aggregation @main
        lib gatv2_bwd_inner_f32 [0,3) @main
        end backward1_central_aggregation @main
        event e5 timing @main
        exposed backward1 e5 timing e4 timing
        wait main e4 timing
        begin backward1_marginal_aggregation @main
        lib gatv2_bwd_inner_f32 [3,6) halo @main
        end backward1_marginal_aggregation @main
        release push1 @main
        record_stream (3, 8) side
    """,
    ("gatv2", "overlap_nosplit"): """
        event e0 @main
        wait side e0
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e1 timing @side
        begin forward1_central_aggregation @main
        lib gatv2_fwd_f32 [0,3) @main
        end forward1_central_aggregation @main
        event e2 timing @main
        exposed forward1 e2 timing e1 timing
        wait main e1 timing
        begin forward1_marginal_aggregation @main
        lib gatv2_fwd_f32 [3,6) halo @main
        end forward1_marginal_aggregation @main
        release forward1 @main
        record_stream (6, 8) side
        --
        lib gatv2_bwd_halo_f32 [0,3) @main
        event e3 @main
        wait side e3
        begin backward1_communication @side
        post push1 (3, 8) @side
        recv push1 @side
        end backward1_communication @side
        event e4 timing @side
        begin backward1_central_aggregation @main
        lib gatv2_bwd_inner_f32 [0,3) @main
        end backward1_central_aggregation @main
        event e5 timing @main
        exposed backward1 e5 timing e4 timing
        wait main e4 timing
        begin backward1_marginal_aggregation @main
        lib gatv2_bwd_inner_f32 [3,6) halo @main
        end backward1_marginal_aggregation @main
        release push1 @main
        record_stream (3, 8) side
    """,
    ("gatv2", "serial"): """
        begin forward1_communication @main
        post forward1 (6, 8) @main
        recv forward1 @main
        end forward1_communication @main
        begin forward1_full_aggregation @main
        lib gatv2_fwd_f32 [0,6) halo @main
        end forward1_full_aggregation @main
        release forward1 @main
        --
        lib gatv2_bwd_halo_f32 [0,3) @main
        begin backward1_communication @main
        post push1 (3, 8) @main
        recv push1 @main
        end backward1_communication @main
        begin backward1_full_aggregation @main
        lib gatv2_bwd_inner_f32 [0,6) halo @main
        end backward1_full_aggregation @main
        release push1 @main
    """,
    ("gcn", "overlap"): """
        event e0 @main
        wait side e0
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e1 timing @side
        begin forward1_central_aggregation @main
        lib spmm_csr_seg_f32 [0,3) @main
        end forward1_central_aggregation @main
        begin forward1_marginal_aggregation_local @main
        lib spmm_csr_seg_f32 [3,6) part=local @main
        end forward1_marginal_aggregation_local @main
        event e2 timing @main
        exposed forward1 e2 timing e1 timing
        wait main e1 timing
        begin forward1_marginal_aggregation_halo @main
        lib spmm_csr_seg_f32 [3,6) part=halo halo @main
        end forward1_marginal_aggregation_halo @main
        release forward1 @main
        record_stream (6, 8) side
        --
        event e3 @main
        wait side e3
        begin backward1_communication @side
        post backward1 (6, 8) @side
        recv backward1 @side
        end backward1_communication @side
        event e4 timing @side
        begin backward1_central_aggregation @main
        lib row_live_f32 @main
        lib spmm_csr_seg_f32 [0,3) live @main
        end backward1_central_aggregation @main
        begin backward1_marginal_aggregation_local @main
        lib spmm_csr_seg_f32 [3,6) part=local live @main
        end backward1_marginal_aggregation_local @main
        event e5 timing @main
        exposed backward1 e5 timing e4 timing
        wait main e4 timing
        begin backward1_marginal_aggregation_halo @main
        lib spmm_csr_seg_f32 [3,6) part=halo halo live @main
        end backward1_marginal_aggregation_halo @main
        release backward1 @main
        record_stream (6, 8) side
        --
        event e6 @main
        wait side e6
        begin forward0_communication @side
        post test0 (6, 8) @side
        recv test0 @side
        end forward0_communication @side
        event e7 timing @side
        begin forward0_central_aggregation @main
        lib spmm_csr_seg_f32 [0,3) @main
        end forward0_central_aggregation @main
        begin forward0_marginal_aggregation_local @main
        lib spmm_csr_seg_f32 [3,6) part=local @main
        end forward0_marginal_aggregation_local @main
        event e8 timing @main
        exposed forward0 e8 timing e7 timing
        wait main e7 timing
        begin forward0_marginal_aggregation_halo @main
        lib spmm_csr_seg_f32 [3,6) part=halo halo @main
        end forward0_marginal_aggregation_halo @main
        release test0 @main
        record_stream (6, 8) side
        --
        event e9 @main
        wait side e9
        begin backward0_communication @side
        post backward0 (6, 8) @side
        recv backward0 @side
        end backward0_communication @side
        event e10 timing @side
        begin backward0_central_aggregation @main
        lib spmm_csr_seg_f32 [0,3) @main
        end backward0_central_aggregation @main
        begin backward0_marginal_aggregation_local @main
        lib spmm_csr_seg_f32 [3,6) part=local @main
        end backward0_marginal_aggregation_local @main
        event e11 timing @main
        exposed backward0 e11 timing e10 timing
        wait main e10 timing
        begin backward0_marginal_aggregation_halo @main
        lib spmm_csr_seg_f32 [3,6) part=halo halo @main
        end backward0_marginal_aggregation_halo @main
        release backward0 @main
        record_stream (6, 8) side
    """,
    ("gcn", "overlap_nosplit"): """
        event e0 @main
        wait side e0
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e1 timing @side
        begin forward1_central_aggregation @main
        lib spmm_csr_seg_f32 [0,3) @main
        end forward1_central_aggregation @main
        event e2 timing @main
        exposed forward1 e2 timing e1 timing
        wait main e1 timing
        begin forward1_marginal_aggregation @main
        lib spmm_csr_seg_f32 [3,6) halo @main
        end forward1_marginal_aggregation @main
        release forward1 @main
        record_stream (6, 8) side
        --
        event e3 @main
        wait side e3
        begin backward1_communication @side
        post backward1 (6, 8) @side
        recv backward1 @side
        end backward1_communication @side
        event e4 timing @side
        begin backward1_central_aggregation @main
        lib row_live_f32 @main
        lib spmm_csr_seg_f32 [0,3) live @main
        end backward1_central_aggregation @main
        event e5 timing @main
        exposed backward1 e5 timing e4 timing
        wait main e4 timing
        begin backward1_marginal_aggregation @main
        lib spmm_csr_seg_f32 [3,6) halo live @main
        end backward1_marginal_aggregation @main
        release backward1 @main
        record_stream (6, 8) side
        --
        event e6 @main
        wait side e6
        begin forward0_communication @side
        post test0 (6, 8) @side
        recv test0 @side
        end forward0_communication @side
        event e7 timing @side
        begin forward0_central_aggregation @main
        lib spmm_csr_seg_f32 [0,3) @main
        end forward0_central_aggregation @main
        event e8 timing @main
        exposed forward0 e8 timing e7 timing
        wait main e7 timing
        begin forward0_marginal_aggregation @main
        lib spmm_csr_seg_f32 [3,6) halo @main
        end forward0_marginal_aggregation @main
        release test0 @main
        record_stream (6, 8) side
        --
        event e9 @main
        wait side e9
        begin backward0_communication @side
        post backward0 (6, 8) @side
        recv backward0 @side
        end backward0_communication @side
        event e10 timing @side
        begin backward0_central_aggregation @main
        lib spmm_csr_seg_f32 [0,3) @main
        end backward0_central_aggregation @main
        event e11 timing @main
        exposed backward0 e11 timing e10 timing
        wait main e10 timing
        begin backward0_marginal_aggregation @main
        lib spmm_csr_seg_f32 [3,6) halo @main
        end backward0_marginal_aggregation @main
        release backward0 @main
        record_stream (6, 8) side
    """,
    ("gcn", "serial"): """
        begin forward1_communication @main
        post forward1 (6, 8) @main
        recv forward1 @main
        end forward1_communication @main
        begin forward1_full_aggregation @main
        lib spmm_csr_seg_f32 [0,6) halo @main
        end forward1_full_aggregation @main
        release forward1 @main
        --
        begin backward1_communication @main
        post backward1 (6, 8) @main
        recv backward1 @main
        end backward1_communication @main
        begin backward1_full_aggregation @main
        lib row_live_f32 @main
        lib spmm_csr_seg_f32 [0,6) halo live @main
        end backward1_full_aggregation @main
        release backward1 @main
        --
        begin forward0_communication @main
        post test0 (6, 8) @main
        recv test0 @main
        end forward0_communication @main
        begin forward0_full_aggregation @main
        lib spmm_csr_seg_f32 [0,6) halo @main
        end forward0_full_aggregation @main
        release test0 @main
        --
        begin backward0_communication @main
        post backward0 (6, 8) @main
        recv backward0 @main
        end backward0_communication @main
        begin backward0_full_aggregation @main
        lib spmm_csr_seg_f32 [0,6) halo @main
        end backward0_full_aggregation @main
        release backward0 @main
    """,
    ("gcn_loss_rows", "overlap"): """
        event e0 @main
        wait side e0
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e1 timing @side
        begin forward1_central_aggregation @main
        zeros (6, 8) @main
        lib spmm_csr_seg_f32 [0,3) rows=1 @main
        end forward1_central_aggregation @main
        begin forward1_marginal_aggregation_local @main
        lib spmm_csr_seg_f32 [3,6) part=local rows=2 @main
        end forward1_marginal_aggregation_local @main
        event e2 timing @main
        exposed forward1 e2 timing e1 timing
        wait main e1 timing
        begin forward1_marginal_aggregation_halo @main
        lib spmm_csr_seg_f32 [3,6) part=halo halo rows=2 @main
        end forward1_marginal_aggregation_halo @main
        release forward1 @main
        record_stream (6, 8) side
        --
        event e3 @main
        wait side e3
        begin forward0_communication @side
        post forward0 (6, 8) @side
        recv forward0 @side
        end forward0_communication @side
        event e4 timing @side
        begin forward0_central_aggregation @main
        lib spmm_csr_seg_f32 [0,3) @main
        end forward0_central_aggregation @main
        begin forward0_marginal_aggregation_local @main
        lib spmm_csr_seg_f32 [3,6) part=local @main
        end forward0_marginal_aggregation_local @main
        event e5 timing @main
        exposed forward0 e5 timing e4 timing
        wait main e4 timing
        begin forward0_marginal_aggregation_halo @main
        lib spmm_csr_seg_f32 [3,6) part=halo halo @main
        end forward0_marginal_aggregation_halo @main
        release forward0 @main
        record_stream (6, 8) side
    """,
    ("gcn_loss_rows", "overlap_nosplit"): """
        event e0 @main
        wait side e0
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e1 timing @side
        begin forward1_central_aggregation @main
        zeros (6, 8) @main
        lib spmm_csr_seg_f32 [0,3) rows=1 @main
        end forward1_central_aggregation @main
        event e2 timing @main
        exposed forward1 e2 timing e1 timing
        wait main e1 timing
        begin forward1_marginal_aggregation @main
        lib spmm_csr_seg_f32 [3,6) halo rows=2 @main
        end forward1_marginal_aggregation @main
        release forward1 @main
        record_stream (6, 8) side
        --
        event e3 @main
        wait side e3
        begin forward0_communication @side
        post forward0 (6, 8) @side
        recv forward0 @side
        end forward0_communication @side
        event e4 timing @side
        begin forward0_central_aggregation @main
        lib spmm_csr_seg_f32 [0,3) @main
        end forward0_central_aggregation @main
        event e5 timing @main
        exposed forward0 e5 timing e4 timing
        wait main e4 timing
        begin forward0_marginal_aggregation @main
        lib spmm_csr_seg_f32 [3,6) halo @main
        end forward0_marginal_aggregation @main
        release forward0 @main
        record_stream (6, 8) side
    """,
    ("gcn_loss_rows", "serial"): """
        begin forward1_communication @main
        post forward1 (6, 8) @main
        recv forward1 @main
        end forward1_communication @main
        begin forward1_full_aggregation @main
        zeros (6, 8) @main
        lib spmm_csr_seg_f32 [0,6) halo rows=3 @main
        end forward1_full_aggregation @main
        release forward1 @main
        --
        begin forward0_communication @main
        post forward0 (6, 8) @main
        recv forward0 @main
        end forward0_communication @main
        begin forward0_full_aggregation @main
        lib spmm_csr_seg_f32 [0,6) halo @main
        end forward0_full_aggregation @main
        release forward0 @main
    """,
    ("gcn_loss_rows_central_only", "overlap"): """
        event e0 @main
        wait side e0
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e1 timing @side
        begin forward1_central_aggregation @main
        zeros (6, 8) @main
        lib spmm_csr_seg_f32 [0,3) rows=2 @main
        end forward1_central_aggregation @main
        begin forward1_marginal_aggregation_local @main
        end forward1_marginal_aggregation_local @main
        event e2 timing @main
        exposed forward1 e2 timing e1 timing
        wait main e1 timing
        begin forward1_marginal_aggregation_halo @main
        end forward1_marginal_aggregation_halo @main
        release forward1 @main
        record_stream (6, 8) side
        --
        event e3 @main
        wait side e3
        begin forward0_communication @side
        post forward0 (6, 8) @side
        recv forward0 @side
        end forward0_communication @side
        event e4 timing @side
        begin forward0_central_aggregation @main
        lib spmm_csr_seg_f32 [0,3) @main
        end forward0_central_aggregation @main
        begin forward0_marginal_aggregation_local @main
        lib spmm_csr_seg_f32 [3,6) part=local @main
        end forward0_marginal_aggregation_local @main
        event e5 timing @main
        exposed forward0 e5 timing e4 timing
        wait main e4 timing
        begin forward0_marginal_aggregation_halo @main
        lib spmm_csr_seg_f32 [3,6) part=halo halo @main
        end forward0_marginal_aggregation_halo @main
        release forward0 @main
        record_stream (6, 8) side
    """,
    ("gcn_loss_rows_central_only", "overlap_nosplit"): """
        event e0 @main
        wait side e0
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e1 timing @side
        begin forward1_central_aggregation @main
        zeros (6, 8) @main
        lib spmm_csr_seg_f32 [0,3) rows=2 @main
        end forward1_central_aggregation @main
        event e2 timing @main
        exposed forward1 e2 timing e1 timing
        wait main e1 timing
        begin forward1_marginal_aggregation @main
        end forward1_marginal_aggregation @main
        release forward1 @main
        record_stream (6, 8) side
        --
        event e3 @main
        wait side e3
        begin forward0_communication @side
        post forward0 (6, 8) @side
        recv forward0 @side
        end forward0_communication @side
        event e4 timing @side
        begin forward0_central_aggregation @main
        lib spmm_csr_seg_f32 [0,3) @main
        end forward0_central_aggregation @main
        event e5 timing @main
        exposed forward0 e5 timing e4 timing
        wait main e4 timing
        begin forward0_marginal_aggregation @main
        lib spmm_csr_seg_f32 [3,6) halo @main
        end forward0_marginal_aggregation @main
        release forward0 @main
        record_stream (6, 8) side
    """,
    ("gcn_loss_rows_central_only", "serial"): """
        begin forward1_communication @main
        post forward1 (6, 8) @main
        recv forward1 @main
        end forward1_communication @main
        begin forward1_full_aggregation @main
        zeros (6, 8) @main
        lib spmm_csr_seg_f32 [0,6) halo rows=2 @main
        end forward1_full_aggregation @main
        release forward1 @main
        --
        begin forward0_communication @main
        post forward0 (6, 8) @main
        recv forward0 @main
        end forward0_communication @main
        begin forward0_full_aggregation @main
        lib spmm_csr_seg_f32 [0,6) halo @main
        end forward0_full_aggregation @main
        release forward0 @main
    """,
    ("gcn_loss_rows_marginal_only", "overlap"): """
        event e0 @main
        wait side e0
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e1 timing @side
        begin forward1_central_aggregation @main
        zeros (6, 8) @main
        end forward1_central_aggregation @main
        begin forward1_marginal_aggregation_local @main
        lib spmm_csr_seg_f32 [3,6) part=local rows=2 @main
        end forward1_marginal_aggregation_local @main
        event e2 timing @main
        exposed forward1 e2 timing e1 timing
        wait main e1 timing
        begin forward1_marginal_aggregation_halo @main
        lib spmm_csr_seg_f32 [3,6) part=halo halo rows=2 @main
        end forward1_marginal_aggregation_halo @main
        release forward1 @main
        record_stream (6, 8) side
        --
        event e3 @main
        wait side e3
        begin forward0_communication @side
        post forward0 (6, 8) @side
        recv forward0 @side
        end forward0_communication @side
        event e4 timing @side
        begin forward0_central_aggregation @main
        lib spmm_csr_seg_f32 [0,3) @main
        end forward0_central_aggregation @main
        begin forward0_marginal_aggregation_local @main
        lib spmm_csr_seg_f32 [3,6) part=local @main
        end forward0_marginal_aggregation_local @main
        event e5 timing @main
        exposed forward0 e5 timing e4 timing
        wait main e4 timing
        begin forward0_marginal_aggregation_halo @main
        lib spmm_csr_seg_f32 [3,6) part=halo halo @main
        end forward0_marginal_aggregation_halo @main
        release forward0 @main
        record_stream (6, 8) side
    """,
    ("gcn_loss_rows_marginal_only", "overlap_nosplit"): """
        event e0 @main
        wait side e0
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e1 timing @side
        begin forward1_central_aggregation @main
        zeros (6, 8) @main
        end forward1_central_aggregation @main
        event e2 timing @main
        exposed forward1 e2 timing e1 timing
        wait main e1 timing
        begin forward1_marginal_aggregation @main
        lib spmm_csr_seg_f32 [3,6) halo rows=2 @main
        end forward1_marginal_aggregation @main
        release forward1 @main
        record_stream (6, 8) side
        --
        event e3 @main
        wait side e3
        begin forward0_communication @side
        post forward0 (6, 8) @side
        recv forward0 @side
        end forward0_communication @side
        event e4 timing @side
        begin forward0_central_aggregation @main
        lib spmm_csr_seg_f32 [0,3) @main
        end forward0_central_aggregation @main
        event e5 timing @main
        exposed forward0 e5 timing e4 timing
        wait main e4 timing
        begin forward0_marginal_aggregation @main
        lib spmm_csr_seg_f32 [3,6) halo @main
        end forward0_marginal_aggregation @main
        release forward0 @main
        record_stream (6, 8) side
    """,
    ("gcn_loss_rows_marginal_only", "serial"): """
        begin forward1_communication @main
        post forward1 (6, 8) @main
        recv forward1 @main
        end forward1_communication @main
        begin forward1_full_aggregation @main
        zeros (6, 8) @main
        lib spmm_csr_seg_f32 [0,6) halo rows=2 @main
        end forward1_full_aggregation @main
        release forward1 @main
        --
        begin forward0_communication @main
        post forward0 (6, 8) @main
        recv forward0 @main
        end forward0_communication @main
        begin forward0_full_aggregation @main
        lib spmm_csr_seg_f32 [0,6) halo @main
        end forward0_full_aggregation @main
        release forward0 @main
    """,
    ("gcnii", "overlap"): """
        event e0 @main
        wait side e0
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e1 timing @side
        begin forward1_central_aggregation @main
        lib appnp_prop_f32 [0,3) @main
        end forward1_central_aggregation @main
        begin forward1_marginal_aggregation_local @main
        lib appnp_prop_f32 [3,6) part=local @main
        end forward1_marginal_aggregation_local @main
        event e2 timing @main
        exposed forward1 e2 timing e1 timing
        wait main e1 timing
        begin forward1_marginal_aggregation_halo @main
        lib appnp_prop_f32 [3,6) part=halo halo @main
        end forward1_marginal_aggregation_halo @main
        release forward1 @main
        record_stream (6, 8) side
        --
        event e3 @main
        wait side e3
        begin backward1_communication @side
        post backward1 (6, 8) @side
        recv backward1 @side
        end backward1_communication @side
        event e4 timing @side
        begin backward1_central_aggregation @main
        lib appnp_prop_f32 [0,3) @main
        end backward1_central_aggregation @main
        begin backward1_marginal_aggregation_local @main
        lib appnp_prop_f32 [3,6) part=local @main
        end backward1_marginal_aggregation_local @main
        event e5 timing @main
        exposed backward1 e5 timing e4 timing
        wait main e4 timing
        begin backward1_marginal_aggregation_halo @main
        lib appnp_prop_f32 [3,6) part=halo halo @main
        end backward1_marginal_aggregation_halo @main
        release backward1 @main
        record_stream (6, 8) side
    """,
    ("gcnii", "overlap_nosplit"): """
        event e0 @main
        wait side e0
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e1 timing @side
        begin forward1_central_aggregation @main
        lib appnp_prop_f32 [0,3) @main
        end forward1_central_aggregation @main
        event e2 timing @main
        exposed forward1 e2 timing e1 timing
        wait main e1 timing
        begin forward1_marginal_aggregation @main
        lib appnp_prop_f32 [3,6) halo @main
        end forward1_marginal_aggregation @main
        release forward1 @main
        record_stream (6, 8) side
        --
        event e3 @main
        wait side e3
        begin backward1_communication @side
        post backward1 (6, 8) @side
        recv backward1 @side
        end backward1_communication @side
        event e4 timing @side
        begin backward1_central_aggregation @main
        lib appnp_prop_f32 [0,3) @main
        end backward1_central_aggregation @main
        event e5 timing @main
        exposed backward1 e5 timing e4 timing
        wait main e4 timing
        begin backward1_marginal_aggregation @main
        lib appnp_prop_f32 [3,6) halo @main
        end backward1_marginal_aggregation @main
        release backward1 @main
        record_stream (6, 8) side
    """,
    ("gcnii", "serial"): """
        begin forward1_communication @main
        post forward1 (6, 8) @main
        recv forward1 @main
        end forward1_communication @main
        begin forward1_full_aggregation @main
        lib appnp_prop_f32 [0,6) halo @main
        end forward1_full_aggregation @main
        release forward1 @main
        --
        begin backward1_communication @main
        post backward1 (6, 8) @main
        recv backward1 @main
        end backward1_communication @main
        begin backward1_full_aggregation @main
        lib appnp_prop_f32 [0,6) halo @main
        end backward1_full_aggregation @main
        release backward1 @main
    """,
    ("sage_pool", "overlap"): """
        event e0 @main
        wait side e0
        begin forward0_communication @side
        post forward0 (6, 8) @side
        recv forward0 @side
        end forward0_communication @side
        event e1 timing @side
        begin forward0_central_aggregation @main
        lib sage_pool_fwd_f32 [0,3) @main
        end forward0_central_aggregation @main
        begin forward0_marginal_aggregation_local @main
        lib sage_pool_fwd_f32 [3,6) part=local @main
        end forward0_marginal_aggregation_local @main
        event e2 timing @main
        exposed forward0 e2 timing e1 timing
        wait main e1 timing
        begin forward0_marginal_aggregation_halo @main
        lib sage_pool_fwd_f32 [3,6) part=halo halo @main
        end forward0_marginal_aggregation_halo @main
        release forward0 @main
        record_stream (6, 8) side
        --
        event e3 @main
        wait side e3
        begin backward0_communication @side
        post pool_arg0 (6, 8) @side
        post backward0 (6, 8) @side
        recv backward0 @side
        recv pool_arg0 @side
        end backward0_communication @side
        event e4 timing @side
        begin backward0_central_aggregation @main
        lib sage_pool_bwd_f32 [0,3) @main
        end backward0_central_aggregation @main
        begin backward0_marginal_aggregation_local @main
        lib sage_pool_bwd_f32 [3,6) part=local @main
        end backward0_marginal_aggregation_local @main
        event e5 timing @main
        exposed backward0 e5 timing e4 timing
        wait main e4 timing
        begin backward0_marginal_aggregation_halo @main
        lib sage_pool_bwd_f32 [3,6) part=halo halo @main
        end backward0_marginal_aggregation_halo @main
        release backward0 @main
        release pool_arg0 @main
        record_stream (6, 8) side
        record_stream (6, 8) side
    """,
    ("sage_pool", "overlap_nosplit"): """
        event e0 @main
        wait side e0
        begin forward0_communication @side
        post forward0 (6, 8) @side
        recv forward0 @side
        end forward0_communication @side
        event e1 timing @side
        begin forward0_central_aggregation @main
        lib sage_pool_fwd_f32 [0,3) @main
        end forward0_central_aggregation @main
        event e2 timing @main
        exposed forward0 e2 timing e1 timing
        wait main e1 timing
        begin forward0_marginal_aggregation @main
        lib sage_pool_fwd_f32 [3,6) halo @main
        end forward0_marginal_aggregation @main
        release forward0 @main
        record_stream (6, 8) side
        --
        event e3 @main
        wait side e3
        begin backward0_communication @side
        post pool_arg0 (6, 8) @side
        post backward0 (6, 8) @side
        recv backward0 @side
        recv pool_arg0 @side
        end backward0_communication @side
        event e4 timing @side
        begin backward0_central_aggregation @main
        lib sage_pool_bwd_f32 [0,3) @main
        end backward0_central_aggregation @main
        event e5 timing @main
        exposed backward0 e5 timing e4 timing
        wait main e4 timing
        begin backward0_marginal_aggregation @main
        lib sage_pool_bwd_f32 [3,6) halo @main
        end backward0_marginal_aggregation @main
        release backward0 @main
        release pool_arg0 @main
        record_stream (6, 8) side
        record_stream (6, 8) side
    """,
    ("sage_pool", "serial"): """
        begin forward0_communication @main
        post forward0 (6, 8) @main
        recv forward0 @main
        end forward0_communication @main
        begin forward0_full_aggregation @main
        lib sage_pool_fwd_f32 [0,6) halo @main
        end forward0_full_aggregation @main
        release forward0 @main
        --
        begin backward0_communication @main
        post pool_arg0 (6, 8) @main
        post backward0 (6, 8) @main
        recv backward0 @main
        recv pool_arg0 @main
        end backward0_communication @main
        begin backward0_full_aggregation @main
        lib sage_pool_bwd_f32 [0,6) halo @main
        end backward0_full_aggregation @main
        release backward0 @main
        release pool_arg0 @main
    """,
}


@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("scenario", sorted(SCENARIOS))
def test_schedule(monkeypatch, scenario, mode):
    want = EXPECTED[(SAME_AS.get(scenario, scenario), mode)].strip().splitlines()
    assert run_scenario(monkeypatch, scenario, mode) == [w.strip() for w in want]


# the loss's rows [1, 4, 5] on a rank whose rows all have a halo neighbour (no central rows) and on one whose rows
# have none (no marginal rows): each launch still gets the listed rows of its own range
EXPECTED_ENDS = {
    0: """
        event e0 @main
        wait side e0
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e1 timing @side
        begin forward1_central_aggregation @main
        zeros (6, 8) @main
        end forward1_central_aggregation @main
        begin forward1_marginal_aggregation_local @main
        lib spmm_csr_seg_f32 [0,6) part=local rows=3 @main
        end forward1_marginal_aggregation_local @main
        event e2 timing @main
        exposed forward1 e2 timing e1 timing
        wait main e1 timing
        begin forward1_marginal_aggregation_halo @main
        lib spmm_csr_seg_f32 [0,6) part=halo halo rows=3 @main
        end forward1_marginal_aggregation_halo @main
        release forward1 @main
        record_stream (6, 8) side
        --
        event e3 @main
        wait side e3
        begin forward0_communication @side
        post forward0 (6, 8) @side
        recv forward0 @side
        end forward0_communication @side
        event e4 timing @side
        begin forward0_central_aggregation @main
        lib spmm_csr_seg_f32 [0,0) @main
        end forward0_central_aggregation @main
        begin forward0_marginal_aggregation_local @main
        lib spmm_csr_seg_f32 [0,6) part=local @main
        end forward0_marginal_aggregation_local @main
        event e5 timing @main
        exposed forward0 e5 timing e4 timing
        wait main e4 timing
        begin forward0_marginal_aggregation_halo @main
        lib spmm_csr_seg_f32 [0,6) part=halo halo @main
        end forward0_marginal_aggregation_halo @main
        release forward0 @main
        record_stream (6, 8) side
    """,
    N_INNER: """
        event e0 @main
        wait side e0
        begin forward1_communication @side
        post forward1 (6, 8) @side
        recv forward1 @side
        end forward1_communication @side
        event e1 timing @side
        begin forward1_central_aggregation @main
        zeros (6, 8) @main
        lib spmm_csr_seg_f32 [0,6) rows=3 @main
        end forward1_central_aggregation @main
        begin forward1_marginal_aggregation_local @main
        end forward1_marginal_aggregation_local @main
        event e2 timing @main
        exposed forward1 e2 timing e1 timing
        wait main e1 timing
        begin forward1_marginal_aggregation_halo @main
        end forward1_marginal_aggregation_halo @main
        release forward1 @main
        record_stream (6, 8) side
        --
        event e3 @main
        wait side e3
        begin forward0_communication @side
        post forward0 (6, 8) @side
        recv forward0 @side
        end forward0_communication @side
        event e4 timing @side
        begin forward0_central_aggregation @main
        lib spmm_csr_seg_f32 [0,6) @main
        end forward0_central_aggregation @main
        begin forward0_marginal_aggregation_local @main
        lib spmm_csr_seg_f32 [6,6) part=local @main
        end forward0_marginal_aggregation_local @main
        event e5 timing @main
        exposed forward0 e5 timing e4 timing
        wait main e4 timing
        begin forward0_marginal_aggregation_halo @main
        lib spmm_csr_seg_f32 [6,6) part=halo halo @main
        end forward0_marginal_aggregation_halo @main
        release forward0 @main
        record_stream (6, 8) side
    """,
}


@pytest.mark.parametrize("n_central", sorted(EXPECTED_ENDS))
def test_loss_rows_at_the_ends_of_the_split(monkeypatch, n_central):
    want = EXPECTED_ENDS[n_central].strip().splitlines()
    assert run_scenario(monkeypatch, "gcn_loss_rows", "overlap", n_central) == [w.strip() for w in want]

"""Distributed aggregation ops (autograd Functions) over the fused exchange + CSR SpMM.

Mirror of AdaQP/model/ops.py: `GCN_aggregation` / `SAGE_aggregation` (:17-67),
`DistAggConv` / `DistAggSAGE` (:69-111), `full_graph_propagation` (:132-154) and
`decomposed_graph_propagation` (:156-193) keep names, arguments and results.

GPU design: the aggregation reads local rows and halo rows in place (no torch.cat), the
central / marginal split is a row range of one CSR (no copy buffers, no host sync), and
in the decomposed path the exchange kernels run on the side stream while the central rows
aggregate on the default stream; ordering is by CUDA events only.
"""
from __future__ import annotations

import contextlib
import math
from typing import Any, Optional, Tuple

import torch
from torch import Tensor
from torch.autograd import Function

from .. import cs, gat, gatv2, sage_pool
from ..communicator import Communicator as comm
from ..communicator.p2p import CS_KEY, attn_keys, pool_arg_key, push_key
from ..helper import BitType, ProprogationMode
from ..manager import DecompGraph
from ..manager import GraphEngine as engine
from ..manager.graph import ACC_FOLD, ACC_ON, ACC_READ, LocalGraph, RowList, appnp_prop, row_list, row_live, spmm
from ..manager.graphEngine import RowRange
from .op_util import halo_exchange, msg_all2all_GLOO


def _split(graph, feats: Tensor, x_halo: Tensor = None):
    g = graph.graph if isinstance(graph, RowRange) else graph
    if x_halo is None and feats.shape[0] > g.n_inner:
        return g, feats[:g.n_inner], feats[g.n_inner:]
    return g, feats, x_halo


def _run(g, x_local, x_halo, pre, post, mean, add_self, lo, hi, out=None, part=None, live=None, rows=None):
    if isinstance(g, LocalGraph):
        return spmm(g, x_local, x_halo, pre, post, mean=mean, add_self=add_self, row_begin=lo, row_end=hi, out=out,
                    part=part, live=live, rows=rows)
    assert rows is None, "row lists are a device-path feature"
    from ..manager.graph_cpu import spmm_cpu          # gloo plumbing mode
    res = spmm_cpu(g, x_local, x_halo, pre, post, mean=mean, add_self=add_self, row_begin=lo, row_end=hi)
    if out is not None:
        out.copy_(res)
        return out
    return res


def GCN_aggregation(graph, feats: Tensor, mode: ProprogationMode = ProprogationMode.Forward,
                    x_halo: Tensor = None, out: Tensor = None, part: str = None, live: Tensor = None,
                    rows: RowList = None) -> Tensor:
    """out[v] = norm2[v] * sum_{u->v} norm1[u] x[u] with global-degree norms (ops.py:17-32).
    `feats` may be cat(local, halo) as in the reference, or the local rows with `x_halo`.  `live`: row liveness
    of the local rows (graph.row_live), so the gather skips the all-zero ones; the result is the same.  `rows`:
    only these destination rows of `out` are computed (graph.RowList), the others are left untouched."""
    g, x_local, x_halo = _split(graph, feats, x_halo)
    lo, hi = (graph.begin, graph.end) if isinstance(graph, RowRange) else (0, g.n_inner)
    if mode == ProprogationMode.Forward:
        pre, post = g.norm["out_-0.5"], g.norm["in_-0.5"]
    elif mode == ProprogationMode.Backward:
        pre, post = g.norm["in_-0.5"], g.norm["out_-0.5"]
    else:
        raise ValueError(f"Invalid mode {mode}")
    return _run(g, x_local, x_halo, pre, post, False, False, lo, hi, out, part, live, rows)


def SAGE_aggregation(graph, feats: Tensor, mode: ProprogationMode = ProprogationMode.Forward,
                     aggregator_type="mean", x_halo: Tensor = None, out: Tensor = None, part: str = None,
                     live: Tensor = None, rows: RowList = None) -> Tensor:
    """ops.py:34-67: 'mean' = mean over in-neighbours (fwd) / sum of x[u]/outdeg[u] (bwd);
    'gcn' = (sum + self) / (indeg + 1) (fwd) / sum + self of x/(outdeg+1) (bwd)."""
    g, x_local, x_halo = _split(graph, feats, x_halo)
    lo, hi = (graph.begin, graph.end) if isinstance(graph, RowRange) else (0, g.n_inner)
    if mode == ProprogationMode.Forward:
        if aggregator_type == "mean":
            return _run(g, x_local, x_halo, None, None, True, False, lo, hi, out, part, live, rows)
        if aggregator_type == "gcn":
            return _run(g, x_local, x_halo, None, g.norm["in_+1_-1"], False, True, lo, hi, out, part, live, rows)
    elif mode == ProprogationMode.Backward:
        if aggregator_type == "mean":
            return _run(g, x_local, x_halo, g.norm["out_-1"], None, False, False, lo, hi, out, part, live, rows)
        if aggregator_type == "gcn":
            return _run(g, x_local, x_halo, g.norm["out_+1_-1"], None, False, True, lo, hi, out, part, live, rows)
    else:
        raise ValueError(f"Invalid mode {mode}")
    raise ValueError(f"Invalid aggregator_type {aggregator_type}")


def _aggregate(class_name: str, graph, x_local, x_halo, mode, out, part=None, live=None, rows=None):
    if class_name == "DistAggConv":
        return GCN_aggregation(graph, x_local, mode=mode, x_halo=x_halo, out=out, part=part, live=live, rows=rows)
    if class_name == "DistAggSAGE":
        return SAGE_aggregation(graph, x_local, mode=mode, aggregator_type=engine.ctx.agg_type, x_halo=x_halo, out=out,
                                part=part, live=live, rows=rows)
    raise ValueError(f"Invalid class_name {class_name}")


def _eval_layer0(class_name: str, ctx, local_messages: Tensor, graph, layer: int, is_train: bool):
    """SURVEY 8f-3: every epoch's evaluation forward (trainer.py:181) exchanges and aggregates the
    CONSTANT input features of layer 0 in fp32 -- the result never changes, so it is computed once
    and reused (keyed on the feature tensor's storage and version).  Off while the Assigner traces
    (eval passes feed its variance statistics, op_util.py:91-99) or with ADAQP_EVAL_CACHE=0."""
    import os
    from ..assigner import Assigner as assigner
    eng = engine.ctx
    fn = decomposed_graph_propagation if eng.use_parallel else full_graph_propagation
    usable = (not is_train and layer == 0 and os.environ.get("ADAQP_EVAL_CACHE", "1") != "0"
              and not (assigner.ctx is not None and assigner.ctx.is_tracing))
    if not usable:
        return fn(ctx, local_messages, graph, layer, is_train, ProprogationMode.Forward, class_name)
    # keyed on the tensor OBJECT (held alive by the cache, so its address cannot be recycled), its version
    # counter, the graph and the aggregator; only the engine's own constant feature matrix is cached, so
    # every rank takes the same branch (a hit skips the exchange: ranks must agree or the key's sequence
    # numbers would diverge)
    if local_messages is not eng.feats:
        return fn(ctx, local_messages, graph, layer, is_train, ProprogationMode.Forward, class_name)
    key = (class_name, local_messages._version, tuple(local_messages.shape), id(graph),
           eng._agg_type if class_name == "DistAggSAGE" else None)
    cache = getattr(eng, "_eval_layer0_cache", None)
    if cache is None or cache[0] is not local_messages or cache[1] != key:
        out = fn(ctx, local_messages, graph, layer, is_train, ProprogationMode.Forward, class_name)
        eng._eval_layer0_cache = (local_messages, key, out)
        return out
    ctx.saved = layer
    return cache[2]


class DistAggConv(Function):
    """Aggregation of local + remote neighbours for GCN (ops.py:69-89)."""

    @staticmethod
    def forward(ctx, local_messages: Tensor, graph, layer: int, is_train: bool) -> Tensor:
        return _eval_layer0(DistAggConv.__name__, ctx, local_messages, graph, layer, is_train)

    @staticmethod
    def backward(ctx: Any, *grad_outputs: Tuple[Tensor, ...]):
        fn = decomposed_graph_propagation if engine.ctx.use_parallel else full_graph_propagation
        return fn(ctx, grad_outputs[0].contiguous(), engine.ctx.bwd_graph, ctx.saved, True,
                  ProprogationMode.Backward, DistAggConv.__name__)


class DistAggSAGE(Function):
    """Aggregation of local + remote neighbours for GraphSAGE (ops.py:91-111)."""

    @staticmethod
    def forward(ctx, local_messages: Tensor, graph, layer: int, is_train: bool) -> Tensor:
        return _eval_layer0(DistAggSAGE.__name__, ctx, local_messages, graph, layer, is_train)

    @staticmethod
    def backward(ctx: Any, *grad_outputs: Tuple[Tensor, ...]):
        fn = decomposed_graph_propagation if engine.ctx.use_parallel else full_graph_propagation
        return fn(ctx, grad_outputs[0].contiguous(), engine.ctx.bwd_graph, ctx.saved, True,
                  ProprogationMode.Backward, DistAggSAGE.__name__)


_SPLIT = None


def _split_marginal() -> bool:
    """Two-pass marginal aggregation (default; ADAQP_MARGINAL_SPLIT=0 restores the reference's
    single pass): local sources overlap the exchange, the halo sources accumulate afterwards.
    Removes the exposed wait at the price of a second pass over the marginal rows."""
    global _SPLIT
    if _SPLIT is None:
        import os
        _SPLIT = os.environ.get("ADAQP_MARGINAL_SPLIT", "1") != "0"
    return _SPLIT


_SKIP = None


def _skip_zero_rows() -> bool:
    """Skip the all-zero gradient rows in the output layer's backward aggregation (default; ADAQP_SKIP_ZERO_ROWS=0
    reads every row, for A/B runs).  The result is the same either way."""
    global _SKIP
    if _SKIP is None:
        import os
        _SKIP = os.environ.get("ADAQP_SKIP_ZERO_ROWS", "1") != "0"
    return _SKIP


def _live_rows(local_messages: Tensor, layer: int, mode: ProprogationMode):
    """Row liveness of the gradient the output layer's backward aggregation reads, or None.  The loss only sees the
    train rows, so dL/dlogits is exactly zero on every other row, and so is that row of dY W^T, the gradient this
    aggregation gathers: at ogbn-products' 8 % train share, 92 % of its rows.  Lower layers' gradients pass through
    LayerNorm and are dense, so they are read as they are."""
    top = getattr(engine.ctx, "top_layer", None)
    if mode != ProprogationMode.Backward or layer != top or not local_messages.is_cuda or not _skip_zero_rows():
        return None
    return row_live(local_messages)


# the rows the loss reads while train_for_one_epoch runs its forward pass (loss_rows); None outside it
_LOSS_MASK: Optional[Tensor] = None


@contextlib.contextmanager
def loss_rows(mask: Tensor):
    """Within this context the output layer's forward aggregation of a training pass computes only the rows `mask`
    selects (a bool mask over the inner rows or their indices) and leaves the other rows zero.  That layer is
    aggregate -> linear, so every other output row depends only on its own aggregated row: the rows the loss reads
    come out bitwise the same.  train_for_one_epoch wraps its forward call in it; a model called directly still
    computes every row."""
    global _LOSS_MASK
    prev = _LOSS_MASK
    _LOSS_MASK = mask
    try:
        yield
    finally:
        _LOSS_MASK = prev


def _loss_row_list(local_messages: Tensor, layer: int, is_train: bool,
                   mode: ProprogationMode) -> Optional[Tuple[RowList, Optional[RowList], Optional[RowList]]]:
    """(all, central, marginal) RowLists of the loss's rows when this aggregation is the output layer's training
    forward on the device path inside loss_rows(), else None (central / marginal: the rows below / from
    num_central, None without the decomposition).  Built once per mask (keyed on the mask object, its version and
    the row split) and kept on the engine, so the launches never read a list that has been freed."""
    mask, eng = _LOSS_MASK, engine.ctx
    if (mask is None or not is_train or mode != ProprogationMode.Forward or layer != getattr(eng, "top_layer", None)
            or not local_messages.is_cuda or comm.ctx.transport != "p2p"):
        return None
    key = (mask._version, eng.num_inner, eng.num_central if eng.use_parallel else None, local_messages.device)
    cache = getattr(eng, "_loss_rows_cache", None)
    if cache is None or cache[0] is not mask or cache[1] != key:
        rows = row_list(mask, eng.num_inner, local_messages.device)
        split = eng.num_central if eng.use_parallel else None
        views = (rows, rows.below(split), rows.from_(split)) if split is not None else (rows, None, None)
        eng._loss_rows_cache = cache = (mask, key, views)
    return cache[2]


def _finish(ctx, out: Tensor, layer: int, mode: ProprogationMode):
    if mode == ProprogationMode.Forward:
        ctx.saved = layer
        return out
    return out, None, None, None


def _full(graph) -> LocalGraph:
    """The whole LocalGraph of a graph argument (a DecompGraph in the overlapped mode)."""
    return graph.full if isinstance(graph, DecompGraph) else graph


def _p2p_only(model: str):
    if comm.ctx.transport != "p2p":
        raise NotImplementedError(f"{model} runs on the p2p transport only (not the CPU gloo plumbing mode)")


def _comm_name(name: str, is_train: bool) -> str:
    """Timer region of an exchange on `name`: quantised in training under the QUANT precision."""
    quant = engine.ctx.bit_type == BitType.QUANT and is_train
    return f"{name}_quantization" if quant else f"{name}_communication"


def _propagate(name: str, comm_name: str, exchange, aggregate, split: bool = False, sent: Tuple[Tensor, ...] = ()):
    """The exchange-and-overlap schedule of every aggregation on the p2p transport.

    exchange(stream) enqueues the exchange on `stream` (the current one when None) and returns (halo, aux, release);
    aggregate(lo, hi, halo, aux, part=None) runs the kernel over inner rows [lo, hi) and the result of its last call
    is returned; release() lets the senders reuse the received rows once their last consumer has been enqueued.
    Without the overlap (engine.ctx.use_parallel off) the exchange and then every row run on the current stream.
    With it the exchange runs on engine.ctx.marginal_stream while the central rows, which have no halo neighbour in
    either direction (so halo and aux are None), run on the current stream; the marginal rows run in one pass once
    the halo has landed, or, with `split` (a kernel whose local and halo sources combine exactly) and
    ADAQP_MARGINAL_SPLIT on, as part='local' while the exchange is in flight and part='halo' after it.  `sent` are
    the tensors the side stream reads."""
    eng, timer = engine.ctx, engine.ctx.timer
    if not eng.use_parallel:
        with timer.record_events(comm_name):
            halo, aux, release = exchange(None)
        with timer.record_events(f"{name}_full_aggregation"):
            kept = aggregate(0, eng.num_inner, halo, aux)
        release()
        return kept
    main, side = torch.cuda.current_stream(), eng.marginal_stream
    ready = torch.cuda.Event()
    ready.record(main)                       # what is sent is produced on the default stream
    side.wait_event(ready)
    with timer.record_events(comm_name, stream=side):
        halo, aux, release = exchange(side)
    landed = torch.cuda.Event(enable_timing=True)
    landed.record(side)
    nc, n = eng.num_central, eng.num_inner
    with timer.record_events(f"{name}_central_aggregation"):
        aggregate(0, nc, None, None)
    region, part = f"{name}_marginal_aggregation", None
    if split and _split_marginal():
        # the marginal rows' local-source neighbours do not need the halo either: aggregate them while the exchange
        # is still in flight; only the halo-source segment of each row waits for it
        with timer.record_events(f"{region}_local"):
            aggregate(nc, n, None, None, part="local")
        region, part = f"{region}_halo", "halo"
    overlappable_done = torch.cuda.Event(enable_timing=True)
    overlappable_done.record(main)
    timer.record_exposed(name, overlappable_done, landed)
    main.wait_event(landed)
    with timer.record_events(region):
        kept = aggregate(nc, n, halo, aux, part=part)
    release()
    for t in sent:
        t.record_stream(side)
    return kept


def _p2p_propagation(name: str, local_messages: Tensor, graph, layer: int, is_train: bool, mode: ProprogationMode,
                     class_name: str) -> Tensor:
    """The p2p transport of full_graph_propagation / decomposed_graph_propagation: _propagate over the halo exchange
    of local_messages.  The output layer's backward pass skips the all-zero gradient rows (_live_rows); its training
    forward inside loss_rows() computes only the loss's rows, each launch the list's rows of its range, and leaves
    the other rows zero.  Both are set up inside the first aggregation region (full, or central)."""
    eng, g = engine.ctx, _full(graph)
    listed = _loss_row_list(local_messages, layer, is_train, mode)
    out = live = None

    def exchange(stream):
        pend = halo_exchange(local_messages, name, is_train, stream=stream)
        return pend.halo, None, pend.release

    def aggregate(lo, hi, halo, _, part=None):
        nonlocal out, live
        if out is None:
            shape = (eng.num_inner, local_messages.shape[1])
            if listed is None:
                out, live = local_messages.new_empty(shape), _live_rows(local_messages, layer, mode)
            else:
                out = local_messages.new_zeros(shape)
        rows = None
        if listed is not None:
            # the whole list, or its central / marginal share; an empty share launches nothing
            rows = listed[0] if (lo, hi) == (0, eng.num_inner) else listed[1] if lo == 0 else listed[2]
            if not rows.n:
                return out
        _aggregate(class_name, RowRange(g, lo, hi), local_messages, halo, mode, out[lo:hi], part=part, live=live,
                   rows=rows)
        return out

    return _propagate(name, _comm_name(name, is_train), exchange, aggregate, split=True, sent=(local_messages,))


def full_graph_propagation(ctx, local_messages: Tensor, graph, layer: int, is_train: bool,
                           mode: ProprogationMode, class_name: str):
    """Exchange, then aggregate every inner row (ops.py:132-154)."""
    name = f"forward{layer}" if mode == ProprogationMode.Forward else f"backward{layer}"
    local_messages = local_messages.contiguous()
    timer = engine.ctx.timer
    g = _full(graph)
    if comm.ctx.transport == "p2p":
        out = _p2p_propagation(name, local_messages, graph, layer, is_train, mode, class_name)
    else:
        send_messages = local_messages[engine.ctx.total_send_idx]
        remote = msg_all2all_GLOO(send_messages, name, is_train)
        with timer.record(f"{name}_full_aggregation"):
            out = _aggregate(class_name, g, local_messages, remote, mode, None)
    return _finish(ctx, out, layer, mode)


def decomposed_graph_propagation(ctx, local_messages: Tensor, graph, layer: int, is_train: bool,
                                 mode: ProprogationMode, class_name: str):
    """Exchange on the side stream || central rows on the default stream, then the marginal
    rows once the halo has landed (ops.py:156-193)."""
    assert isinstance(graph, DecompGraph), f"graph must be a DecompGraph, but got {type(graph)}"
    name = f"forward{layer}" if mode == ProprogationMode.Forward else f"backward{layer}"
    local_messages = local_messages.contiguous()
    eng, timer = engine.ctx, engine.ctx.timer
    if comm.ctx.transport != "p2p":
        # gloo plumbing transport: the exchange runs in the helper thread while this thread aggregates the central
        # rows, as in the reference (ops.py:164-177: marginal_pool.apply_async ... response.get())
        send_messages = local_messages[eng.total_send_idx]
        pool = getattr(eng, "marginal_pool", None)
        response = pool.apply_async(msg_all2all_GLOO, (send_messages, name, is_train)) if pool is not None else None
        out = local_messages.new_empty((eng.num_inner, local_messages.shape[1]))
        with timer.record(f"{name}_central_aggregation"):
            _aggregate(class_name, graph.central_graph, local_messages, None, mode, out[:eng.num_central])
        remote = response.get() if response is not None else msg_all2all_GLOO(send_messages, name, is_train)
        with timer.record(f"{name}_marginal_aggregation"):
            _aggregate(class_name, graph.marginal_graph, local_messages, remote, mode, out[eng.num_central:])
        return _finish(ctx, out, layer, mode)
    return _finish(ctx, _p2p_propagation(name, local_messages, graph, layer, is_train, mode, class_name), layer, mode)


# ---------------------------------------------------------------- GAT
def _gat_exchange(rows: Tensor, name: str, is_train: bool, scalars: Tensor, aux_key: str, stream=None):
    """Exchange the boundary rows of one layer key (quantised per mode, as halo_exchange does for GCN / SAGE) and
    their per-row attention scalars in fp32 on `aux_key`: both ranks must compute the softmax from identical
    scalars.  Returns (halo rows, received scalar rows [num_remote, width], release), as _propagate's exchange."""
    ex = comm.ctx.comm_buffer.p2p
    ex.post_send_fp(aux_key, scalars, stream=stream)
    pend = halo_exchange(rows, name, is_train, stream=stream)
    aux_halo = ex.complete_recv_fp(aux_key, stream=stream)

    def release():
        pend.release()
        ex.release_fp(aux_key)
    return pend.halo, aux_halo, release


def _exchange(rows: Tensor, name: str, is_train: bool, scalars: Tensor = None, aux_key: str = None):
    """_propagate's exchange for the models with their own kernels: `rows` on `name`, and with `scalars` their
    per-row scalars in fp32 on `aux_key` (_gat_exchange)."""
    def exchange(stream):
        if scalars is not None:
            return _gat_exchange(rows, name, is_train, scalars, aux_key, stream=stream)
        pend = halo_exchange(rows, name, is_train, stream=stream)
        return pend.halo, None, pend.release
    return exchange


class DistAggGAT(Function):
    """Attention aggregation of local + remote neighbours for GAT (an extension beyond the reference).

    forward(z, a_l, a_r, graph, layer, is_train, heads) -> out: the exchange moves the projected rows z (key
    forward{l}, quantised per mode; test{l} in evaluation) and each row's el in fp32 (attn_fwd{l}); the received
    halo z / el are copied out of the slab because the backward pass needs them.  backward exchanges dL/dout
    (backward{l}) and each row's [er | lse | s] in fp32 (attn_bwd{l}), then gat_bwd gives dz, del and der; da_l /
    da_r are deterministic torch reductions.  p2p transport only.  The layer-0 evaluation cache never applies: the
    exchanged rows are z, not the input features."""

    @staticmethod
    def forward(ctx, z: Tensor, a_l: Tensor, a_r: Tensor, graph, layer: int, is_train: bool, heads: int) -> Tensor:
        _p2p_only("GAT")
        z = z.contiguous()
        n, F = z.shape
        el, er = gat.scores(z, a_l, a_r, heads)
        g = _full(graph)
        out = z.new_empty((n, F))
        lse = z.new_empty((n, heads))
        fwd_key, _ = attn_keys(layer)
        name = f"forward{layer}"

        def aggregate(lo, hi, z_halo, el_halo, part=None):
            if z_halo is not None and is_train:          # kept for the backward pass; the slab rows are reused
                z_halo, el_halo = z_halo.clone(), el_halo.clone()
            gat.forward(g, z, z_halo, el, el_halo, er, heads, lo, hi, out[lo:hi], lse[lo:hi])
            return z_halo, el_halo

        z_halo, el_halo = _propagate(name, _comm_name(name, is_train), _exchange(z, name, is_train, el, fwd_key),
                                     aggregate, sent=(z, el))
        if is_train:
            ctx.save_for_backward(z, z_halo, el, el_halo, er, out, lse, a_l, a_r)
            ctx.graph, ctx.layer, ctx.heads = graph, layer, heads
        return out

    @staticmethod
    def backward(ctx: Any, *grad_outputs: Tuple[Tensor, ...]):
        z, z_halo, el, el_halo, er, out, lse, a_l, a_r = ctx.saved_tensors
        grad = grad_outputs[0].contiguous()
        heads, layer = ctx.heads, ctx.layer
        n, F = z.shape
        D = F // heads
        s = (grad.view(n, heads, D) * out.view(n, heads, D)).sum(-1)
        aux = torch.cat([er, lse, s], 1).contiguous()
        g = _full(ctx.graph)
        dz = z.new_empty((n, F))
        dl = z.new_empty((n, heads))
        dr = z.new_empty((n, heads))
        _, bwd_key = attn_keys(layer)
        name = f"backward{layer}"

        def aggregate(lo, hi, g_halo, aux_halo, part=None):
            halo = (g_halo, z_halo, el_halo, aux_halo) if g_halo is not None else (None,) * 4
            gat.backward(g, grad, halo[0], z, halo[1], el, halo[2], aux, halo[3], a_l, a_r, heads, lo, hi,
                         dz[lo:hi], dl[lo:hi], dr[lo:hi])

        _propagate(name, _comm_name(name, True), _exchange(grad, name, True, aux, bwd_key), aggregate,
                   sent=(grad, aux))
        zh = z.view(n, heads, D)
        da_l = (dl.unsqueeze(-1) * zh).sum(0)
        da_r = (dr.unsqueeze(-1) * zh).sum(0)
        return dz, da_l.view_as(a_l), da_r.view_as(a_r), None, None, None, None


# ---------------------------------------------------------------- GATv2
class DistAggGATv2(Function):
    """GATv2 attention aggregation of local + remote neighbours (an extension beyond the reference).

    forward(zs, zd, attn, graph, layer, is_train, heads) -> out: the exchange moves the source projection zs (key
    forward{l}, quantised per mode; test{l} in evaluation); zd never leaves its rank.  The received halo zs is copied
    out of the slab because the backward pass needs it.  The central rows run while the exchange is in flight, the
    marginal rows in one pass after it lands.  The logit of an edge u -> v needs zs[u] and zd[v] together, so only
    v's rank can evaluate it: backward computes the source-side gradient of every received halo row
    (gatv2_bwd_halo), pushes it back to the row's owner in fp32 on push{l} while the central rows run, then runs the
    marginal rows with the pushed rows folded into dzs.  da is a deterministic torch sum of per-row shares.  The
    pushed gradient is the straight-through gradient of the (possibly dequantised) halo copy each rank used.  p2p
    transport only.  The layer-0 evaluation cache never applies: the exchanged rows are zs, not the input
    features."""

    @staticmethod
    def forward(ctx, zs: Tensor, zd: Tensor, attn: Tensor, graph, layer: int, is_train: bool, heads: int) -> Tensor:
        _p2p_only("GATv2")
        zs, zd = zs.contiguous(), zd.contiguous()
        n, F = zs.shape
        g = _full(graph)
        out = zs.new_empty((n, F))
        lse = zs.new_empty((n, heads))
        name = f"forward{layer}"

        def aggregate(lo, hi, zs_halo, _, part=None):
            if zs_halo is not None and is_train:          # kept for the backward pass; the slab rows are reused
                zs_halo = zs_halo.clone()
            gatv2.forward(g, zs, zs_halo, zd, attn, heads, lo, hi, out[lo:hi], lse[lo:hi])
            return zs_halo

        zs_halo = _propagate(name, _comm_name(name, is_train), _exchange(zs, name, is_train), aggregate, sent=(zs,))
        if is_train:
            if zs_halo is None:
                zs_halo = zs.new_empty((0, F))
            ctx.save_for_backward(zs, zs_halo, zd, out, lse, attn)
            ctx.graph, ctx.layer, ctx.heads = graph, layer, heads
        return out

    @staticmethod
    def backward(ctx: Any, *grad_outputs: Tuple[Tensor, ...]):
        zs, zs_halo, zd, out, lse, attn = ctx.saved_tensors
        grad = grad_outputs[0].contiguous()
        heads, layer = ctx.heads, ctx.layer
        n, F = zs.shape
        D = F // heads
        eng, ex = engine.ctx, comm.ctx.comm_buffer.p2p
        g = _full(ctx.graph)
        S = (grad.view(n, heads, D) * out.view(n, heads, D)).sum(-1).contiguous()
        halo_indptr, halo_dst = eng.gatv2_halo
        fold = eng.gatv2_fold
        key, name = push_key(layer), f"backward{layer}"
        dzs_halo = gatv2.backward_halo(halo_indptr, halo_dst, zs_halo, zd, grad, lse, S, attn, heads)
        dzs, dzd, da = (zs.new_empty((n, F)) for _ in range(3))

        def exchange(stream):
            ex.post_send_fp(key, dzs_halo, stream=stream)
            return ex.complete_recv_fp(key, stream=stream), None, lambda: ex.release_fp(key)

        def aggregate(lo, hi, push, _, part=None):
            # central rows are sent to no peer, so nothing is pushed to them (push is None)
            gatv2.backward_inner(g, zs, zs_halo, zd, grad, lse, S, attn, heads, push, fold if push is not None else None,
                                 lo, hi, dzs[lo:hi], dzd[lo:hi], da[lo:hi])

        # the push is fp32 in every mode
        _propagate(name, f"{name}_communication", exchange, aggregate, sent=(dzs_halo,))
        return dzs, dzd, da.sum(0).view_as(attn), None, None, None, None


# ---------------------------------------------------------------- SAGE max-pool
class DistAggSAGEPool(Function):
    """Max-pool aggregation of local + remote neighbours for GraphSAGE (DGL's aggregator_type='pool'; an extension
    beyond the reference, whose aggregators are mean and gcn).

    forward(p, graph, layer, is_train) -> m: the exchange moves the pooled rows p (key forward{l}, quantised per
    mode; test{l} in evaluation) and sage_pool_fwd takes the column-wise max and its arg; the local / halo sources of
    the marginal rows combine exactly, so they keep the two-pass overlap.  backward exchanges dL/dm (backward{l},
    every layer) and the arg rows in fp32 (pool_arg{l}): the owner of a source cannot recompute the arg of a remote
    destination, whose owner saw the dequantised copy of p.  sage_pool_bwd then routes the gradient to the arg
    source through engine.ctx.pool_want.  p2p transport only.  The layer-0 evaluation cache never applies: the
    exchanged rows are p, which depends on the weights."""

    @staticmethod
    def forward(ctx, p: Tensor, graph, layer: int, is_train: bool) -> Tensor:
        _p2p_only("SAGE max-pool")
        p = p.contiguous()
        n, F = p.shape
        g = _full(graph)
        m = p.new_empty((n, F))
        arg = torch.empty((n, F), dtype=torch.int32, device=p.device)
        name = f"forward{layer}"

        def aggregate(lo, hi, p_halo, _, part=None):
            sage_pool.forward(g, p, p_halo, lo, hi, m[lo:hi], arg[lo:hi], part=part)

        _propagate(name, _comm_name(name, is_train), _exchange(p, name, is_train), aggregate, split=True, sent=(p,))
        if is_train:
            ctx.save_for_backward(arg)
            ctx.graph, ctx.layer = graph, layer
        return m

    @staticmethod
    def backward(ctx: Any, *grad_outputs: Tuple[Tensor, ...]):
        arg, = ctx.saved_tensors
        grad = grad_outputs[0].contiguous()
        g = _full(ctx.graph)
        want = engine.ctx.pool_want
        dp = grad.new_empty(grad.shape)
        arg_rows, name = arg.view(torch.float32), f"backward{ctx.layer}"

        def aggregate(lo, hi, g_halo, arg_halo, part=None):
            a_halo = arg_halo.view(torch.int32) if arg_halo is not None else None
            sage_pool.backward(g, want, grad, g_halo, arg, a_halo, lo, hi, dp[lo:hi], part=part)

        _propagate(name, _comm_name(name, True), _exchange(grad, name, True, arg_rows, pool_arg_key(ctx.layer)),
                   aggregate, split=True, sent=(grad, arg_rows))
        return dp, None, None, None


# ---------------------------------------------------------------- APPNP / GCNII propagation steps
def _teleport_step(name: str, g: LocalGraph, h: Tensor, z: Tensor, alpha: float, is_train: bool) -> Tensor:
    """out = (1 - alpha) A h + alpha z over the exchange of h on `name` (A with the GCN forward norms): one
    appnp_prop launch per row range of _propagate's overlap, the teleport term in the kernel's epilogue."""
    pre, post = g.norm["out_-0.5"], g.norm["in_-0.5"]
    out = torch.empty_like(z)

    def aggregate(lo, hi, h_halo, _, part=None):
        appnp_prop(g, h, h_halo, pre, post, 1.0 - alpha, alpha, lo, hi, out[lo:hi], tele=z[lo:hi], part=part)

    _propagate(name, _comm_name(name, is_train), _exchange(h, name, is_train), aggregate, split=True, sent=(h,))
    return out


def _cs_step(step: int, g: LocalGraph, x: Tensor, alpha: float, tele: Tensor = None, y: Tensor = None,
             fix: Tensor = None, lo: float = -math.inf, hi: float = math.inf) -> Tensor:
    """One Correct & Smooth step over the fp32 exchange of x on CS_KEY (A with the GCN forward norms):
    out = clamp(alpha A x + (1 - alpha) tele, lo, hi), or with `fix` out = alpha A x with every row of y >= 0 reset to
    its row of fix.  The central rows run while the exchange is in flight; the marginal rows run in one pass once the
    halo has landed: a clamp or a fixed row cannot be applied to two partial sums.  Every step of a pass reuses the
    key; its sequence numbers pace them.  `step` names the timer regions."""
    ex = comm.ctx.comm_buffer.p2p
    pre, post = g.norm["out_-0.5"], g.norm["in_-0.5"]
    out = torch.empty_like(x)

    def exchange(stream):
        ex.post_send_fp(CS_KEY, x, stream=stream)
        return ex.complete_recv_fp(CS_KEY, stream=stream), None, lambda: ex.release_fp(CS_KEY)

    def aggregate(lo_, hi_, halo, _, part=None):
        cs.prop(g, x, halo, pre, post, alpha, 1.0 - alpha, lo_, hi_, out[lo_:hi_],
                tele=tele[lo_:hi_] if tele is not None else None, y=y[lo_:hi_] if y is not None else None,
                fix=fix[lo_:hi_] if fix is not None else None, lo=lo, hi=hi)

    name = f"cs{step}"
    _propagate(name, f"{name}_communication", exchange, aggregate, sent=(x,))
    return out


def correct_and_smooth(graph, logits: Tensor, y: Tensor, params: "cs.CSParams", n_train: int) -> Tensor:
    """Correct & Smooth (DESIGN §16) of this rank's [n_inner, C] base logits; every rank calls it together.  `y`:
    int32 per inner row, the label of the rank's train rows and -1 elsewhere; `n_train`: the train rows of all ranks.
    Returns the smoothed probabilities G_K.  fp32 exchange in every mode; p2p transport only."""
    _p2p_only("Correct & Smooth")
    g = _full(graph)
    z = logits.detach().float().contiguous()
    yhat, e0, l1 = cs.init(z, y)
    total = torch.tensor([l1], dtype=torch.float64)
    comm.all_reduce_sum(total)
    sigma = float(total[0]) / max(int(n_train), 1)
    a1, a2 = params.correct_alpha, params.smooth_alpha
    e, step = e0, 0
    for _ in range(params.correct_layers):
        if params.scale is None:
            e = _cs_step(step, g, e, a1, tele=e0, lo=-1.0, hi=1.0)
        else:
            e = _cs_step(step, g, e, a1, y=y, fix=e0)
        step += 1
    g0 = cs.combine(yhat, e, y, sigma=sigma) if params.scale is None else cs.combine(yhat, e, y, scale=params.scale)
    h = g0
    for _ in range(params.smooth_layers):
        h = _cs_step(step, g, h, a2, tele=g0, lo=0.0, hi=1.0)
        step += 1
    engine.ctx.timer.clear(is_train=False)
    return h


def _accum_step(name: str, g: LocalGraph, grad: Tensor, acc: Tensor, alpha: float, mode: int) -> Tensor:
    """out = (1 - alpha) A^T grad over the exchange of grad on `name` (the swapped norms), and in the same pass the
    acc term alpha * grad of each row, stored into / added to `acc` or folded into out per `mode` (ACC_* bits)."""
    pre, post = g.norm["in_-0.5"], g.norm["out_-0.5"]
    out = torch.empty_like(grad)

    def aggregate(lo, hi, g_halo, _, part=None):
        appnp_prop(g, grad, g_halo, pre, post, 1.0 - alpha, alpha, lo, hi, out[lo:hi], acc=acc[lo:hi], acc_mode=mode,
                   part=part)

    _propagate(name, _comm_name(name, True), _exchange(grad, name, True), aggregate, split=True, sent=(grad,))
    return out


class DistAPPNPProp(Function):
    """K personalized-PageRank steps of APPNP over the halo exchange (an extension beyond the reference):

        h_0 = z,   h_{k+1} = (1 - alpha) A h_k + alpha z,   returns h_K      A = D^-1/2 A D^-1/2 (the GCN norms)

    Step k exchanges h_k on forward{k} (quantised per mode; test{k} in evaluation) and runs appnp_prop_kernel, whose
    epilogue adds the teleport term alpha z.  The propagation is linear in z, so backward saves nothing:
    g_k = (1 - alpha) A^T g_{k+1} exchanges g_{k+1} on backward{k} (k = K-1 .. 0), the kernel also accumulates
    alpha g_{k+1} of each row, and the last step writes dz = alpha sum_{k=1..K} g_k + g_0 directly.  Quantisation is
    the identity in backward (straight-through), as in DistAggConv.  Every step keeps the overlap of
    _propagate with the two-pass marginal rows.  p2p transport only; the layer-0 evaluation cache does not apply
    (z depends on the weights)."""

    @staticmethod
    def forward(ctx, z: Tensor, graph, k: int, alpha: float, is_train: bool) -> Tensor:
        _p2p_only("APPNP")
        z = z.contiguous()
        g = _full(graph)
        h = z
        for step in range(k):
            h = _teleport_step(f"forward{step}", g, h, z, alpha, is_train)
        ctx.graph, ctx.k, ctx.alpha = graph, k, alpha
        return h

    @staticmethod
    def backward(ctx: Any, *grad_outputs: Tuple[Tensor, ...]):
        grad = grad_outputs[0].contiguous()
        k, alpha = ctx.k, ctx.alpha
        g = _full(ctx.graph)
        acc = torch.empty_like(grad)             # alpha * sum of the g_{k+1} seen so far
        nxt = grad                               # g_{k+1}
        for step in range(k - 1, -1, -1):
            mode = ACC_ON | (ACC_READ if step < k - 1 else 0) | (ACC_FOLD if step == 0 else 0)
            nxt = _accum_step(f"backward{step}", g, nxt, acc, alpha, mode)
        return nxt, None, None, None, None


# ---------------------------------------------------------------- GCNII
class DistGCNIIProp(Function):
    """The propagation of one GCNII layer over the halo exchange (an extension beyond the reference):

        s = (1 - alpha) A d + alpha h0        A = D^-1/2 A D^-1/2 (the GCN norms)

    with d the layer's (dropped-out) input and h0 the initial representation.  Layer l exchanges d on forward{l}
    (quantised per mode; test{l} in evaluation) and runs the teleport step, which is the column-sliced
    appnp_prop_sliced_kernel at hidden widths that are multiples of 128 above 128.  The step is linear in (d, h0), so
    backward saves nothing: one accumulate step over backward{l} writes dd = (1 - alpha) A^T ds and, in the same
    pass, dh0 = alpha ds (autograd sums the L layers' dh0).  backward0 is exchanged too: layer 1's gradient flows
    into h0 and on to the input weights.  Quantisation is the identity in backward (straight-through), as in
    DistAggConv.  p2p transport only; the layer-0 evaluation cache does not apply (h0 depends on the weights)."""

    @staticmethod
    def forward(ctx, d: Tensor, h0: Tensor, graph, alpha: float, is_train: bool, layer: int) -> Tensor:
        _p2p_only("GCNII")
        s = _teleport_step(f"forward{layer}", _full(graph), d.contiguous(), h0.contiguous(), alpha, is_train)
        ctx.graph, ctx.alpha, ctx.layer = graph, alpha, layer
        return s

    @staticmethod
    def backward(ctx: Any, *grad_outputs: Tuple[Tensor, ...]):
        ds = grad_outputs[0].contiguous()
        dh0 = torch.empty_like(ds)
        dd = _accum_step(f"backward{ctx.layer}", _full(ctx.graph), ds, dh0, ctx.alpha, ACC_ON)
        return dd, dh0, None, None, None, None

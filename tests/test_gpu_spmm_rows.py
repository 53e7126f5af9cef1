"""Aggregating only listed destination rows (spmm(..., rows=RowList)) and the training forward that uses it.

  * kernel: the output is prefilled with a NaN sentinel; the listed rows must be bitwise those of the same launch
    without a list, every other row must still hold the sentinel.  F = 100 (unsliced), 256 and 384 (column-sliced)
    and a forced slice width; GCN norms, SAGE mean and SAGE gcn (self term); the whole range, the central and the
    marginal range, and the two-pass local + halo form that accumulates; empty, one-row, first-and-last, all-rows
    and random 8 % lists; a hub row of in-degree above 100 000;
  * training: one train_for_one_epoch step (output layer restricted to the train rows) against the same step
    written out without loss_rows, same seeds, Adam update: loss, every gradient and every parameter bitwise equal,
    for GCN and SAGE mean / gcn at one rank (Vanilla) and two ranks (AdaQP-p, AdaQP), with the restricted launches
    counted (the output layer's forward only); a two-rank run where one rank has no train rows; the context is
    cleared after the step and when the forward raises; the evaluation forward still aggregates every row."""
import contextlib
import os
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def lib():
    from adaqp_b200 import build as b
    b.build()
    from adaqp_b200 import _lib
    return _lib


@contextlib.contextmanager
def slice_cols(w):
    _lib = lib()
    old = _lib.get_option("spmm_slice_cols")
    _lib.set_option("spmm_slice_cols", w)
    try:
        yield
    finally:
        _lib.set_option("spmm_slice_cols", old)


def bits(t):
    return t.contiguous().view(torch.int32)


def assert_bitwise(a, b, msg):
    assert a.shape == b.shape, (msg, a.shape, b.shape)
    if torch.equal(bits(a), bits(b)):
        return
    bad = torch.nonzero(bits(a) != bits(b))
    i = tuple(bad[0].tolist())
    raise AssertionError(f"{msg}: {bad.shape[0]} elements differ, first at {i}: {a[i].item()!r} vs {b[i].item()!r}")


SENTINEL = float("nan")


def check_rows(got, ref, listed_local, msg):
    """got: output prefilled with the sentinel; listed_local: listed row ids relative to the output's first row."""
    keep = torch.zeros(got.shape[0], dtype=torch.bool, device=got.device)
    keep[listed_local] = True
    assert_bitwise(got[keep], ref[keep], (msg, "listed rows"))
    sentinel = torch.full_like(got[~keep], SENTINEL)
    assert_bitwise(got[~keep], sentinel, (msg, "rows outside the list"))


def fwd_kinds(g):
    """The forward aggregations the output layer runs: GCN norms, SAGE mean, SAGE gcn (self term)."""
    return {"gcn": dict(pre=g.norm["out_-0.5"], post=g.norm["in_-0.5"]),
            "sage_mean": dict(pre=None, post=None, mean=True),
            "sage_gcn": dict(pre=None, post=g.norm["in_+1_-1"], add_self=True)}


def lists_for(lo, hi, gen):
    """Lists inside [lo, hi): empty, one row, first and last row, every row, a random 8 %."""
    n = hi - lo
    out = {"empty": np.zeros(0, np.int64), "all": np.arange(lo, hi)}
    if n:
        out["one"] = np.array([lo + n // 2])
        out["ends"] = np.unique([lo, hi - 1])
        pick = torch.rand(n, generator=gen) < 0.08
        out["p8"] = lo + torch.nonzero(pick).flatten().numpy()
    return out


def layouts(W, n, deg, F, seed):
    lib()
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    spec = SynthSpec(name="t", num_nodes=n, num_edges=n * deg, num_parts=W, num_feats=F, num_classes=5,
                     cross_fraction=0.3 if W > 1 else 0.0, community_size=64, seed=seed)
    return prepare_all_in_process(spec)


def run_range(g, xl, xh, kw, lo, hi, rows, two_pass):
    """One aggregation over [lo, hi) into a sentinel-filled output: one pass, or local + accumulated halo."""
    from adaqp_b200.manager.graph import spmm
    out = torch.full((hi - lo, xl.shape[1]), SENTINEL, device=xl.device)
    if two_pass:
        spmm(g, xl, None, row_begin=lo, row_end=hi, out=out, part="local", rows=rows, **kw)
        spmm(g, xl, xh, row_begin=lo, row_end=hi, out=out, part="halo", rows=rows, **kw)
    else:
        spmm(g, xl, xh, row_begin=lo, row_end=hi, out=out, rows=rows, **kw)
    return out


@pytest.mark.parametrize("F", [100, 256, 384])
@pytest.mark.parametrize("W", [1, 3])
def test_listed_rows_are_bitwise_the_full_launch(F, W):
    from adaqp_b200.manager.graph import LocalGraph, row_list
    dev = torch.device("cuda:0")
    L = layouts(W, 1500, 14, F, seed=F + W)[-1]
    g = LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, dev)
    gen = torch.Generator().manual_seed(F * 7 + W)
    xl = torch.randn(L.n_inner, F, generator=gen).to(dev)
    xh = torch.randn(L.n_halo, F, generator=gen).to(dev) if L.n_halo else None
    ranges = [("full", 0, L.n_inner, False)]
    if W > 1:
        assert L.n_halo > 0 and 0 < L.n_central < L.n_inner
        ranges += [("central", 0, L.n_central, False), ("marginal", L.n_central, L.n_inner, False),
                   ("marginal_two_pass", L.n_central, L.n_inner, True)]
    widths = [0, F] + ([64] if F % 128 == 0 else [])          # automatic rule, unsliced, a forced slice width
    n_checked = 0
    for kname, kw in fwd_kinds(g).items():
        for rname, lo, hi, two in ranges:
            with slice_cols(F):
                ref = run_range(g, xl, xh, kw, lo, hi, None, two)
            assert not torch.isnan(ref).any()
            for lname, ids in lists_for(lo, hi, gen).items():
                rl = row_list(torch.from_numpy(ids), L.n_inner, dev)
                for w in widths:
                    with slice_cols(w):
                        got = run_range(g, xl, xh, kw, lo, hi, rl, two)
                    torch.cuda.synchronize()
                    check_rows(got, ref, torch.from_numpy(ids - lo).to(dev), (kname, rname, lname, w))
                    n_checked += 1
    assert n_checked > 0
    # the frontier counter is clean after all of that: a launch without a list still covers every row
    with slice_cols(0):
        again = run_range(g, xl, xh, fwd_kinds(g)["gcn"], 0, L.n_inner, None, False)
    assert not torch.isnan(again).any()


def test_hub_row_in_a_list():
    """A destination row with 120 000 in-neighbours, listed with a few ordinary rows."""
    from adaqp_b200.manager.graph import LocalGraph, row_list, spmm
    dev = torch.device("cuda:0")
    rng = np.random.RandomState(7)
    n_inner, n_halo, hub = 3000, 400, 17
    deg = rng.randint(0, 20, size=n_inner)
    deg[hub] = 120_000
    cols = [np.sort(rng.randint(0, n_inner + n_halo, size=d)).astype(np.int32) for d in deg]
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = np.concatenate(cols).astype(np.int32)
    in_deg = np.concatenate([deg, rng.randint(1, 20, size=n_halo)]).astype(np.int64)
    out_deg = np.bincount(indices, minlength=n_inner + n_halo).astype(np.int64)
    g = LocalGraph(indptr, indices, in_deg, out_deg, n_inner, n_halo, dev)
    gen = torch.Generator().manual_seed(5)
    ids = np.array([0, 5, hub, 1000, n_inner - 1])
    rl = row_list(torch.from_numpy(ids), n_inner, dev)
    for F in [256, 100]:
        xl = torch.randn(n_inner, F, generator=gen).to(dev)
        xh = torch.randn(n_halo, F, generator=gen).to(dev)
        for kw in fwd_kinds(g).values():
            with slice_cols(F):
                ref = spmm(g, xl, xh, **kw)
            for w in [F, 0]:
                with slice_cols(w):
                    got = torch.full((n_inner, F), SENTINEL, device=dev)
                    spmm(g, xl, xh, out=got, rows=rl, **kw)
                torch.cuda.synchronize()
                check_rows(got, ref, torch.from_numpy(ids).to(dev), (F, w))
    assert int(indptr[hub + 1] - indptr[hub]) > 100_000


def test_library_refuses_bad_lists():
    """The C entry point rejects a count outside [0, row_end - row_begin] and a list combined with liveness."""
    _lib = lib()
    from adaqp_b200.manager.graph import LocalGraph, row_list
    dev = torch.device("cuda:0")
    L = layouts(1, 200, 8, 16, seed=3)[-1]
    g = LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, dev)
    x = torch.randn(L.n_inner, 16, device=dev)
    out = torch.empty_like(x)
    rl = row_list(torch.arange(4), L.n_inner, dev)
    live = torch.ones(L.n_inner, dtype=torch.uint8, device=dev)
    L_ = _lib.load()

    def call(n_list, live_ptr=None, lo=0, hi=None):
        hi = L.n_inner if hi is None else hi
        return L_.adaqp_spmm_csr_seg_f32(g.indptr.data_ptr(), None, None, g.indices.data_ptr(), x.data_ptr(), 16,
                                         L.n_inner, None, 0, None, None, 0, 0, 0, lo, hi, 16, out.data_ptr(), 16,
                                         live_ptr, rl.ids.data_ptr(), n_list, _lib.stream_ptr(None))
    assert call(-1) != 0
    assert call(L.n_inner + 1) != 0
    assert call(3, lo=0, hi=2) != 0
    assert call(4, live_ptr=live.data_ptr()) != 0
    assert call(0) == 0 and call(4) == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------ full training step, restricted and not
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def step_worker(rank, world, port, tmp, cfg, out):
    try:
        _step(rank, world, port, tmp, cfg, out)
    except BaseException:
        import traceback
        out.put((cfg["restrict"], rank, {"error": traceback.format_exc()}))
        raise


def _step(rank, world, port, tmp, cfg, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "ADAQP_SYNTH_SCALE": "0.002", "ADAQP_SEED": "11", "ADAQP_SYNTHETIC": "1",
                       "LOCAL_RANK": str(rank % torch.cuda.device_count())})
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    from adaqp_b200.communicator import Communicator as comm
    from adaqp_b200.manager import GraphEngine as engine
    from adaqp_b200.model import ops
    from adaqp_b200.trainer import runtime_util as ru
    tr = Trainer(Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                           model_name=cfg["model"], mode=cfg["mode"], assign_scheme="uniform", logger_level="WARNING",
                           num_epoches=1, exp_path=f"{tmp}/exp", aggregator_type=cfg.get("agg", "mean")))
    eng = engine.ctx
    if rank in cfg.get("no_train_on", ()):
        eng.train_mask = eng.train_mask[:0]
    ru.sync_seed()
    tr.model.reset_parameters()
    ru.sync_model(tr.model)
    calls = []                                     # (phase, part, number of listed rows or None)
    phase = ["forward"]
    real_spmm = ops.spmm

    def counted(g, x, *a, **k):
        rows = k.get("rows")
        calls.append((phase[0], k.get("part"), None if rows is None else rows.n))
        return real_spmm(g, x, *a, **k)

    ops.spmm = counted
    opt = torch.optim.Adam(tr.model.parameters(), lr=0.01)
    crit = torch.nn.CrossEntropyLoss(reduction="sum")
    n_train = torch.LongTensor([eng.train_mask.numel()])
    comm.all_reduce_sum(n_train)
    n_train = int(n_train)
    real_backward = torch.Tensor.backward

    def tagged_backward(self, *a, **k):
        phase[0] = "backward"
        return real_backward(self, *a, **k)

    torch.Tensor.backward = tagged_backward
    torch.manual_seed(1234 + rank)                 # dropout masks: equal in both runs
    if cfg["restrict"]:
        _, loss, _, _ = ru.train_for_one_epoch(1, eng.graph, tr.model, eng.feats, eng.labels, opt, crit, n_train,
                                               eng.train_mask)
        cleared = ops._LOSS_MASK is None
    else:
        # the same step written out, without loss_rows
        tr.model.train()
        logits = tr.model(eng.graph, eng.feats)
        loss = crit(logits[eng.train_mask], eng.labels[eng.train_mask]) / n_train
        opt.zero_grad()
        loss.backward()
        ru.average_gradients(tr.model)
        opt.step()
        cleared = True
    torch.Tensor.backward = real_backward
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().cpu().numpy().copy() for k, p in tr.model.named_parameters()}
    params = {k: p.detach().cpu().numpy().copy() for k, p in tr.model.named_parameters()}
    extra = {}
    if cfg["restrict"]:
        # evaluation forward inside the context: is_train is false, so every row is aggregated
        phase[0] = "eval"
        tr.model.eval()
        with torch.no_grad():
            plain = tr.model(eng.graph, eng.feats)
            eng.timer.clear(is_train=False)
            with ops.loss_rows(eng.train_mask):
                inside = tr.model(eng.graph, eng.feats)
            eng.timer.clear(is_train=False)
        extra["eval_equal"] = bool(torch.equal(bits(plain), bits(inside)))
        # a forward that raises inside train_for_one_epoch leaves the context cleared
        phase[0] = "raise"
        real_fwd = tr.model.forward

        def boom(*a, **k):
            assert ops._LOSS_MASK is eng.train_mask
            raise RuntimeError("forward failed")

        tr.model.forward = boom
        try:
            ru.train_for_one_epoch(1, eng.graph, tr.model, eng.feats, eng.labels, opt, crit, n_train, eng.train_mask)
        except RuntimeError as e:
            extra["raised"] = str(e)
        tr.model.forward = real_fwd
        extra["cleared_after_raise"] = ops._LOSS_MASK is None
    ops.spmm = real_spmm
    if comm.ctx.comm_buffer.p2p is not None:
        comm.ctx.comm_buffer.p2p.check_status()
    comm.ctx.delete_buffer()
    out.put((cfg["restrict"], rank, {"loss": loss.detach().cpu().numpy().copy(), "grads": grads, "params": params,
                                     "calls": calls, "top": eng.top_layer, "cleared": cleared,
                                     "n_train": int(eng.train_mask.numel()), "n_inner": eng.num_inner,
                                     "n_central": eng.num_central, "parallel": eng.use_parallel, **extra}))


def spawn_pair(world, cfg, timeout=400):
    """The restricted run and the reference run, as two process groups side by side."""
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    res = {True: {}, False: {}}
    with tempfile.TemporaryDirectory() as t1, tempfile.TemporaryDirectory() as t2:
        procs, ports = [], set()
        for restrict, tmp in ((True, t1), (False, t2)):
            port = _free_port()
            while port in ports:
                port = _free_port()
            ports.add(port)
            c = dict(cfg, restrict=restrict)
            procs += [ctx.Process(target=step_worker, args=(r, world, port, tmp, c, out)) for r in range(world)]
        for p in procs:
            p.start()
        for _ in procs:
            restrict, rank, r = out.get(timeout=timeout)
            assert "error" not in r, f"rank {rank} of the {'restricted' if restrict else 'reference'} run:\n{r['error']}"
            res[restrict][rank] = r
        for p in procs:
            p.join(timeout=60)
        assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return res[True], res[False]


def compare(on, off, world):
    for r in range(world):
        a, b = on[r], off[r]
        assert a["cleared"] and a["top"] == 2
        assert_bitwise(torch.from_numpy(a["loss"]), torch.from_numpy(b["loss"]), (r, "loss"))
        assert sorted(a["grads"]) == sorted(b["grads"])
        for k in a["grads"]:
            for what in ("grads", "params"):
                assert_bitwise(torch.from_numpy(a[what][k]), torch.from_numpy(b[what][k]), (r, what, k))
        assert a["eval_equal"] and a["raised"] == "forward failed" and a["cleared_after_raise"]
        # the reference run never lists rows; the restricted run lists them in the training forward only, in place
        # of the output layer's launches: 1 (whole range) or 3 (central, marginal local, marginal halo), less the
        # ones whose share of the list is empty
        assert all(c[2] is None for c in b["calls"])
        listed = [c for c in a["calls"] if c[2] is not None]
        assert all(c[0] == "forward" for c in listed), listed
        per_layer = 3 if a["parallel"] else 1
        fwd_ref = [c for c in b["calls"] if c[0] == "forward"]
        fwd_plain = [c for c in a["calls"] if c[0] == "forward" and c[2] is None]
        assert len(fwd_plain) == len(fwd_ref) - per_layer, (a["calls"], b["calls"])
        assert 0 < len(listed) <= per_layer if a["n_train"] else not listed, (listed, a["n_train"])
        assert all(c[2] > 0 for c in listed)
        # every train row is listed exactly once (the halo pass re-lists the marginal rows it accumulates into)
        assert sum(c[2] for c in listed if c[1] != "halo") == a["n_train"], (listed, a["n_train"])
        # the backward passes are the reference run's
        assert [c for c in a["calls"] if c[0] == "backward"] == [c for c in b["calls"] if c[0] == "backward"]


@pytest.mark.parametrize("world,mode", [(1, "Vanilla"), (2, "AdaQP-p"), (2, "AdaQP")])
@pytest.mark.parametrize("model,agg", [("gcn", "mean"), ("sage", "mean"), ("sage", "gcn")])
def test_training_step_bitwise_with_and_without_loss_rows(model, agg, world, mode):
    on, off = spawn_pair(world, dict(model=model, agg=agg, mode=mode))
    compare(on, off, world)


def test_rank_without_train_rows():
    """Rank 1 holds no train row: its output-layer forward launches nothing restricted, the step still matches."""
    on, off = spawn_pair(2, dict(model="gcn", mode="AdaQP-p", no_train_on=(1,)))
    assert on[1]["n_train"] == 0 and on[0]["n_train"] > 0
    compare(on, off, 2)

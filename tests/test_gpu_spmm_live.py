"""Skipping all-zero source rows in the aggregation (spmm(..., live=row_live(x))) changes no output bit.

  * row_live against (x != 0).any(1): rows of -0.0, NaN and inf rows, 16-byte and odd widths, strided views;
  * the skipping gather against the gather without liveness, compared bit for bit (int32 views, so NaN rows and
    the sign of zeros count too; the inputs keep every partial sum clear of underflow, the one case where the sign
    of a zero result may differ, DESIGN §3): random CSRs with 0 %, 8 %, 50 % and 100 % zero rows, rows of -0.0, NaN rows, a
    `pre` with an inf entry on a zero row, F = 256 and 384 (column-sliced), F = 100, 48 and 128 (unsliced), forced
    slice widths, every aggregation form the trainer runs (GCN norms, SAGE mean and gcn with its self term,
    central / marginal row ranges, the two-pass local + halo form that accumulates) and a hub of in-degree
    above 100 000;
  * one GCN and one SAGE-mean training step with an Adam update, with the path on and with ADAQP_SKIP_ZERO_ROWS=0:
    loss, every gradient and every parameter after the step bitwise equal, at one rank and at two ranks."""
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


def layouts(W, n, deg, F, seed):
    lib()
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    spec = SynthSpec(name="t", num_nodes=n, num_edges=n * deg, num_parts=W, num_feats=F, num_classes=5,
                     cross_fraction=0.3 if W > 1 else 0.0, community_size=64, seed=seed)
    return prepare_all_in_process(spec)


def kinds(g):
    return {"gcn_fwd": dict(pre=g.norm["out_-0.5"], post=g.norm["in_-0.5"]),
            "gcn_bwd": dict(pre=g.norm["in_-0.5"], post=g.norm["out_-0.5"]),
            "sage_mean": dict(pre=None, post=None, mean=True),
            "sage_mean_bwd": dict(pre=g.norm["out_-1"], post=None),
            "sage_gcn_bwd": dict(pre=g.norm["out_+1_-1"], post=None, add_self=True)}


def all_outputs(g, L, xl, xh, live, extra_kinds=()):
    """Every aggregation form the trainer runs, as one list of tensors."""
    from adaqp_b200.manager.graph import spmm
    outs = []
    for kw in list(kinds(g).values()) + list(extra_kinds):
        outs.append(spmm(g, xl, xh, live=live, **kw))
        outs.append(spmm(g, xl, None, row_begin=0, row_end=L.n_central, live=live, **kw))
        outs.append(spmm(g, xl, xh, row_begin=L.n_central, row_end=L.n_inner, live=live, **kw))
        if L.n_halo:
            two = torch.empty(L.n_inner - L.n_central, xl.shape[1], device=xl.device)
            spmm(g, xl, None, row_begin=L.n_central, row_end=L.n_inner, out=two, part="local", live=live, **kw)
            spmm(g, xl, xh, row_begin=L.n_central, row_end=L.n_inner, out=two, part="halo", live=live, **kw)
            outs.append(two)
    torch.cuda.synchronize()
    return outs


def with_zero_rows(x, share, gen, specials=True):
    """x with round(share * rows) rows zeroed (half of them to -0.0), plus, with `specials`, a NaN row and a row
    whose only nonzero is its last element."""
    n = x.shape[0]
    perm = torch.randperm(n, generator=gen)
    k = int(round(share * n))
    dead = perm[:k]
    x[dead] = 0.0
    x[dead[: k // 2]] = -0.0
    if specials and n > 8 and share < 1.0:
        live_rows = perm[k:]
        if live_rows.numel() >= 2:
            x[live_rows[0]] = float("nan")
            x[live_rows[1]] = 0.0
            x[live_rows[1], -1] = 1e-3
    return x


def test_row_live_matches_any_nonzero():
    from adaqp_b200.manager.graph import row_live
    lib()
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(3)
    for F in [256, 384, 100, 48, 128, 13, 1]:
        x = with_zero_rows(torch.randn(5000, F, generator=gen), 0.6, gen)
        x[7] = 0.0
        x[7, F // 2] = float("inf")
        x[9] = -0.0
        x = x.to(dev)
        want = (x != 0).any(1)
        assert_bitwise(row_live(x).bool().to(torch.int32), want.to(torch.int32), F)
        assert not want[9] and want[7]
    big = torch.randn(3000, 300, generator=gen).to(dev)
    big[::3, 4:260] = 0.0
    for lo, F in [(4, 256), (3, 97)]:            # views with row pitch 300: float4 and scalar loads
        v = big[:, lo:lo + F]
        assert torch.equal(row_live(v).bool(), (v != 0).any(1)), (lo, F)
    assert row_live(big[:0]).numel() == 0


@pytest.mark.parametrize("share", [0.0, 0.08, 0.5, 1.0])
@pytest.mark.parametrize("F", [256, 384, 100, 48, 128])
@pytest.mark.parametrize("W", [1, 3])
def test_live_path_is_bitwise_the_full_gather(F, share, W):
    from adaqp_b200.manager.graph import LocalGraph, row_live
    dev = torch.device("cuda:0")
    L = layouts(W, 1500, 14, F, seed=F + W)[-1]
    g = LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, dev)
    gen = torch.Generator().manual_seed(F + int(share * 100))
    xl = with_zero_rows(torch.randn(L.n_inner, F, generator=gen), share, gen).to(dev)
    xh = torch.randn(L.n_halo, F, generator=gen).to(dev) if L.n_halo else None
    if xh is not None:
        xh[::4] = 0.0                            # halo rows are always read, zero or not
    if W > 1:
        assert L.n_halo > 0 and 0 < L.n_central < L.n_inner
    live = row_live(xl)
    assert int(live.sum()) == int((xl != 0).any(1).sum())
    # a zero row whose weight is inf: inf * 0 = NaN reaches its destinations on both paths
    dead = torch.nonzero(live == 0).flatten()
    pre_inf = g.norm["in_-0.5"].clone()
    extra = []
    if dead.numel():
        pre_inf[dead[0]] = float("inf")
        extra.append(dict(pre=pre_inf, post=g.norm["out_-0.5"]))
    with slice_cols(F):
        ref = all_outputs(g, L, xl, xh, None, extra)
    for w in [F, 0, 64, 128]:                     # unsliced, the automatic rule, forced widths
        with slice_cols(w):
            got = all_outputs(g, L, xl, xh, live, extra)
        for i, (a, b) in enumerate(zip(got, ref)):
            assert_bitwise(a, b, (w, i))


def test_hub_row_with_dead_sources():
    """A destination row with 120 000 in-neighbours, 92 % of the local source rows zero."""
    from adaqp_b200.manager.graph import LocalGraph, row_live, spmm
    dev = torch.device("cuda:0")
    rng = np.random.RandomState(7)
    n_inner, n_halo, hub = 3000, 400, 17
    deg = rng.randint(0, 20, size=n_inner)
    deg[hub] = 120_000
    cols = [np.sort(rng.randint(0, n_inner + n_halo, size=d)).astype(np.int32) for d in deg]
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = np.concatenate(cols).astype(np.int32)
    # degrees of every source row, halo rows included: the norms are indexed by source id
    in_deg = np.concatenate([deg, rng.randint(1, 20, size=n_halo)]).astype(np.int64)
    out_deg = np.bincount(indices, minlength=n_inner + n_halo).astype(np.int64)
    g = LocalGraph(indptr, indices, in_deg, out_deg, n_inner, n_halo, dev)
    gen = torch.Generator().manual_seed(5)
    for F in [256, 100]:
        xl = with_zero_rows(torch.randn(n_inner, F, generator=gen), 0.92, gen, specials=False).to(dev)
        xh = torch.randn(n_halo, F, generator=gen).to(dev)
        live = row_live(xl)
        for kw in kinds(g).values():
            with slice_cols(F):
                ref = spmm(g, xl, xh, **kw)
            for w in [F, 0]:
                with slice_cols(w):
                    got = spmm(g, xl, xh, live=live, **kw)
                assert_bitwise(got, ref, (F, w))
    assert int(indptr[hub + 1] - indptr[hub]) > 100_000


# ------------------------------------------------------------------ full training step, path on and off
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def step_worker(rank, world, port, tmp, cfg, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "ADAQP_SYNTH_SCALE": "0.002", "ADAQP_SEED": "11", "ADAQP_SYNTHETIC": "1",
                       # read once, at the first backward aggregation: set before the package is imported
                       "ADAQP_SKIP_ZERO_ROWS": cfg["skip"],
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
    ru.sync_seed()
    tr.model.reset_parameters()
    ru.sync_model(tr.model)
    calls = []
    real_live = ops.row_live

    def counted(x, *a, **k):
        live = real_live(x, *a, **k)
        calls.append((int(x.shape[0]), int((live == 0).sum())))
        return live

    ops.row_live = counted
    opt = torch.optim.Adam(tr.model.parameters(), lr=0.01)
    tr.model.train()
    torch.manual_seed(1234 + rank)                 # dropout masks: equal in both runs
    logits = tr.model(eng.graph, eng.feats)
    n_train = torch.LongTensor([eng.train_mask.numel()])
    comm.all_reduce_sum(n_train)
    loss = torch.nn.functional.cross_entropy(logits[eng.train_mask], eng.labels[eng.train_mask], reduction="sum") / int(n_train)
    opt.zero_grad()
    loss.backward()
    ru.average_gradients(tr.model)
    grads = {k: p.grad.detach().cpu().numpy().copy() for k, p in tr.model.named_parameters()}
    opt.step()
    torch.cuda.synchronize()
    ops.row_live = real_live
    params = {k: p.detach().cpu().numpy().copy() for k, p in tr.model.named_parameters()}
    if comm.ctx.comm_buffer.p2p is not None:
        comm.ctx.comm_buffer.p2p.check_status()
    comm.ctx.delete_buffer()
    # numpy arrays travel by value: torch tensors would be shared through the worker, which exits after the put
    out.put((rank, {"loss": loss.detach().cpu().numpy().copy(), "grads": grads, "params": params, "calls": calls,
                    "top": eng.top_layer}))


def spawn(world, cfg, timeout=900):
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    with tempfile.TemporaryDirectory() as tmp:
        procs = [ctx.Process(target=step_worker, args=(r, world, port, tmp, cfg, out)) for r in range(world)]
        for p in procs:
            p.start()
        res = dict(out.get(timeout=timeout) for _ in procs)
        for p in procs:
            p.join(timeout=60)
        assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
        return res


@pytest.mark.parametrize("world,mode", [(1, "Vanilla"), (2, "AdaQP-p"), (2, "AdaQP")])
@pytest.mark.parametrize("model", ["gcn", "sage"])
def test_training_step_bitwise_with_and_without_skipping(model, world, mode):
    on = spawn(world, dict(model=model, mode=mode, skip="1"))
    off = spawn(world, dict(model=model, mode=mode, skip="0"))
    for r in range(world):
        a, b = on[r], off[r]
        assert a["top"] == 2 and b["calls"] == []
        # the output layer's backward aggregation only, over the local gradient rows, most of them zero
        assert len(a["calls"]) == 1, a["calls"]
        rows, dead = a["calls"][0]
        assert dead > 0.5 * rows, a["calls"]
        assert_bitwise(torch.from_numpy(a["loss"]), torch.from_numpy(b["loss"]), (r, "loss"))
        assert sorted(a["grads"]) == sorted(b["grads"])
        for k in a["grads"]:
            for what in ("grads", "params"):
                assert_bitwise(torch.from_numpy(a[what][k]), torch.from_numpy(b[what][k]), (r, what, k))

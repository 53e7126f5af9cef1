"""GATv2 without a GPU: the float64 oracle against torch autograd, the distributed protocol (forward exchange and the
push of halo gradients) against the monolithic layer, the push items and fold table against brute force, the key
tables, argument rejection by the C entry points, and the configurations GATv2 refuses."""
import os
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gatv2_oracle as G  # noqa: E402


def _sym_graph(n, deg, seed):
    """Random symmetric graph with one self-loop per node, CSR with sorted columns."""
    import scipy.sparse as sp
    rng = np.random.RandomState(seed)
    m = n * deg // 2
    a, b = rng.randint(0, n, m), rng.randint(0, n, m)
    A = sp.coo_matrix((np.ones(2 * m), (np.r_[a, b], np.r_[b, a])), shape=(n, n)).tocsr()
    A.setdiag(0)
    A.eliminate_zeros()
    A = (A + sp.eye(n)).tocsr()
    A.sort_indices()
    return A.indptr.astype(np.int64), A.indices.astype(np.int64)


def _rel(a, ref):
    a, ref = np.asarray(a), np.asarray(ref)
    return np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-30)


@pytest.mark.parametrize("H,D", [(1, 1), (1, 47), (4, 16), (4, 64)])
def test_oracle_matches_torch_autograd(H, D):
    n, fin = 60, 13
    indptr, indices = _sym_graph(n, 6, seed=H * 100 + D)
    rng = np.random.RandomState(D)
    x = rng.randn(n, fin)
    Ws, Wd = rng.randn(fin, H * D) * 0.3, rng.randn(fin, H * D) * 0.3
    bs, bd = rng.randn(H * D) * 0.1, rng.randn(H * D) * 0.1
    attn, g = rng.randn(H, D), rng.randn(n, H * D)
    res = G.layer(indptr, indices, x, Ws, bs, Wd, bd, attn, H, g)
    t = {k: torch.tensor(v, requires_grad=True)
         for k, v in (("x", x), ("Ws", Ws), ("bs", bs), ("Wd", Wd), ("bd", bd), ("attn", attn))}
    dst = torch.from_numpy(np.repeat(np.arange(n), np.diff(indptr)))
    src = torch.from_numpy(indices)
    y = G.torch_gatv2_layer(src, dst, t["x"], t["Ws"], t["bs"], t["Wd"], t["bd"], t["attn"], H)
    (y * torch.from_numpy(g)).sum().backward()
    assert _rel(res["out"], y.detach().numpy()) <= 1e-10
    for k, name in (("dx", "x"), ("dWs", "Ws"), ("dbs", "bs"), ("dWd", "Wd"), ("dbd", "bd"), ("da", "attn")):
        assert _rel(res[k], t[name].grad.numpy()) <= 1e-10, k


def _layouts(W, seed=None):
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    spec = SynthSpec(name="gatv2", num_nodes=900, num_edges=900 * 10, num_parts=W, num_feats=11, num_classes=5,
                     cross_fraction=0.25, community_size=64, seed=W if seed is None else seed)
    lays = prepare_all_in_process(spec, DistGNNType.DistGATv2)
    assert all(L.is_bidirected for L in lays)
    assert sum(L.n_halo for L in lays) > 0
    return lays


@pytest.mark.parametrize("W,H,D", [(2, 4, 8), (3, 1, 47), (3, 2, 16)])
def test_distributed_oracle_equals_monolithic(W, H, D):
    """Every inner row's out / lse / dzs / dzd, and dW_s, dW_d, db_s, db_d, da summed over ranks, equal the layer on
    the unpartitioned graph to 1e-10 relative: the protocol (forward zs, push of the halo rows' source-side
    gradients) loses nothing."""
    lays = _layouts(W)
    rng = np.random.RandomState(1)
    Ws, Wd = rng.randn(11, H * D) * 0.3, rng.randn(11, H * D) * 0.3
    bs, bd, attn = rng.randn(H * D) * 0.1, rng.randn(H * D) * 0.1, rng.randn(H, D)
    xs = [L.feat.astype(np.float64) for L in lays]
    gs = [rng.randn(L.n_inner, H * D) for L in lays]
    dist = G.dist_gatv2_layer(lays, xs, Ws, bs, Wd, bd, attn, H, gs)
    assert sum(d["dzs_halo"].shape[0] for d in dist) > 0 and any(np.abs(d["push"]).max() > 0 for d in dist)
    indptr, indices, base = G.global_from_layouts(lays)
    mono = G.layer(indptr, indices, np.concatenate(xs), Ws, bs, Wd, bd, attn, H, np.concatenate(gs))
    for key in ("out", "lse", "dzs", "dzd"):
        got = np.concatenate([d[key] for d in dist])
        assert _rel(got, mono[key]) <= 1e-10, key
    for key in ("dWs", "dWd", "dbs", "dbd", "da"):
        assert _rel(sum(d[key] for d in dist), mono[key]) <= 1e-10, key
    # without the push, the owners' dzs are wrong: the pushed rows carry real gradient
    got = np.concatenate([d["dzs_inner"] for d in dist])
    assert _rel(got, mono["dzs"]) > 1e-3


def test_push_items_and_tables_match_brute_force():
    """At W = 3: the holder's push items put halo row recv_idx[p][j] at row lo + j of owner p's region; the fold
    table lists each inner row's send positions in send-peer order; the halo-transposed table lists each halo row's
    inner destinations ascending."""
    from adaqp_b200 import gatv2
    from adaqp_b200.communicator.p2p import build_push_items
    lays = _layouts(3)
    for r, L in enumerate(lays):
        owner = {p: lays[p].send_idx[r] for p in L.recv_idx}
        items = build_push_items(list(L.recv_idx), L.recv_idx, owner)
        got = {(int(it["chan"]), int(it["src_row"]), int(it["dst_row"])) for it in items}
        want = set()
        for ci, p in enumerate(L.recv_idx):
            lo, hi = lays[p].send_idx[r]
            for j, h in enumerate(np.asarray(L.recv_idx[p])):
                want.add((ci, int(h), lo + j))
        assert got == want and items.size == len(want)
        fi, fp = gatv2.fold_table(L.n_inner, list(L.send_idx), L.send_idx, L.total_send_idx)
        bi, bp = G.fold_table(L)
        assert np.array_equal(fi, bi) and np.array_equal(fp, bp)
        hi_, hd = gatv2.halo_table(L.indptr, L.indices, L.n_inner, L.n_halo)
        ip, ix = np.asarray(L.indptr), np.asarray(L.indices)
        for h in range(L.n_halo):
            want_v = [v for v in range(L.n_inner) if (ix[ip[v]:ip[v + 1]] == L.n_inner + h).any()]
            assert hd[hi_[h]:hi_[h + 1]].tolist() == want_v
    with pytest.raises(RuntimeError, match="expected"):
        build_push_items([1], {1: np.arange(3)}, {1: (0, 2)})


def test_key_lists_and_existing_layouts():
    from adaqp_b200.communicator.p2p import (SlabLayout, appnp_key_dims, gat_key_dims, gatv2_key_dims, layer_keys,
                                             push_key, quantisable, sage_pool_key_dims)
    dims = gatv2_key_dims([256, 256, 47])
    assert list(dims) == ["test0", "test1", "test2", "forward0", "forward1", "forward2", "push0", "push1", "push2"]
    assert dims["push2"] == 47 and dims["forward0"] == 256 and push_key(1) == "push1"
    assert not quantisable("push0") and quantisable("forward0")
    # the push region has one row per send position, every other region one row per halo row
    lay = SlabLayout.build(2, list(dims), dims, {1: 10}, 10, push_rows=30)
    assert lay.halo_off["push0"] - lay.halo_off["forward2"] == 47 * 4 * 10 + 256 - (47 * 4 * 10) % 256
    assert lay.halo_off["push1"] - lay.halo_off["push0"] == 256 * 4 * 30
    # the layout of every existing key table is unchanged by the number of rows sent
    tables = [({k: (100 if k.endswith("0") else 256) for k in layer_keys(3)}),
              gat_key_dims([256, 256, 47], [4, 4, 1]), sage_pool_key_dims([100, 256]), appnp_key_dims(47, 10),
              appnp_key_dims(256, 8)]
    for t in tables:
        a = SlabLayout.build(3, list(t), t, {1: 10, 2: 7}, 17)
        b = SlabLayout.build(3, list(t), t, {1: 10, 2: 7}, 17, push_rows=1234)
        assert (a.flag_off, a.ack_off, a.qdata_off, a.params_off, a.halo_off, a.work_off, a.status_off, a.total) == \
            (b.flag_off, b.ack_off, b.qdata_off, b.params_off, b.halo_off, b.work_off, b.status_off, b.total)
    from adaqp_b200.assigner.assigner import Assigner
    for scheme in ("uniform", "random"):                  # adaptive needs a running engine: the GPU CLI test runs it
        a = Assigner(100, 256, 3, 10, scheme, 8, {}, 100, 0.5, 50, key_dims=dims)
        assert a.key_dims == {"forward0": 256, "forward1": 256, "forward2": 47}
        assert sorted(a.get_assignment({1: (0, 5)})) == ["forward0", "forward1", "forward2"]


def test_gatv2_score_is_gat_score():
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    spec = SynthSpec(name="gatv2", num_nodes=500, num_edges=5000, num_parts=2, num_feats=4, num_classes=3,
                     cross_fraction=0.2, community_size=32, seed=3)
    v2 = prepare_all_in_process(spec, DistGNNType.DistGATv2)
    v1 = prepare_all_in_process(spec, DistGNNType.DistGAT)
    for a, b in zip(v2, v1):
        for p in a.scores:
            assert np.array_equal(a.scores[p][0], b.scores[p][0]) and np.array_equal(a.scores[p][1], b.scores[p][1])


@pytest.fixture(scope="module")
def lib():
    from adaqp_b200 import _lib, build
    build.build()
    return _lib.load()


def test_entry_points_reject_bad_arguments(lib):
    err = lambda: lib.adaqp_last_error().decode()  # noqa: E731
    fwd = lib.adaqp_gatv2_fwd_f32
    assert fwd(None, None, 10, None, 300, None, 0, None, 300, None, 1, 300, 0, 2, None, 300, None, None) == -3 \
        and "F=300" in err()
    assert fwd(None, None, 10, None, 48, None, 0, None, 48, None, 5, 48, 0, 2, None, 48, None, None) == -1 \
        and "H=5" in err()
    assert fwd(None, None, 10, None, 48, None, 0, None, 48, None, 4, 48, 0, 2, None, 48, None, None) == -3 \
        and "D=12" in err()
    assert fwd(None, None, 10, None, 64, None, 0, None, 64, None, 4, 64, 5, 2, None, 64, None, None) == -1 \
        and "row range" in err()
    assert fwd(None, None, 10, None, 64, None, 0, None, 64, None, 4, 64, 0, 11, None, 64, None, None) == -1 \
        and "n_split" in err()
    assert fwd(None, None, 10, None, 64, None, 0, None, 32, None, 4, 64, 0, 2, None, 64, None, None) == -1 \
        and "pitch" in err()
    assert fwd(None, None, 10, None, 64, None, 0, None, 64, None, 4, 64, 0, 2, None, 64, None, None) == -1 \
        and "null" in err()
    inner = lib.adaqp_gatv2_bwd_inner_f32
    base = [None, None, 10, None, 64, None, 0, None, 64, None, 64, None, None, None, None, 0, None, None, 4, 64, 0, 2,
            None, 64, None, 64, None, 64, None]
    assert inner(*base) == -1 and "null" in err()
    a = list(base)
    a[21] = 11
    assert inner(*a) == -1 and "n_split" in err()
    a = list(base)
    a[16] = 8                                          # fold_indptr without push
    assert inner(*a) == -1 and "together" in err()
    a = list(base)
    a[27] = 32
    assert inner(*a) == -1 and "pitch" in err()
    a = list(base)
    a[18], a[19] = 3, 64
    assert inner(*a) == -1 and "H=3" in err()
    halo = lib.adaqp_gatv2_bwd_halo_f32
    assert halo(None, None, None, 64, None, 64, None, 64, None, None, None, 4, 64, 0, 2, None, 64, None) == -1 \
        and "null" in err()
    assert halo(None, None, None, 64, None, 64, None, 64, None, None, None, 4, 64, 3, 2, None, 64, None) == -1 \
        and "row range" in err()
    assert halo(None, None, None, 512, None, 512, None, 512, None, None, None, 1, 512, 0, 2, None, 512, None) == -3 \
        and "F=512" in err()
    # an empty range is a no-op
    assert halo(None, None, None, 64, None, 64, None, 64, None, None, None, 4, 64, 2, 2, None, 64, None) == 0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _refusal_worker(port, tmp, heads, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": "0", "WORLD_SIZE": "1",
                       "LOCAL_RANK": "0", "ADAQP_DEVICE": "cpu", "ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": "0.001"})
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    args = Namespace(dataset="reddit", num_parts=1, backend="gloo", init_method="env://", model_name="gatv2",
                     mode="Vanilla", assign_scheme="uniform", logger_level="WARNING", num_epoches=1,
                     exp_path=f"{tmp}/exp", gat_heads=heads)
    try:
        Trainer(args)
        out.put(("no error", ""))
    except Exception as e:                      # noqa: BLE001 - the type and message are what is checked
        out.put((type(e).__name__, str(e)))


@pytest.mark.parametrize("heads,want,text", [(3, "ValueError", "not divisible by gat_heads=3"),
                                             (4, "NotImplementedError", "model 'gatv2' runs on the p2p transport")])
def test_trainer_refuses(heads, want, text):
    """hidden_dim % gat_heads != 0 and the CPU gloo plumbing mode are refused before any partition is loaded."""
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    with tempfile.TemporaryDirectory() as tmp:
        p = ctx.Process(target=_refusal_worker, args=(_free_port(), tmp, heads, out))
        p.start()
        p.join(timeout=300)
        assert p.exitcode == 0
        kind, msg = out.get(timeout=5)
    assert kind == want and text in msg, (kind, msg)

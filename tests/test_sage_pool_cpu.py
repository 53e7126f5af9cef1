"""GraphSAGE max-pool without a GPU: the float64 oracle against torch autograd, the distributed protocol against the
monolithic layer, the match table against a brute-force construction, the exchange key lists, argument rejection by
the C entry points, and the configurations pool refuses."""
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

from oracle import sage_pool_oracle as P  # noqa: E402


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


def _weights(rng, fin, fout):
    return (rng.randn(fin, fin) * 0.5, rng.randn(fin) * 0.5, rng.randn(fout, fin) * 0.5, rng.randn(fout, fin) * 0.5,
            rng.randn(fout) * 0.1)


def _rel(a, ref):
    return np.abs(np.asarray(a) - ref).max() / max(np.abs(ref).max(), 1e-30)


@pytest.mark.parametrize("fin,fout", [(1, 3), (13, 7), (47, 41), (64, 5)])
def test_oracle_matches_torch_autograd(fin, fout):
    """Continuous random inputs: the only exact ties are ReLU zeros, whose gradient the mask kills on both sides."""
    n = 60
    indptr, indices = _sym_graph(n, 6, seed=fin)
    rng = np.random.RandomState(fout)
    x, g = rng.randn(n, fin), rng.randn(n, fout)
    Wp, bp, Ws, Wn, b = _weights(rng, fin, fout)
    res = P.layer(indptr, indices, x, Wp, bp, Ws, Wn, b, g)
    names = ("x", "Wp", "bp", "Ws", "Wn", "b")
    t = {k: torch.tensor(v, requires_grad=True) for k, v in zip(names, (x, Wp, bp, Ws, Wn, b))}
    dst = torch.from_numpy(np.repeat(np.arange(n), np.diff(indptr)))
    y = P.torch_pool_layer(torch.from_numpy(indices), dst, *(t[k] for k in names))
    (y * torch.from_numpy(g)).sum().backward()
    assert _rel(res["rst"], y.detach().numpy()) <= 1e-10
    for key, name in (("dx", "x"), ("dW_pool", "Wp"), ("db_pool", "bp"), ("dW_self", "Ws"), ("dW_neigh", "Wn"),
                      ("db", "b")):
        assert _rel(res[key], t[name].grad.numpy()) <= 1e-10, key


def test_oracle_tie_rule_and_hub():
    """arg is the first maximum in CSR order, also over a hub row wider than one column block."""
    n = 300
    indptr = np.concatenate([[0, n], n + np.arange(1, n)]).astype(np.int64)
    indices = np.concatenate([np.arange(n), np.arange(1, n)]).astype(np.int64)   # row 0: all nodes; row v: itself
    x = np.zeros((n, 70))
    x[[5, 9, 200], :] = 2.0            # three-way tie: the first in CSR order wins
    x[7, 3] = 3.0
    m, arg = P.forward(indptr, indices, x, n)
    assert np.all(m[0] == np.where(np.arange(70) == 3, 3.0, 2.0))
    assert np.all(arg[0] == np.where(np.arange(70) == 3, 7, 5) - n)
    assert np.all(arg[1:] == (np.arange(1, n) - n)[:, None])
    # two-pass (first 150 sources, then the rest merged with strict '>') equals one pass
    cut = 150
    m1, a1 = P.forward(np.array([0, cut]), indices[:cut], x, n)
    m2, a2 = P.forward(np.array([0, n - cut]), indices[cut:n], x, n)
    merged = np.where(m2[0] > m1[0], a2[0], a1[0])
    assert np.array_equal(merged, arg[0])


def _layouts(W, seed, nodes=900):
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    spec = SynthSpec(name="pool", num_nodes=nodes, num_edges=nodes * 10, num_parts=W, num_feats=11, num_classes=5,
                     cross_fraction=0.25, community_size=64, seed=seed)
    lays = prepare_all_in_process(spec, DistGNNType.DistSAGE)
    assert all(L.is_bidirected for L in lays)
    assert sum(L.n_halo for L in lays) > 0
    return lays


@pytest.mark.parametrize("W,fout", [(2, 7), (3, 5), (3, 16)])
def test_distributed_oracle_equals_monolithic(W, fout):
    """Every inner row's m / rst / dp / dx, and every weight gradient summed over ranks, equal the layer on the
    unpartitioned graph to 1e-10 relative: the protocol (forward p; backward gm and the encoded arg rows, matched
    through want) loses nothing."""
    lays = _layouts(W, seed=W)
    rng = np.random.RandomState(1)
    fin = 11
    Wp, bp, Ws, Wn, b = _weights(rng, fin, fout)
    xs = [L.feat.astype(np.float64) for L in lays]
    gs = [rng.randn(L.n_inner, fout) for L in lays]
    dist = P.dist_pool_layer(lays, xs, Wp, bp, Ws, Wn, b, gs)
    indptr, indices, base = P.global_from_layouts(lays)
    mono = P.layer(indptr, indices, np.concatenate(xs), Wp, bp, Ws, Wn, b, np.concatenate(gs))
    for key in ("m", "rst", "dx"):
        assert _rel(np.concatenate([d[key] for d in dist]), mono[key]) <= 1e-10, key
    # a column whose maximum is a ReLU zero ties between sources numbered differently on each side; its gradient is
    # masked, so dp is compared where p > 0
    dpre = np.concatenate([d["dp"] * (d["p"] > 0) for d in dist])
    assert _rel(dpre, mono["dp"] * (mono["p"] > 0)) <= 1e-10
    for key in ("dW_pool", "db_pool", "dW_self", "dW_neigh", "db"):
        assert _rel(sum(d[key] for d in dist), mono[key]) <= 1e-10, key
    # where the maximum is positive (unique for continuous inputs) the encoded arg names the monolithic arg source
    gids = P._gids(lays)
    for r, (L, d) in enumerate(zip(lays, dist)):
        got = gids[r][d["arg"] + L.n_inner]
        want = mono["arg"][base[r]:base[r] + L.n_inner] + base[-1]
        pos = d["m"] > 0
        assert pos.mean() > 0.3 and np.array_equal(got[pos], want[pos])


@pytest.mark.parametrize("W", [2, 3, 4])
def test_pool_want_matches_bruteforce(W):
    from adaqp_b200.sage_pool import pool_want
    lays = _layouts(W, seed=10 + W, nodes=700)
    for r, L in enumerate(lays):
        peer = {p: np.asarray(lays[p].recv_idx[r]) for p in L.send_idx}
        got = pool_want(L.indptr, L.indices, L.n_inner, L.recv_idx, L.send_idx, L.total_send_idx, peer)
        assert got.dtype == np.int32 and got.shape == (L.indices.size,)
        assert np.array_equal(got.astype(np.int64), P.pool_want_bruteforce(lays, r))


def test_key_lists():
    from adaqp_b200.communicator.p2p import SlabLayout, layer_keys, pool_arg_key, quantisable, sage_pool_key_dims
    dims = sage_pool_key_dims([602, 256, 256])
    assert list(dims) == ["test0", "test1", "test2", "forward0", "forward1", "forward2", "backward0", "backward1",
                          "backward2", "pool_arg0", "pool_arg1", "pool_arg2"]
    assert dims["forward0"] == dims["backward0"] == dims["test0"] == dims["pool_arg0"] == 602
    assert dims["pool_arg2"] == 256 and pool_arg_key(1) == "pool_arg1"
    assert not quantisable("pool_arg0") and quantisable("backward0")
    assert layer_keys(3) == ["test0", "test1", "test2", "forward0", "forward1", "forward2", "backward1", "backward2"]
    lay = SlabLayout.build(2, list(dims), dims, {1: 10}, 10)
    assert ("pool_arg0", 1) not in lay.qdata_off and ("backward0", 1) in lay.qdata_off
    assert lay.halo_off["pool_arg1"] - lay.halo_off["pool_arg0"] == (602 * 4 * 10 + 255) // 256 * 256   # aligned
    from adaqp_b200.assigner.assigner import Assigner
    a = Assigner(602, 256, 3, 10, "uniform", 8, {}, 100, 0.5, 50, key_dims=dims)
    assert sorted(a.get_assignment({1: (0, 5)})) == sorted(["forward0", "forward1", "forward2", "backward0",
                                                             "backward1", "backward2"])
    assert a.key_dims["backward0"] == 602


@pytest.fixture(scope="module")
def lib():
    from adaqp_b200 import _lib, build
    build.build()
    return _lib.load()


def test_entry_points_reject_bad_arguments(lib):
    err = lambda: lib.adaqp_last_error().decode()  # noqa: E731
    fwd, bwd = lib.adaqp_sage_pool_fwd_f32, lib.adaqp_sage_pool_bwd_f32
    assert fwd(None, None, None, None, 10, None, 1025, None, 0, 1025, 0, 2, 0, None, 1025, None, 1025, None) == -3 \
        and "F=1025" in err()
    assert fwd(None, None, None, None, 10, None, 64, None, 0, 0, 0, 2, 0, None, 64, None, 64, None) == -3 and "F=0" in err()
    assert fwd(None, None, None, None, 10, None, 64, None, 0, 64, 5, 2, 0, None, 64, None, 64, None) == -1 \
        and "row range" in err()
    assert fwd(None, None, None, None, 10, None, 64, None, 0, 64, 0, 2, 0, None, 64, None, 32, None) == -1 \
        and "pitch" in err()
    assert fwd(None, None, None, None, 10, None, 64, None, 0, 64, 0, 2, 0, None, 64, None, 64, None) == -1 \
        and "null" in err()
    assert fwd(None, None, None, None, 10, None, 64, None, 0, 64, 3, 3, 0, None, 64, None, 64, None) == 0   # empty range
    assert bwd(None, None, None, None, None, 10, None, 64, None, 0, None, 64, None, 0, 64, 0, 11, 0, None, 64,
               None) == -1 and "n_split" in err()
    assert bwd(None, None, None, None, None, 10, None, 64, None, 0, None, 60, None, 0, 64, 0, 4, 0, None, 64,
               None) == -1 and "pitch" in err()
    assert bwd(None, None, None, None, None, 10, None, 64, None, 0, None, 64, None, 0, 2000, 0, 4, 0, None, 2000,
               None) == -3 and "F=2000" in err()
    assert bwd(None, None, None, None, None, 10, None, 64, None, 0, None, 64, None, 0, 64, 0, 4, 0, None, 64,
               None) == -1 and "null" in err()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _refusal_worker(port, tmp, agg, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": "0", "WORLD_SIZE": "1",
                       "LOCAL_RANK": "0", "ADAQP_DEVICE": "cpu", "ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": "0.001"})
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    args = Namespace(dataset="reddit", num_parts=1, backend="gloo", init_method="env://", model_name="sage",
                     mode="Vanilla", assign_scheme="uniform", logger_level="WARNING", num_epoches=1,
                     exp_path=f"{tmp}/exp", aggregator_type=agg)
    try:
        Trainer(args)
        out.put(("no error", ""))
    except Exception as e:                      # noqa: BLE001 - the type and message are what is checked
        out.put((type(e).__name__, str(e)))


@pytest.mark.parametrize("agg,want,text", [("pool", "NotImplementedError", "p2p transport only"),
                                           ("lstm", "ValueError", "'lstm'")])
def test_trainer_refuses(agg, want, text):
    """The CPU gloo plumbing mode refuses pool; lstm (and any other unknown name) stays a ValueError."""
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    with tempfile.TemporaryDirectory() as tmp:
        p = ctx.Process(target=_refusal_worker, args=(_free_port(), tmp, agg, out))
        p.start()
        p.join(timeout=300)
        assert p.exitcode == 0
        kind, msg = out.get(timeout=5)
    assert kind == want and text in msg, (kind, msg)


def test_module_refuses_unknown_aggregator():
    from adaqp_b200.model.distSAGE import DistSAGEConv
    with pytest.raises(ValueError, match="lstm"):
        DistSAGEConv(4, 3, aggregator_type="lstm")
    conv = DistSAGEConv(4, 3, aggregator_type="pool")
    conv.reset_parameters()
    assert tuple(conv.fc_pool.weight.shape) == (4, 4) and torch.all(conv.fc_pool.bias == 0)

"""GAT without a GPU: the float64 oracle against torch autograd, the distributed protocol against the monolithic
layer, the exchange key lists, argument rejection by the C entry points, and the configurations GAT refuses."""
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

from oracle import gat_oracle as G  # noqa: E402


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


@pytest.mark.parametrize("H,D", [(1, 1), (1, 47), (1, 64), (4, 1), (4, 47), (4, 64)])
def test_oracle_matches_torch_autograd(H, D):
    n, fin = 60, 13
    indptr, indices = _sym_graph(n, 6, seed=H * 100 + D)
    rng = np.random.RandomState(D)
    x, W = rng.randn(n, fin), rng.randn(fin, H * D) * 0.3
    a_l, a_r, g = rng.randn(H, D), rng.randn(H, D), rng.randn(n, H * D)
    res = G.layer(indptr, indices, x, W, a_l, a_r, H, g)
    t = {k: torch.tensor(v, requires_grad=True) for k, v in (("x", x), ("W", W), ("a_l", a_l), ("a_r", a_r))}
    b = torch.zeros(H * D, dtype=torch.float64)
    dst = torch.from_numpy(np.repeat(np.arange(n), np.diff(indptr)))
    src = torch.from_numpy(indices)
    y = G.torch_gat_layer(src, dst, t["x"], t["W"], t["a_l"], t["a_r"], b, H)
    (y * torch.from_numpy(g)).sum().backward()

    def close(a, ref):
        a, ref = np.asarray(a), np.asarray(ref)
        return np.abs(a - ref).max() <= 1e-10 * max(np.abs(ref).max(), 1e-30)

    assert close(res["out"], y.detach().numpy())
    assert close(res["dx"], t["x"].grad.numpy())
    assert close(res["dW"], t["W"].grad.numpy())
    assert close(res["da_l"], t["a_l"].grad.numpy())
    assert close(res["da_r"], t["a_r"].grad.numpy())


@pytest.mark.parametrize("W,H,D", [(2, 4, 8), (3, 1, 47), (3, 2, 16)])
def test_distributed_oracle_equals_monolithic(W, H, D):
    """Every inner row's out / lse / dz / del / der, and dW, da_l, da_r summed over ranks, equal the layer on the
    unpartitioned graph to 1e-10 relative: the exchange protocol (forward z, el; backward g, [er | lse | s]) loses
    nothing."""
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    spec = SynthSpec(name="gat", num_nodes=900, num_edges=900 * 10, num_parts=W, num_feats=11, num_classes=5,
                     cross_fraction=0.25, community_size=64, seed=W)
    lays = prepare_all_in_process(spec, DistGNNType.DistGAT)
    assert all(L.is_bidirected for L in lays)
    assert sum(L.n_halo for L in lays) > 0
    rng = np.random.RandomState(1)
    Wt, a_l, a_r = rng.randn(11, H * D) * 0.3, rng.randn(H, D), rng.randn(H, D)
    xs = [L.feat.astype(np.float64) for L in lays]
    gs = [rng.randn(L.n_inner, H * D) for L in lays]
    dist = G.dist_gat_layer(lays, xs, Wt, a_l, a_r, H, gs)
    indptr, indices, base = G.global_from_layouts(lays)
    mono = G.layer(indptr, indices, np.concatenate(xs), Wt, a_l, a_r, H, np.concatenate(gs))

    def rel(a, ref):
        return np.abs(a - ref).max() / max(np.abs(ref).max(), 1e-30)

    for key in ("out", "lse", "dz", "del", "der"):
        got = np.concatenate([d[key] for d in dist])
        assert rel(got, mono[key]) <= 1e-10, key
    for key in ("dW", "da_l", "da_r"):
        assert rel(sum(d[key] for d in dist), mono[key]) <= 1e-10, key


def test_key_lists():
    from adaqp_b200.communicator.p2p import SlabLayout, gat_key_dims, layer_keys, quantisable
    dims = gat_key_dims([256, 256, 47], [4, 4, 1])
    assert [k for k in dims if k.startswith("backward")] == ["backward0", "backward1", "backward2"]
    assert dims["forward0"] == 256 and dims["forward2"] == 47 and dims["test2"] == 47 and dims["backward0"] == 256
    assert (dims["attn_fwd0"], dims["attn_bwd0"], dims["attn_fwd2"], dims["attn_bwd2"]) == (4, 12, 1, 3)
    assert not quantisable("attn_fwd0") and not quantisable("test1") and quantisable("backward0")
    # GCN / SAGE keep forward0..L-1, backward1..L-1 and the test keys
    assert layer_keys(3) == ["test0", "test1", "test2", "forward0", "forward1", "forward2", "backward1", "backward2"]
    lay = SlabLayout.build(2, list(dims), dims, {1: 10}, 10)
    assert ("attn_fwd0", 1) not in lay.qdata_off and ("backward0", 1) in lay.qdata_off
    assert lay.halo_off["attn_bwd2"] - lay.halo_off["attn_fwd2"] == 256       # 1 float x 10 rows, aligned
    from adaqp_b200.assigner.assigner import Assigner
    a = Assigner(100, 256, 3, 10, "uniform", 8, {}, 100, 0.5, 50, key_dims=dims)
    got = a.get_assignment({1: (0, 5)})
    assert sorted(got) == sorted(["forward0", "forward1", "forward2", "backward0", "backward1", "backward2"])
    assert a.key_dims["forward0"] == 256 and a.key_dims["backward2"] == 47
    b = Assigner(100, 256, 3, 10, "uniform", 8, {}, 100, 0.5, 50)
    assert list(b.get_assignment({1: (0, 5)})) == ["forward0", "forward1", "forward2", "backward1", "backward2"]
    assert b.key_dims == {"forward0": 100, "forward1": 256, "forward2": 256, "backward1": 256, "backward2": 256}


def test_gat_score_is_sage_mean_proxy():
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    spec = SynthSpec(name="gat", num_nodes=500, num_edges=5000, num_parts=2, num_feats=4, num_classes=3,
                     cross_fraction=0.2, community_size=32, seed=3)
    gat = prepare_all_in_process(spec, DistGNNType.DistGAT)
    sage = prepare_all_in_process(spec, DistGNNType.DistSAGE)
    for a, b in zip(gat, sage):
        for p in a.scores:
            assert np.array_equal(a.scores[p][0], b.scores[p][0])
            assert np.array_equal(a.scores[p][1], a.scores[p][0])


@pytest.fixture(scope="module")
def lib():
    from adaqp_b200 import _lib, build
    build.build()
    return _lib.load()


def test_entry_points_reject_bad_arguments(lib):
    err = lambda: lib.adaqp_last_error().decode()  # noqa: E731
    assert lib.adaqp_gat_scores_f32(None, 48, 4, 5, 48, None, None, None, None, None) == -1 and "H=5" in err()
    assert lib.adaqp_gat_scores_f32(None, 300, 4, 1, 300, None, None, None, None, None) == -3 and "F=300" in err()
    assert lib.adaqp_gat_scores_f32(None, 48, 4, 4, 48, None, None, None, None, None) == -3 and "D=12" in err()
    assert lib.adaqp_gat_scores_f32(None, 64, 4, 4, 64, None, None, None, None, None) == -1 and "null" in err()
    assert lib.adaqp_gat_fwd_f32(None, None, 10, None, 64, None, 0, None, None, None, 4, 64, 5, 2, None, 64, None,
                                 None) == -1 and "row range" in err()
    assert lib.adaqp_gat_fwd_f32(None, None, 10, None, 32, None, 0, None, None, None, 4, 64, 0, 2, None, 64, None,
                                 None) == -1 and "pitch" in err()
    assert lib.adaqp_gat_fwd_f32(None, None, 10, None, 64, None, 0, None, None, None, 4, 64, 0, 2, None, 64, None,
                                 None) == -1 and "null" in err()
    assert lib.adaqp_gat_bwd_f32(None, None, 10, None, 256, None, 0, None, 256, None, 0, None, None, None, None, None, None,
                                 4, 256, 0, 11, None, 256, None, None, None) == -1 and "n_split" in err()
    assert lib.adaqp_gat_bwd_f32(None, None, 10, None, 256, None, 0, None, 256, None, 0, None, None, None, None, None, None,
                                 3, 256, 0, 4, None, 256, None, None, None) == -1 and "H=3" in err()


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
    args = Namespace(dataset="reddit", num_parts=1, backend="gloo", init_method="env://", model_name="gat",
                     mode="Vanilla", assign_scheme="uniform", logger_level="WARNING", num_epoches=1,
                     exp_path=f"{tmp}/exp", gat_heads=heads)
    try:
        Trainer(args)
        out.put(("no error", ""))
    except Exception as e:                      # noqa: BLE001 - the type and message are what is checked
        out.put((type(e).__name__, str(e)))


@pytest.mark.parametrize("heads,want,text", [(3, "ValueError", "not divisible by gat_heads=3"),
                                             (4, "NotImplementedError", "p2p transport only")])
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

"""APPNP without a GPU: the float64 oracle against torch autograd, the distributed protocol against the monolithic
propagation, the exchange keys (multi-digit steps included), argument rejection by the C entry point, the refused
configurations and the checkpoint field."""
import json
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

from oracle import appnp_oracle as P  # noqa: E402


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
    return np.abs(np.asarray(a) - np.asarray(ref)).max() / max(np.abs(np.asarray(ref)).max(), 1e-30)


@pytest.mark.parametrize("k,alpha,C", [(1, 0.1, 5), (3, 0.0, 7), (10, 0.1, 47), (12, 0.25, 3), (4, 1.0, 2)])
def test_oracle_matches_torch_autograd(k, alpha, C):
    n = 70
    indptr, indices = _sym_graph(n, 6, seed=k * 10 + C)
    rng = np.random.RandomState(C)
    z, gk = rng.randn(n, C), rng.randn(n, C)
    res = P.monolithic(indptr, indices, z, gk, k, alpha)
    zt = torch.tensor(z, requires_grad=True)
    dst = torch.from_numpy(np.repeat(np.arange(n), np.diff(indptr)))
    src = torch.from_numpy(indices)
    h = P.torch_appnp(src, dst, zt, k, alpha)
    (h * torch.from_numpy(gk)).sum().backward()
    assert _rel(res["h"][-1], h.detach().numpy()) <= 1e-12
    assert _rel(res["dz"], zt.grad.numpy()) <= 1e-12
    # dz = alpha * sum_{k=1..K} g_k + g_0, g_k the gradient at h_k
    gs = res["g"]                      # g_K .. g_0
    assert len(gs) == k + 1 and np.array_equal(gs[0], gk)
    assert _rel(res["dz"], alpha * sum(gs[:k]) + gs[k]) <= 1e-14


@pytest.mark.parametrize("W,k,C", [(2, 3, 5), (3, 4, 7), (2, 11, 3)])
def test_distributed_oracle_equals_monolithic(W, k, C):
    """Every inner row's h_1..h_K and dz equal the unpartitioned propagation to 1e-10 relative: the protocol
    (forward{k} moves h_k, backward{k} moves g_{k+1}, backward0 included) loses nothing."""
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    spec = SynthSpec(name="appnp", num_nodes=900, num_edges=900 * 10, num_parts=W, num_feats=11, num_classes=5,
                     cross_fraction=0.25, community_size=64, seed=W + k)
    lays = prepare_all_in_process(spec, DistGNNType.DistAPPNP)
    assert all(L.is_bidirected for L in lays) and sum(L.n_halo for L in lays) > 0
    rng = np.random.RandomState(k)
    zs = [rng.randn(L.n_inner, C) for L in lays]
    gs = [rng.randn(L.n_inner, C) for L in lays]
    hs, fwd_halos = P.dist_forward(lays, zs, k, 0.15)
    dz, bwd_halos = P.dist_backward(lays, gs, k, 0.15)
    assert len(fwd_halos) == k and len(bwd_halos) == k
    indptr, indices, base = P.global_from_layouts(lays)
    mono = P.monolithic(indptr, indices, np.concatenate(zs), np.concatenate(gs), k, 0.15)
    for step in range(k):
        assert _rel(np.concatenate([h[step] for h in hs]), mono["h"][step]) <= 1e-10, step
    assert _rel(np.concatenate(dz), mono["dz"]) <= 1e-10


def test_appnp_partitions_are_gcn_partitions():
    """APPNP weighs halo rows with the GCN scores (its weights are the GCN norms times 1 - alpha)."""
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    spec = SynthSpec(name="appnp", num_nodes=500, num_edges=5000, num_parts=2, num_feats=4, num_classes=3,
                     cross_fraction=0.2, community_size=32, seed=3)
    a = prepare_all_in_process(spec, DistGNNType.DistAPPNP)
    b = prepare_all_in_process(spec, DistGNNType.DistGCN)
    for x, y in zip(a, b):
        assert np.array_equal(x.indices, y.indices) and x.scores.keys() == y.scores.keys()
        for p in x.scores:
            assert np.array_equal(x.scores[p][0], y.scores[p][0]) and np.array_equal(x.scores[p][1], y.scores[p][1])


def test_key_dims_and_multi_digit_keys():
    from adaqp_b200.communicator.p2p import SlabLayout, appnp_key_dims, key_dim, layer_index, quantisable
    dims = appnp_key_dims(47, 12)
    assert list(dims) == ([f"test{i}" for i in range(12)] + [f"forward{i}" for i in range(12)]
                          + [f"backward{i}" for i in range(12)])
    assert set(dims.values()) == {47}
    assert sum(quantisable(k) for k in dims) == 24
    # the whole trailing index: forward10 is step 10 (the last character alone would make it test0)
    assert layer_index("forward10") == 10 and layer_index("backward11") == 11 and layer_index("test3") == 3
    for key in ("forward0", "backward2", "test1"):          # every key of the other models keeps its meaning
        assert layer_index(key) == int(key[-1])
    assert key_dim("backward11", [47] * 12) == 47
    with pytest.raises(ValueError):
        layer_index("forward")
    lay = SlabLayout.build(2, list(dims), dims, {1: 10}, 10)
    assert ("backward0", 1) in lay.qdata_off and ("test11", 1) not in lay.qdata_off
    from adaqp_b200.assigner.assigner import Assigner
    a = Assigner(100, 256, 3, 10, "uniform", 8, {}, 100, 0.5, 50, key_dims=dims)
    got = a.get_assignment({1: (0, 5)})
    assert sorted(got) == sorted([f"forward{i}" for i in range(12)] + [f"backward{i}" for i in range(12)])
    assert all(v == 47 for v in a.key_dims.values())


def test_eval_key_of_step_ten_and_eleven(monkeypatch):
    """halo_exchange maps the evaluation exchange of forward10 / backward11 to test10 / test11 (not test0 / test1)."""
    from types import SimpleNamespace
    from adaqp_b200.communicator import Communicator
    from adaqp_b200.helper import BitType
    from adaqp_b200.manager import GraphEngine
    from adaqp_b200.model import op_util
    seen = []

    class FakeExchange:
        def post_send_fp(self, key, messages, gathered=False, stream=None):
            seen.append(key)

        def complete_recv_fp(self, key, stream=None):
            return None

    monkeypatch.setattr(Communicator, "ctx", SimpleNamespace(comm_buffer=SimpleNamespace(p2p=FakeExchange())))
    monkeypatch.setattr(GraphEngine, "ctx", SimpleNamespace(bit_type=BitType.FULL))
    for name in ("forward10", "backward11", "forward1", "forward0"):
        op_util.halo_exchange(torch.zeros(2, 3), name, is_train=False)
    op_util.halo_exchange(torch.zeros(2, 3), "forward10", is_train=True)
    assert seen == ["test10", "test11", "test1", "test0", "forward10"]


@pytest.fixture(scope="module")
def lib():
    from adaqp_b200 import _lib, build
    build.build()
    return _lib.load()


def test_entry_point_rejects_bad_arguments(lib):
    err = lambda: lib.adaqp_last_error().decode()  # noqa: E731
    f = lib.adaqp_appnp_prop_f32
    # (indptr, seg_start, seg_end, indices, x0, ld0, n_split, x1, ld1, pre, post, scale, alpha, tele, ldt, acc, lda,
    #  acc_mode, accumulate, row_begin, row_end, F, out, ldo, stream)
    assert f(None, None, None, None, None, 47, 100, None, 0, None, None, 0.9, 0.1, None, 0, None, 0, 0, 0, 0, 10, 47,
             None, 47, None) == -1 and "null pointer" in err()
    assert f(None, None, None, None, None, 1025, 100, None, 0, None, None, 0.9, 0.1, None, 0, None, 0, 0, 0, 0, 10,
             1025, None, 1025, None) == -3 and "F=1025" in err()
    assert f(None, None, None, None, None, 47, 100, None, 0, None, None, 0.9, 0.1, None, 0, None, 0, 0, 0, 0, 10, 0,
             None, 47, None) == -3 and "F=0" in err()
    assert f(None, None, None, None, None, 47, 100, None, 0, None, None, 0.9, 0.1, None, 0, None, 0, 0, 0, 5, 2, 47,
             None, 47, None) == -1 and "row range" in err()
    assert f(None, None, None, None, None, 47, 100, None, 0, None, None, 0.9, 0.1, None, 0, None, 0, 0, 0, 0, 101, 47,
             None, 47, None) == -1 and "row range" in err()
    assert f(None, None, None, None, None, 47, 100, None, 0, None, None, 0.9, 0.1, None, 0, None, 0, 6, 0, 0, 10, 47,
             None, 47, None) == -1 and "acc_mode" in err()
    assert f(None, None, None, None, None, 47, 100, None, 0, None, None, 0.9, 0.1, None, 0, None, 0, 1, 0, 0, 10, 47,
             None, 47, None) == -1 and "null pointer" in err()
    # an empty row range is a no-op even without pointers
    assert f(None, None, None, None, None, 47, 100, None, 0, None, None, 0.9, 0.1, None, 0, None, 0, 0, 0, 4, 4, 47,
             None, 47, None) == 0


def test_model_refuses_bad_parameters():
    from adaqp_b200.model.distAPPNP import appnp_params
    assert appnp_params(10, 0.1) == (10, 0.1) and appnp_params(3.0, 0) == (3, 0.0) and appnp_params(1, 1) == (1, 1.0)
    for k, a in ((0, 0.1), (-2, 0.1), (2.5, 0.1), ("3", 0.1), (True, 0.1), (3, -0.01), (3, 1.5), (3, "0.1"),
                 (3, float("nan"))):
        with pytest.raises(ValueError):
            appnp_params(k, a)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _refusal_worker(port, tmp, k, alpha, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": "0", "WORLD_SIZE": "1",
                       "LOCAL_RANK": "0", "ADAQP_DEVICE": "cpu", "ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": "0.001"})
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    args = Namespace(dataset="reddit", num_parts=1, backend="gloo", init_method="env://", model_name="appnp",
                     mode="Vanilla", assign_scheme="uniform", logger_level="WARNING", num_epoches=1,
                     exp_path=f"{tmp}/exp", appnp_k=k, appnp_alpha=alpha)
    try:
        Trainer(args)
        out.put(("no error", ""))
    except Exception as e:                      # noqa: BLE001 - the type and message are what is checked
        out.put((type(e).__name__, str(e)))


@pytest.mark.parametrize("k,alpha,want,text", [(0, 0.1, "ValueError", "appnp_k=0"),
                                               (2.5, 0.1, "ValueError", "not an integer"),
                                               (10, 1.5, "ValueError", "outside [0, 1]"),
                                               (10, 0.1, "NotImplementedError", "p2p transport only")])
def test_trainer_refuses(k, alpha, want, text):
    """Bad K / alpha and the CPU gloo plumbing mode are refused before any partition is loaded."""
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    with tempfile.TemporaryDirectory() as tmp:
        p = ctx.Process(target=_refusal_worker, args=(_free_port(), tmp, k, alpha, out))
        p.start()
        p.join(timeout=300)
        assert p.exitcode == 0
        kind, msg = out.get(timeout=5)
    assert kind == want and text in msg, (kind, msg)


# ----------------------------------------------------------------------------- checkpoint field
def _cfg(model_name, k=10, alpha=0.1):
    return {"data": {"num_feats": 100, "num_classes": 47},
            "model": {"num_layers": 3, "hidden_dim": 256, "aggregator_type": "mean", "gat_heads": 4,
                      "appnp_k": k, "appnp_alpha": alpha},
            "runtime": {"dataset": "ogbn-products", "model_name": model_name, "num_parts": 2, "mode": "AdaQP",
                        "assign_scheme": "random"}}


def _fake_checkpoint(path, fields, digests, epoch=3):
    from adaqp_b200.trainer import checkpoint as ck
    os.makedirs(path)
    with open(os.path.join(path, "manifest.json"), "w") as f:
        json.dump({"format": ck.FORMAT_VERSION, "epoch": epoch, "run": fields, "partitions": digests}, f)
    for name in ("model.pt", "rank0.pt", "rank1.pt"):
        open(os.path.join(path, name), "wb").close()


def test_checkpoint_propagation_field(tmp_path):
    from adaqp_b200.communicator.p2p import appnp_key_dims
    from adaqp_b200.trainer import checkpoint as ck
    appnp = ck.run_fields(_cfg("appnp"), appnp_key_dims(47, 10))
    assert appnp["propagation"] == {"k": 10, "alpha": 0.1}
    gcn = ck.run_fields(_cfg("gcn"), None)
    assert gcn["propagation"] is None
    digest = {"n_inner": 10, "n_halo": 3, "send_idx": {"1": [0, 4]}, "csr_sha256": "ab"}
    _fake_checkpoint(str(tmp_path / "appnp"), appnp, [digest, digest])
    assert ck.resume_error(str(tmp_path / "appnp"), appnp, digest, 0, 5) is None
    for k, alpha in ((12, 0.1), (10, 0.2)):
        other = ck.run_fields(_cfg("appnp", k, alpha), appnp_key_dims(47, k))
        err = ck.resume_error(str(tmp_path / "appnp"), dict(other, key_dims=appnp["key_dims"]), digest, 0, 5)
        assert isinstance(err, ValueError) and "'propagation'" in str(err), err
    # predicting with another K or alpha is refused; the model fields alone would match
    other = ck.run_fields(_cfg("appnp", 10, 0.2), appnp_key_dims(47, 10))
    with pytest.raises(ValueError, match="propagation"):
        ck.load_weights(str(tmp_path / "appnp"), None, other)
    # a manifest written before the field existed still matches a GCN run
    old = {k: v for k, v in gcn.items() if k != "propagation"}
    _fake_checkpoint(str(tmp_path / "old"), old, [digest, digest])
    assert ck.resume_error(str(tmp_path / "old"), gcn, digest, 0, 5) is None
    assert ck.resume_error(str(tmp_path / "old"), appnp, digest, 0, 5) is not None

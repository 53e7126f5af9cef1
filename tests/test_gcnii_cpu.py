"""GCNII without a GPU: the float64 oracle against torch autograd, the distributed protocol against the monolithic
model, the exchange keys (multi-digit layers included), argument rejection, the refused configurations, the
checkpoint field and the command-line flags."""
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

from oracle import gcnii_oracle as G  # noqa: E402


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


@pytest.mark.parametrize("L,alpha,theta", [(1, 0.1, 0.5), (3, 0.0, 1.0), (8, 0.1, 0.5), (11, 0.25, 1.5), (2, 1.0, 0.5)])
def test_oracle_matches_torch_autograd(L, alpha, theta):
    n, F, H, C = 60, 9, 12, 5
    indptr, indices = _sym_graph(n, 6, seed=L * 7 + F)
    rng = np.random.RandomState(L)
    x = rng.randn(n, F)
    P = G.init_params(rng, F, H, C, L)
    Gl = rng.randn(n, C)
    logits, grads = G.monolithic(indptr, indices, x, P, Gl, L, alpha, theta)
    Pt = {k: torch.tensor(v, requires_grad=True) for k, v in P.items()}
    dst = torch.from_numpy(np.repeat(np.arange(n), np.diff(indptr)))
    src = torch.from_numpy(indices)
    out = G.torch_gcnii(src, dst, torch.from_numpy(x), Pt, L, alpha, theta)
    (out * torch.from_numpy(Gl)).sum().backward()
    assert _rel(logits, out.detach().numpy()) <= 1e-12
    assert set(grads) == set(P)
    for k in P:
        assert grads[k].shape == P[k].shape, k
        assert _rel(grads[k], Pt[k].grad.numpy()) <= 1e-11, k


@pytest.mark.parametrize("W,L", [(2, 3), (3, 4), (2, 11)])
def test_distributed_oracle_equals_monolithic(W, L):
    """Every rank's logits and the summed parameter gradients equal the unpartitioned model to 1e-10 relative: the
    protocol (forward{l-1} moves h_{l-1}, backward{l-1} moves ds_l, backward0 included) loses nothing."""
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    spec = SynthSpec(name="gcnii", num_nodes=700, num_edges=700 * 10, num_parts=W, num_feats=11, num_classes=5,
                     cross_fraction=0.25, community_size=64, seed=W + L)
    lays = prepare_all_in_process(spec, DistGNNType.DistGCNII)
    assert all(Lr.is_bidirected for Lr in lays) and sum(Lr.n_halo for Lr in lays) > 0
    rng = np.random.RandomState(L)
    H = 8
    P = G.init_params(rng, 11, H, 5, L)
    xs = [rng.randn(Lr.n_inner, 11) for Lr in lays]
    Gs = [rng.randn(Lr.n_inner, 5) for Lr in lays]
    logits, grads, halos = G.dist_step(lays, xs, P, Gs, L, 0.15, 0.7)
    assert sorted(halos) == sorted([f"forward{i}" for i in range(L)] + [f"backward{i}" for i in range(L)])
    indptr, indices, base = G.global_from_layouts(lays)
    mono_logits, mono_grads = G.monolithic(indptr, indices, np.concatenate(xs), P, np.concatenate(Gs), L, 0.15, 0.7)
    assert _rel(np.concatenate(logits), mono_logits) <= 1e-10
    for k in P:
        assert _rel(grads[k], mono_grads[k]) <= 1e-10, k


def test_gcnii_partitions_are_gcn_partitions():
    """GCNII weighs halo rows with the GCN scores (its weights are the GCN norms times 1 - alpha)."""
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    spec = SynthSpec(name="gcnii", num_nodes=500, num_edges=5000, num_parts=2, num_feats=4, num_classes=3,
                     cross_fraction=0.2, community_size=32, seed=3)
    a = prepare_all_in_process(spec, DistGNNType.DistGCNII)
    b = prepare_all_in_process(spec, DistGNNType.DistGCN)
    for x, y in zip(a, b):
        assert np.array_equal(x.indices, y.indices) and x.scores.keys() == y.scores.keys()
        for p in x.scores:
            assert np.array_equal(x.scores[p][0], y.scores[p][0]) and np.array_equal(x.scores[p][1], y.scores[p][1])


@pytest.mark.parametrize("L", [3, 11])
def test_key_dims(L):
    from adaqp_b200.communicator.p2p import appnp_key_dims, key_dim, layer_index
    dims = appnp_key_dims(256, L)
    assert list(dims) == ([f"test{i}" for i in range(L)] + [f"forward{i}" for i in range(L)]
                          + [f"backward{i}" for i in range(L)])
    assert set(dims.values()) == {256}
    last = L - 1
    assert layer_index(f"forward{last}") == last and key_dim(f"test{last}", [256] * L) == 256
    if L == 11:
        assert "forward10" in dims and "test10" in dims and "backward10" in dims
    from adaqp_b200.assigner.assigner import Assigner
    a = Assigner(100, 256, 3, 10, "uniform", 8, {}, 100, 0.5, 50, key_dims=dims)
    got = a.get_assignment({1: (0, 5)})
    assert sorted(got) == sorted([f"forward{i}" for i in range(L)] + [f"backward{i}" for i in range(L)])


def test_model_refuses_bad_parameters():
    from adaqp_b200.model.distGCNII import gcnii_beta, gcnii_params
    assert gcnii_params(8, 0.1, 0.5) == (8, 0.1, 0.5) and gcnii_params(3.0, 0, 1) == (3, 0.0, 1.0)
    assert gcnii_params(1, 1, 2.5) == (1, 1.0, 2.5)
    for args in ((0, 0.1, 0.5), (2.5, 0.1, 0.5), (True, 0.1, 0.5), (-1, 0.1, 0.5), ("8", 0.1, 0.5),
                 (8, -0.1, 0.5), (8, 1.1, 0.5), (8, float("nan"), 0.5), (8, True, 0.5),
                 (8, 0.1, 0), (8, 0.1, -1), (8, 0.1, float("nan")), (8, 0.1, float("inf")), (8, 0.1, "0.5")):
        with pytest.raises(ValueError):
            gcnii_params(*args)
    assert abs(gcnii_beta(0.5, 1) - np.log(1.5)) < 1e-15 and abs(gcnii_beta(0.5, 8) - np.log(0.5 / 8 + 1)) < 1e-15


def test_model_parameter_names_and_init():
    from adaqp_b200.model.distGCNII import DistGCNII
    torch.manual_seed(0)
    m = DistGCNII(100, 64, 47, 0.5, layers=3)
    names = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert names == {"lins.0.weight": (100, 64), "lins.0.bias": (64,), "lins.1.weight": (64, 47), "lins.1.bias": (47,),
                     "convs.0.weight": (64, 64), "convs.1.weight": (64, 64), "convs.2.weight": (64, 64)}
    assert all(float(v.abs().max()) == 0.0 for k, v in m.state_dict().items() if k.endswith("bias"))
    bound = np.sqrt(6.0 / 128)                      # xavier_uniform_ of a 64 x 64 weight
    w = m.convs[1].weight.detach()
    assert float(w.abs().max()) <= bound and float(w.std()) > 0.5 * bound / np.sqrt(3)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _refusal_worker(port, tmp, layers, alpha, theta, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": "0", "WORLD_SIZE": "1",
                       "LOCAL_RANK": "0", "ADAQP_DEVICE": "cpu", "ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": "0.001"})
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    args = Namespace(dataset="reddit", num_parts=1, backend="gloo", init_method="env://", model_name="gcnii",
                     mode="Vanilla", assign_scheme="uniform", logger_level="WARNING", num_epoches=1,
                     exp_path=f"{tmp}/exp", gcnii_layers=layers, gcnii_alpha=alpha, gcnii_theta=theta)
    try:
        Trainer(args)
        out.put(("no error", ""))
    except Exception as e:                      # noqa: BLE001 - the type and message are what is checked
        out.put((type(e).__name__, str(e)))


@pytest.mark.parametrize("layers,alpha,theta,want,text", [(0, 0.1, 0.5, "ValueError", "gcnii_layers=0"),
                                                          (2.5, 0.1, 0.5, "ValueError", "not an integer"),
                                                          (8, 1.1, 0.5, "ValueError", "outside [0, 1]"),
                                                          (8, 0.1, -1.0, "ValueError", "gcnii_theta"),
                                                          (8, 0.1, 0.5, "NotImplementedError", "p2p transport only")])
def test_trainer_refuses(layers, alpha, theta, want, text):
    """Bad L / alpha / theta and the CPU gloo plumbing mode are refused before any partition is loaded."""
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    with tempfile.TemporaryDirectory() as tmp:
        p = ctx.Process(target=_refusal_worker, args=(_free_port(), tmp, layers, alpha, theta, out))
        p.start()
        p.join(timeout=300)
        assert p.exitcode == 0
        kind, msg = out.get(timeout=5)
    assert kind == want and text in msg, (kind, msg)


# ----------------------------------------------------------------------------- checkpoint field
def _cfg(model_name, layers=8, alpha=0.1, theta=0.5):
    return {"data": {"num_feats": 100, "num_classes": 47},
            "model": {"num_layers": 3, "hidden_dim": 256, "aggregator_type": "mean", "gat_heads": 4,
                      "appnp_k": 10, "appnp_alpha": 0.1, "gcnii_layers": layers, "gcnii_alpha": alpha,
                      "gcnii_theta": theta},
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
    gcnii = ck.run_fields(_cfg("gcnii"), appnp_key_dims(256, 8))
    assert gcnii["propagation"] == {"layers": 8, "alpha": 0.1, "theta": 0.5}
    assert ck.run_fields(_cfg("appnp"), appnp_key_dims(47, 10))["propagation"] == {"k": 10, "alpha": 0.1}
    assert ck.run_fields(_cfg("gcn"), None)["propagation"] is None
    digest = {"n_inner": 10, "n_halo": 3, "send_idx": {"1": [0, 4]}, "csr_sha256": "ab"}
    _fake_checkpoint(str(tmp_path / "gcnii"), gcnii, [digest, digest])
    assert ck.resume_error(str(tmp_path / "gcnii"), gcnii, digest, 0, 5) is None
    for layers, alpha, theta in ((8, 0.1, 1.0), (8, 0.2, 0.5)):
        other = ck.run_fields(_cfg("gcnii", layers, alpha, theta), appnp_key_dims(256, layers))
        err = ck.resume_error(str(tmp_path / "gcnii"), other, digest, 0, 5)
        assert isinstance(err, ValueError) and "'propagation'" in str(err), err
    # another L changes the key table as well: refused either way
    other = ck.run_fields(_cfg("gcnii", 4), appnp_key_dims(256, 4))
    assert isinstance(ck.resume_error(str(tmp_path / "gcnii"), other, digest, 0, 5), ValueError)
    # predicting with another theta is refused; the model fields alone would match
    other = ck.run_fields(_cfg("gcnii", 8, 0.1, 1.0), appnp_key_dims(256, 8))
    with pytest.raises(ValueError, match="propagation"):
        ck.load_weights(str(tmp_path / "gcnii"), None, other)


# ----------------------------------------------------------------------------- main.py flags
def test_main_flags_parse(monkeypatch):
    import importlib
    monkeypatch.setattr(sys, "argv", ["main.py", "--model_name", "gcnii", "--gcnii_layers", "11", "--gcnii_alpha", "0.2",
                                      "--gcnii_theta", "1.5"])
    main = importlib.import_module("main")
    a = main.parse()
    assert (a.model_name, a.gcnii_layers, a.gcnii_alpha, a.gcnii_theta) == ("gcnii", 11, 0.2, 1.5)
    monkeypatch.setattr(sys, "argv", ["main.py"])
    a = main.parse()
    assert a.gcnii_layers is None and a.gcnii_alpha is None and a.gcnii_theta is None

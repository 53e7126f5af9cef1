"""Correct & Smooth without a GPU: the float64 oracle against an independent dense restatement of the algorithm, the
distributed protocol against the whole-graph run, the parameter and configuration refusals, the exchange key table
and argument rejection by the C entry points."""
import os
import socket
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import cs_oracle as CS  # noqa: E402


def _graph(n, deg, seed, isolated=0):
    """Random symmetric graph with one self-loop per node; the last `isolated` nodes have only their self-loop."""
    import scipy.sparse as sp
    rng = np.random.RandomState(seed)
    m = n * deg // 2
    a, b = rng.randint(0, n - isolated, m), rng.randint(0, n - isolated, m)
    A = sp.coo_matrix((np.ones(2 * m), (np.r_[a, b], np.r_[b, a])), shape=(n, n)).tocsr()
    A.setdiag(0)
    A.eliminate_zeros()
    A = (A + sp.eye(n)).tocsr()
    A.sort_indices()
    return A.indptr.astype(np.int64), A.indices.astype(np.int64)


def _dense_cs(indptr, indices, z, y, k1, a1, k2, a2, scale):
    """The algorithm of DESIGN §16 step by step on dense matrices, written apart from the oracle."""
    n, C = z.shape
    deg = np.diff(indptr).astype(np.float64)
    A = np.zeros((n, n))
    for v in range(n):
        for u in indices[indptr[v]:indptr[v + 1]]:
            A[v, u] += deg[u] ** -0.5 * deg[v] ** -0.5
    lab = y >= 0
    Y = np.zeros((n, C))
    for v in range(n):
        if lab[v]:
            Y[v, y[v]] = 1.0
    P = np.exp(z - z.max(1, keepdims=True))
    P /= P.sum(1, keepdims=True)
    E0 = (Y - P) * lab[:, None]
    sigma = np.abs(E0).sum() / lab.sum()
    E = E0.copy()
    for _ in range(k1):
        T = a1 * (A @ E) + (1 - a1) * E0
        if scale is None:
            E = np.minimum(np.maximum(T, -1.0), 1.0)
        else:
            T[lab] = E0[lab]
            E = T
    if scale is None:
        s = np.ones(n)
        for v in range(n):
            l1 = np.abs(E[v]).sum()
            if l1 > 0 and sigma / l1 <= 1000:
                s[v] = sigma / l1
    else:
        s = np.full(n, scale)
    G0 = P + s[:, None] * E
    G0[lab] = Y[lab]
    G = G0
    for _ in range(k2):
        G = np.minimum(np.maximum(a2 * (A @ G) + (1 - a2) * G0, 0.0), 1.0)
    return G, E, s


@pytest.mark.parametrize("scale", [None, 0.7, 2.5])
@pytest.mark.parametrize("alpha", [0.0, 0.8, 1.0])
def test_oracle_matches_dense_restatement(alpha, scale):
    n, C = 60, 5
    indptr, indices = _graph(n, 5, seed=int(alpha * 10) + 3, isolated=4)
    rng = np.random.RandomState(7)
    z = rng.randn(n, C) * 2
    y = np.where(rng.rand(n) < 0.3, rng.randint(0, C, n), -1)
    y[-4:] = -1                               # isolated and unlabelled: their error rows stay zero
    k1, k2 = 6, 5
    res = CS.monolithic(indptr, indices, z, y, k1, alpha, k2, alpha, scale)
    G, E, s = _dense_cs(indptr, indices, z, y, k1, alpha, k2, alpha, scale)
    assert np.abs(res["g"][0] - G).max() <= 1e-12
    assert np.abs(res["e"][0] - E).max() <= 1e-12
    zero = np.abs(res["e"][0]).sum(1) == 0
    assert zero[-4:].all()
    if scale is None:
        # rows with a zero error get scale 1, not 0 / 0
        assert np.array_equal(CS.autoscale(res["sigma"], res["e"][0])[zero], np.ones(int(zero.sum())))
        assert np.isfinite(res["g"][0]).all()
    assert (res["g"][0] >= 0).all() and (res["g"][0] <= 1).all()
    lab = y >= 0
    assert np.array_equal(res["g0"][0][lab], CS.onehot(y, C)[lab])


def test_autoscale_cutoff():
    e = np.array([[0.0, 0.0], [1e-6, 0.0], [0.5, -0.5], [2e-3, 0.0]])
    s = CS.autoscale(1.5, e)
    assert s[0] == 1.0 and s[1] == 1.0 and s[2] == 1.5 and s[3] == 750.0


@pytest.mark.parametrize("W,scale", [(2, None), (3, None), (2, 1.3), (3, 0.9)])
def test_distributed_oracle_equals_monolithic(W, scale):
    """Every inner row's result equals the whole-graph run to 1e-10: the protocol (each step exchanges the rows it
    propagates; sigma sums every rank's labelled errors) loses nothing."""
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    C = 6
    spec = SynthSpec(name="cs", num_nodes=900, num_edges=900 * 10, num_parts=W, num_feats=8, num_classes=C,
                     cross_fraction=0.25, community_size=64, seed=W + 5)
    lays = prepare_all_in_process(spec, DistGNNType.DistGCN)
    assert sum(L.n_halo for L in lays) > 0
    rng = np.random.RandomState(W)
    zs = [rng.randn(L.n_inner, C) * 2 for L in lays]
    ys = [np.where(np.asarray(L.train_mask, bool), np.asarray(L.label, np.int64) % C, -1) for L in lays]
    assert sum(int((y >= 0).sum()) for y in ys) > 0
    dist = CS.distributed(lays, zs, ys, 7, 0.8, 6, 0.7, scale)
    indptr, indices, _ = CS.global_from_layouts(lays)
    mono = CS.monolithic(indptr, indices, np.concatenate(zs), np.concatenate(ys), 7, 0.8, 6, 0.7, scale)
    assert abs(dist["sigma"] - mono["sigma"]) <= 1e-12 * max(mono["sigma"], 1.0)
    for f in ("e", "g"):
        assert np.abs(np.concatenate(dist[f]) - mono[f][0]).max() <= 1e-10, f


# ----------------------------------------------------------------------------- parameters and refusals
def test_cs_params():
    from adaqp_b200.cs import cs_params
    p = cs_params()
    assert (p.correct_layers, p.correct_alpha, p.smooth_layers, p.smooth_alpha, p.scale) == (50, 0.8, 50, 0.8, None)
    assert p.as_dict() == {"correct_layers": 50, "correct_alpha": 0.8, "smooth_layers": 50, "smooth_alpha": 0.8,
                           "scale": "auto"}
    q = cs_params(3.0, 0, 1, 1, "2.5")
    assert (q.correct_layers, q.correct_alpha, q.smooth_layers, q.smooth_alpha, q.scale) == (3, 0.0, 1, 1.0, 2.5)
    assert cs_params(scale=0.5).scale == 0.5


@pytest.mark.parametrize("kw", [dict(correct_layers=0), dict(smooth_layers=-1), dict(correct_layers=2.5),
                                dict(smooth_layers="3"), dict(correct_layers=True), dict(correct_alpha=-0.1),
                                dict(smooth_alpha=1.01), dict(correct_alpha=float("nan")), dict(smooth_alpha="0.5"),
                                dict(scale=0), dict(scale=-1.0), dict(scale=float("inf")), dict(scale="nan"),
                                dict(scale="big"), dict(scale=None), dict(scale=True)])
def test_cs_params_refusals(kw):
    from adaqp_b200.cs import cs_params
    with pytest.raises(ValueError):
        cs_params(**kw)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _refusal_worker(port, tmp, dataset, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": "0", "WORLD_SIZE": "1",
                       "LOCAL_RANK": "0", "ADAQP_DEVICE": "cpu", "ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": "0.001"})
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    args = Namespace(dataset=dataset, num_parts=1, backend="gloo", init_method="env://", model_name="gcn",
                     mode="Vanilla", assign_scheme="uniform", logger_level="WARNING", num_epoches=1,
                     exp_path=f"{tmp}/exp", correct_and_smooth=True, predict_out=f"{tmp}/pred")
    try:
        Trainer(args)
        out.put(("no error", ""))
    except Exception as e:                      # noqa: BLE001 - the type and message are what is checked
        out.put((type(e).__name__, str(e)))


@pytest.mark.parametrize("dataset,want,text", [("yelp", "ValueError", "softmax"),
                                               ("amazonProducts", "ValueError", "multilabel"),
                                               ("reddit", "NotImplementedError", "p2p transport only")])
def test_trainer_refuses(dataset, want, text):
    """A multilabel dataset and the CPU gloo plumbing mode are refused before any partition is loaded."""
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    with tempfile.TemporaryDirectory() as tmp:
        p = ctx.Process(target=_refusal_worker, args=(_free_port(), tmp, dataset, out))
        p.start()
        p.join(timeout=300)
        assert p.exitcode == 0
        kind, msg = out.get(timeout=5)
    assert kind == want and text in msg, (kind, msg)


def test_cli_needs_predict_out():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "main.py"), "--correct_and_smooth"], cwd=ROOT,
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 2 and "--correct_and_smooth needs --predict_out" in r.stderr, r.stderr[-2000:]


# ----------------------------------------------------------------------------- key table
def _config(model_name, agg="mean"):
    return {"data": {"num_feats": 100, "num_classes": 47, "is_multilabel": False},
            "model": {"num_layers": 3, "hidden_dim": 256, "aggregator_type": agg, "gat_heads": 4, "dropout_rate": 0.5,
                      "use_norm": True, "appnp_k": 10, "appnp_alpha": 0.1, "gcnii_layers": 8, "gcnii_alpha": 0.1,
                      "gcnii_theta": 0.5},
            "runtime": {"dataset": "ogbn-products", "model_name": model_name, "num_parts": 2, "mode": "AdaQP",
                        "assign_scheme": "random"}}


@pytest.mark.parametrize("model_name,agg", [(m, "mean") for m in ("gcn", "sage", "gat", "gatv2", "appnp", "gcnii")]
                         + [("sage", "pool"), ("sage", "gcn")])
def test_key_table(model_name, agg):
    from adaqp_b200.communicator.p2p import CS_KEY, SlabLayout, layer_key_dims
    from adaqp_b200.model.registry import MODELS, buffer_shape
    from adaqp_b200.trainer import checkpoint as ck
    from adaqp_b200.trainer.trainer import exchange_key_dims
    cfg = _config(model_name, agg)
    spec = MODELS[model_name]
    own = spec.key_dims(cfg)
    # without C&S: the table the exchange is built with today (None: PeerExchange's layer_key_dims(buffer_shape))
    assert exchange_key_dims(cfg, own, False) is own
    with_cs = exchange_key_dims(cfg, own, True)
    today = own if own is not None else layer_key_dims(buffer_shape(cfg, None))
    assert with_cs == {**today, CS_KEY: 47} and list(with_cs)[:-1] == list(today) and list(with_cs)[-1] == CS_KEY
    assert buffer_shape(cfg, with_cs) == buffer_shape(cfg, own)
    lay = SlabLayout.build(2, list(with_cs), with_cs, {1: 10}, 10)
    assert (CS_KEY, 1) not in lay.qdata_off and CS_KEY in lay.halo_off
    # what checkpoints record does not see the C&S flags
    flags = {"correct_and_smooth": True, "cs_correct_layers": 3, "cs_correct_alpha": 0.5, "cs_smooth_layers": 4,
             "cs_smooth_alpha": 0.6, "cs_scale": "auto"}
    cfg_cs = dict(cfg, runtime=dict(cfg["runtime"], **flags))
    assert ck.run_fields(cfg_cs, own) == ck.run_fields(cfg, own)


# ----------------------------------------------------------------------------- C entry points
@pytest.fixture(scope="module")
def lib():
    from adaqp_b200 import _lib, build
    build.build()
    return _lib.load()


def test_entry_points_reject_bad_arguments(lib):
    import ctypes as C
    err = lambda: lib.adaqp_last_error().decode()  # noqa: E731
    inf = float("inf")
    p = C.c_void_p(8)                           # never dereferenced: every call below fails its checks first
    f = lib.adaqp_cs_prop_f32
    # (indptr, indices, x0, ld0, n_split, x1, ld1, pre, post, scale, alpha, tele, ldt, y, fix, ldf, post_mode, lo, hi,
    #  row_begin, row_end, C, out, ldo, stream)
    ok = [p, p, p, 47, 100, None, 0, None, None, 0.8, 0.2, p, 47, None, None, 0, 0, -1.0, 1.0, 0, 10, 47, p, 47, None]

    def call(**kw):
        a = list(ok)
        names = ["indptr", "indices", "x0", "ld0", "n_split", "x1", "ld1", "pre", "post", "scale", "alpha", "tele",
                 "ldt", "y", "fix", "ldf", "post_mode", "lo", "hi", "row_begin", "row_end", "C", "out", "ldo"]
        for k, v in kw.items():
            a[names.index(k)] = v
        return f(*a)

    assert call(C=0) == -1 and "C=0" in err()
    assert call(C=1025, ld0=1025, ldo=1025) == -1 and "C=1025" in err()
    assert call(row_begin=5, row_end=2) == -1 and "row range" in err()
    assert call(row_end=101) == -1 and "row range" in err()
    assert call(row_begin=-1) == -1 and "row range" in err()
    assert call(lo=1.0, hi=-1.0) == -1 and "lo=" in err()
    assert call(lo=float("nan")) == -1 and "lo=" in err()
    assert call(post_mode=2) == -1 and "post_mode" in err()
    assert call(indptr=None) == -1 and "null pointer" in err()
    assert call(out=None) == -1 and "null pointer" in err()
    assert call(post_mode=1, y=p, fix=None) == -1 and "null pointer" in err()
    assert call(post_mode=1, y=None, fix=p) == -1 and "null pointer" in err()
    assert call(row_begin=4, row_end=4, indptr=None, lo=-inf, hi=inf) == 0      # an empty range is a no-op
    g = lib.adaqp_cs_init_f32
    # (z, ldz, y, rows, C, yhat, ldy, e0, lde, partials, n_partials, stream)
    assert g(p, 0, p, 10, 0, p, 0, p, 0, p, 8, None) == -1 and "C=0" in err()
    assert g(p, 1025, p, 10, 1025, p, 1025, p, 1025, p, 8, None) == -1 and "C=1025" in err()
    assert g(p, 47, p, -1, 47, p, 47, p, 47, p, 8, None) == -1 and "bad shape" in err()
    assert g(p, 47, p, 10, 47, p, 47, p, 47, p, 0, None) == -1 and "n_partials" in err()
    assert g(None, 47, p, 10, 47, p, 47, p, 47, p, 8, None) == -1 and "null pointer" in err()
    assert g(p, 47, p, 10, 47, p, 47, p, 47, None, 8, None) == -1 and "null pointer" in err()
    h = lib.adaqp_cs_combine_f32
    # (yhat, ldy, e, lde, y, rows, C, autoscale, value, g0, ldg, stream)
    assert h(p, 47, p, 47, p, 10, 1025, 1, 0.5, p, 47, None) == -1 and "C=1025" in err()
    assert h(p, 47, p, 47, p, -3, 47, 1, 0.5, p, 47, None) == -1 and "bad shape" in err()
    for auto, v in ((0, 0.0), (0, -1.0), (0, inf), (0, float("nan")), (1, -0.5), (1, inf)):
        assert h(p, 47, p, 47, p, 10, 47, auto, v, p, 47, None) == -1 and ("scale" in err() or "sigma" in err())
    assert h(p, 47, None, 47, p, 10, 47, 1, 0.5, p, 47, None) == -1 and "null pointer" in err()
    assert h(p, 47, p, 47, p, 10, 47, 0, 1.5, None, 47, None) == -1 and "null pointer" in err()

"""Dataset readers, partition assembly, host initial partitioner and the partitioner's boundaries -- no GPU.

* each reader on a tiny fixture in its raw format: restated semantics, self-loops removed then one per node,
  duplicate edges collapsed, asymmetric input refused, missing files named;
* raw_partitions + the shared layout chain on the synthetic graph cut along its planted blocks equal
  prepare_all_in_process field by field (and after the file round trip);
* the host greedy graph-growing recursive bisection;
* the new C entry points reject bad arguments before any CUDA call; graph_partition.py skips an existing
  partition directory and raises, without falling back, when no GPU is visible.
"""
import dataclasses
import gzip
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adaqp_b200.helper import DistGNNType
from adaqp_b200.helper import dataset as ds
from adaqp_b200.manager.layout import layouts_from_raw, prepare_all_in_process, raw_partitions
from adaqp_b200.manager.partition_synth import SynthSpec, global_graph
from adaqp_b200 import partition as gp


# ----------------------------------------------------------------------------- readers
def _gz_csv(path, rows):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with gzip.open(path, "wt") as f:
        for r in rows:
            f.write(",".join(str(x) for x in np.atleast_1d(r)) + "\n")


def _edges(g):
    rows = np.repeat(np.arange(g.num_nodes), np.diff(g.indptr))
    return set(zip(rows.tolist(), g.indices.tolist()))


def _check_common(g, n):
    assert g.indptr.dtype == np.int64 and g.indices.dtype == np.int32 and g.feat.dtype == np.float32
    e = _edges(g)
    assert all((v, u) in e for u, v in e), "symmetric"
    assert all((v, v) in e for v in range(n)), "one self-loop per node"
    assert len(e) == g.indices.size, "no multi-edges"
    assert np.array_equal(g.degrees, np.diff(g.indptr))


def test_ogbn_products_reader(tmp_path):
    d = tmp_path / "ogbn_products"
    n = 6
    edge = [(0, 1), (1, 2), (2, 2), (3, 4), (0, 1), (4, 5)]      # a self-loop and a duplicate
    _gz_csv(str(d / "raw" / "edge.csv.gz"), edge)
    feat = np.arange(n * 3, dtype=np.float32).reshape(n, 3) / 7
    _gz_csv(str(d / "raw" / "node-feat.csv.gz"), feat.tolist())
    _gz_csv(str(d / "raw" / "node-label.csv.gz"), [[x] for x in [3, 1, 4, 1, 5, 9]])
    for s, idx in (("train", [0, 1, 2]), ("valid", [3]), ("test", [4, 5])):
        _gz_csv(str(d / "split" / "sales_ranking" / f"{s}.csv.gz"), [[i] for i in idx])
    g = ds.load_dataset("ogbn-products", str(tmp_path))
    _check_common(g, n)
    e = _edges(g)
    assert (1, 0) in e and (0, 1) in e and (5, 4) in e          # inverse edges added
    assert g.n_collapsed == 2                                    # (0,1) twice, in both directions
    assert len(e) == n + 2 * 4
    assert np.allclose(g.feat, feat, atol=1e-6)
    assert g.label.dtype == np.int64 and g.label.tolist() == [3, 1, 4, 1, 5, 9]
    assert g.train_mask.tolist() == [1, 1, 1, 0, 0, 0] and g.val_mask.tolist() == [0, 0, 0, 1, 0, 0]
    assert g.test_mask.tolist() == [0, 0, 0, 0, 1, 1]


def _reddit_fixture(root, A):
    d = os.path.join(root, "reddit")
    os.makedirs(d, exist_ok=True)
    n = A.shape[0]
    np.savez(os.path.join(d, "reddit_data.npz"), feature=np.ones((n, 4), np.float32) * np.arange(n)[:, None],
             label=np.arange(n) % 3, node_types=np.array([1, 2, 3, 1, 1][:n]))
    sp.save_npz(os.path.join(d, "reddit_graph.npz"), A)


def test_reddit_reader_and_asymmetric_refusal(tmp_path):
    u = np.array([0, 1, 1, 2, 3, 3, 0, 4])
    v = np.array([1, 0, 2, 1, 3, 4, 1, 3])                       # self-loop (3,3), duplicate (0,1)
    A = sp.coo_matrix((np.ones(u.size), (u, v)), shape=(5, 5))
    _reddit_fixture(str(tmp_path / "a"), A)
    g = ds.load_reddit(str(tmp_path / "a"))
    _check_common(g, 5)
    assert g.n_collapsed == 1
    assert g.train_mask.tolist() == [1, 0, 0, 1, 1] and g.val_mask.tolist() == [0, 1, 0, 0, 0]
    assert g.test_mask.tolist() == [0, 0, 1, 0, 0] and g.label.tolist() == [0, 1, 2, 0, 1]
    B = sp.coo_matrix((np.ones(2), ([0, 1], [1, 2])), shape=(5, 5))
    _reddit_fixture(str(tmp_path / "b"), B)
    with pytest.raises(NotImplementedError):
        ds.load_reddit(str(tmp_path / "b"))


def _saint_fixture(root, name, A, feats, class_map, role, save_csr_arrays=False):
    d = os.path.join(root, name)
    os.makedirs(d, exist_ok=True)
    if save_csr_arrays:
        A = sp.csr_matrix(A)
        np.savez(os.path.join(d, "adj_full.npz"), data=A.data, indices=A.indices, indptr=A.indptr, shape=A.shape)
    else:
        sp.save_npz(os.path.join(d, "adj_full.npz"), sp.csr_matrix(A))
    np.save(os.path.join(d, "feats.npy"), feats)
    with open(os.path.join(d, "class_map.json"), "w") as f:
        json.dump(class_map, f)
    with open(os.path.join(d, "role.json"), "w") as f:
        json.dump(role, f)


def _sym(n, rng, m):
    u, v = rng.integers(0, n, m), rng.integers(0, n, m)
    return sp.coo_matrix((np.ones(2 * m), (np.r_[u, v], np.r_[v, u])), shape=(n, n))


def test_yelp_reader_scaling_and_label_order(tmp_path):
    rng = np.random.default_rng(0)
    n = 8
    feats = rng.standard_normal((n, 5)) * 3 + 1
    feats[:, 2] = 4.0                                            # zero-std column keeps scale 1
    class_map = {str(i): [int(i % 2), int(i % 3 == 0)] for i in [5, 0, 7, 1, 2, 3, 4, 6]}
    role = {"tr": [0, 1, 2, 3, 4], "va": [5], "te": [6, 7]}
    _saint_fixture(str(tmp_path), "yelp", _sym(n, rng, 12), feats, class_map, role)
    g = ds.load_dataset("yelp", str(tmp_path))
    _check_common(g, n)
    tr = feats[:5]
    want = (feats - tr.mean(0)) / np.where(tr.std(0) == 0, 1.0, tr.std(0))
    assert np.allclose(g.feat, want, atol=1e-5)
    try:
        from sklearn.preprocessing import StandardScaler
        assert np.allclose(g.feat, StandardScaler().fit(tr).transform(feats), atol=1e-5)
    except ImportError:
        pass
    # class_map FILE order, as the reference's list(class_map.values())
    assert g.label.dtype == np.float32 and np.array_equal(g.label, np.array(list(class_map.values()), np.float32))
    assert g.train_mask.sum() == 5 and g.val_mask[5] and g.test_mask[6] and g.test_mask[7]


def test_amazon_products_reader_label_rows(tmp_path):
    rng = np.random.default_rng(1)
    n = 7
    feats = rng.standard_normal((n, 3)).astype(np.float32)
    class_map = {str(i): [int(i == 1), int(i > 3), 1] for i in [6, 2, 0, 5, 1, 4, 3]}
    role = {"tr": [0, 1, 2], "va": [3, 4], "te": [5, 6]}
    _saint_fixture(str(tmp_path), "amazonProducts", _sym(n, rng, 10), feats, class_map, role, save_csr_arrays=True)
    g = ds.load_dataset("amazonProducts", str(tmp_path))
    _check_common(g, n)
    for k, v in class_map.items():
        assert g.label[int(k)].tolist() == v                     # row int(key) = class_map[key]
    assert np.array_equal(g.feat, feats)
    assert g.val_mask.tolist() == [0, 0, 0, 1, 1, 0, 0]


@pytest.mark.parametrize("dataset,missing", [
    ("ogbn-products", "ogbn_products/raw/edge.csv.gz"), ("reddit", "reddit/reddit_data.npz"),
    ("yelp", "yelp/adj_full.npz"), ("amazonProducts", "amazonProducts/adj_full.npz")])
def test_missing_file_is_named(dataset, missing, tmp_path):
    with pytest.raises(FileNotFoundError) as e:
        ds.load_dataset(dataset, str(tmp_path))
    assert os.path.join(str(tmp_path), missing) in str(e.value)


# ----------------------------------------------------------------------------- assembly
def _assert_layouts_equal(got, want):
    for f in dataclasses.fields(want):
        a, b = getattr(got, f.name), getattr(want, f.name)
        if isinstance(b, dict):
            assert set(a) == set(b), f.name
            for k in b:
                x, y = a[k], b[k]
                if isinstance(y, tuple) and isinstance(y[0], np.ndarray):
                    assert all(np.array_equal(p, q) for p, q in zip(x, y)), (f.name, k)
                elif isinstance(y, tuple):
                    assert tuple(int(t) for t in x) == tuple(int(t) for t in y), (f.name, k)
                else:
                    assert np.array_equal(x, y), (f.name, k)
        elif isinstance(b, np.ndarray):
            assert np.array_equal(a, b), f.name
        else:
            assert a == b, f.name


@pytest.mark.parametrize("model", [DistGNNType.DistGCN, DistGNNType.DistSAGE])
@pytest.mark.parametrize("W", [2, 4])
def test_raw_partitions_match_the_generators_layout(W, model, tmp_path):
    spec = SynthSpec(name="fixture", num_nodes=2000, num_edges=2000 * 12, num_parts=W, num_feats=16, num_classes=5,
                     cross_fraction=0.2, community_size=64, seed=4)
    want = prepare_all_in_process(spec, model)
    g, part = global_graph(spec)
    # the relabelling must not depend on the order of ids: shuffle the global graph, then cut along the same blocks
    perm = np.random.default_rng(0).permutation(spec.num_nodes)          # new id -> old id
    gs = g.permuted(perm)
    pshuf = part[perm]
    got = layouts_from_raw(raw_partitions(g, part), model)
    from adaqp_b200.manager.graphEngine import read_rank_layout, save_rank_layout
    for a, b in zip(got, want):
        _assert_layouts_equal(a, b)
        _assert_layouts_equal(read_rank_layout(save_rank_layout(a, str(tmp_path), "fixture")), b)
    # shuffled ids: same blocks, same per-rank inner node SETS and halo sizes
    got_s = layouts_from_raw(raw_partitions(gs, pshuf), model)
    for a, b in zip(got_s, want):
        assert (a.n_inner, a.n_halo, a.indices.size) == (b.n_inner, b.n_halo, b.indices.size)


# ----------------------------------------------------------------------------- host initial partitioner
def _csr(n, u, v):
    A = sp.coo_matrix((np.ones(2 * len(u)), (np.r_[u, v], np.r_[v, u])), shape=(n, n)).tocsr()
    A.sum_duplicates()
    A.data[:] = 1
    return A


def test_two_cliques_cut_zero():
    m = 20
    iu = np.triu_indices(m, 1)
    A = _csr(2 * m, np.r_[iu[0], iu[0] + m], np.r_[iu[1], iu[1] + m])
    part = gp.initial_partition(A.indptr, A.indices, A.data, np.ones(2 * m), 2, seed=3)
    assert gp.edge_cut(A.indptr, A.indices, part) == 0
    assert np.bincount(part).tolist() == [m, m]


def test_path_graph_k3_balanced_and_seeded():
    n = 301
    A = _csr(n, np.arange(n - 1), np.arange(1, n))
    part = gp.initial_partition(A.indptr, A.indices, A.data, np.ones(n), 3, seed=1)
    sizes = np.bincount(part, minlength=3)
    assert sizes.min() >= 1 and sizes.max() <= gp.max_block_weight(n, 3), sizes
    again = gp.initial_partition(A.indptr, A.indices, A.data, np.ones(n), 3, seed=1)
    assert np.array_equal(part, again)


def test_max_block_weight():
    assert gp.max_block_weight(100, 1) == 103 and gp.max_block_weight(122451, 8) == 15766
    with pytest.raises(ValueError):
        gp.check_k(10, 65)
    with pytest.raises(ValueError):
        gp.check_k(3, 4)


# ----------------------------------------------------------------------------- boundaries
@pytest.fixture(scope="module")
def lib():
    from adaqp_b200 import build, _lib
    build.build()
    return _lib.load()


def test_abi_rejects_bad_arguments_without_gpu(lib):
    EINVAL = -1
    for k in (0, 65, -3):
        assert lib.adaqp_lp_rate_blocks(None, None, None, None, 10, None, None, k, 5, 0, 0, 0, 0,
                                        None, None, None, None) == EINVAL
        assert b"k=" in lib.adaqp_last_error()
    assert lib.adaqp_lp_rate_blocks(None, None, None, None, -1, None, None, 4, 5, 0, 0, 0, 0,
                                    None, None, None, None) == EINVAL
    assert lib.adaqp_lp_rate_blocks(None, None, None, None, 10, None, None, 4, 5, 0, 0, 0, 0,
                                    None, None, None, None) == EINVAL          # null pointers
    assert lib.adaqp_lp_rate_clusters(None, None, None, None, -5, None, None, 1, None, 0, None, 0, 0, 0, 0,
                                      None, None, None, None) == EINVAL
    assert lib.adaqp_lp_rate_clusters(None, None, None, None, 5, None, None, 1, None, 0, None, 0, 0, 0, 2,
                                      None, None, None, None) == EINVAL
    assert lib.adaqp_lp_apply(None, -1, None, None, None, None, None, 1, None, None) == EINVAL
    assert lib.adaqp_lp_apply(None, 3, None, None, None, None, None, 1, None, None) == EINVAL
    assert lib.adaqp_lp_rebalance_select(None, -2, None, None, None, None, 1, None, None) == EINVAL
    assert lib.adaqp_contract_edges(None, None, -1, None, None, None) == EINVAL
    assert lib.adaqp_contract_edges(None, None, 4, None, None, None) == EINVAL


def _run_cli(tmp_path, env_extra, *args):
    env = dict(os.environ, **env_extra)
    return subprocess.run([sys.executable, os.path.join(ROOT, "graph_partition.py"), *args], cwd=str(tmp_path),
                          env=env, capture_output=True, text=True, timeout=600)


def test_cli_skips_existing_partition_dir(tmp_path):
    (tmp_path / "pd" / "reddit" / "2part").mkdir(parents=True)
    r = _run_cli(tmp_path, {}, "--partition_dir", "pd", "--raw_dir", "nowhere")
    assert r.returncode == 0, r.stderr
    assert "nothing to do" in r.stdout
    assert os.listdir(tmp_path / "pd" / "reddit" / "2part") == []


def test_cli_without_gpu_raises(tmp_path):
    r = _run_cli(tmp_path, {"CUDA_VISIBLE_DEVICES": ""}, "--partition_dir", "pd", "--raw_dir", "nowhere")
    assert r.returncode != 0
    assert "no CUDA device" in r.stderr
    assert not (tmp_path / "pd" / "reddit" / "2part").exists()

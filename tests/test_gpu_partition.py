"""GPU multilevel partitioner (csrc/partition.cu + adaqp_b200/partition.py) and the two-step workflow.

* one clustering and one refinement sub-round equal the numpy oracle (oracle/partition_oracle.py) on a random
  graph with a hub, labels and label weights exactly;
* the same seed gives the identical `part`; another seed still gives a valid partition;
* quality on the products-shaped synthetic graph (scale 0.05, node ids shuffled) at W = 2, 4, 8;
* edge cases: isolated vertices, more blocks than components, a 100 000-leaf star, k = 1, 3, 64;
* end to end: graph_partition.py on an ogbn-products-format fixture, then two ranks train from the files.
"""
import gzip
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import scipy.sparse as sp
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from adaqp_b200 import partition as gp
from oracle import partition_oracle as PO

DEV = torch.device("cuda:0")


def _sym_csr(n, u, v, w=None):
    w = np.ones(len(u), np.int64) if w is None else w
    A = sp.coo_matrix((np.r_[w, w], (np.r_[u, v], np.r_[v, u])), shape=(n, n)).tocsr()
    A.setdiag(0)
    A.eliminate_zeros()
    A.sort_indices()
    return A


def _hub_graph(seed=0, n=900, m=2500, hub_deg=700):
    rng = np.random.default_rng(seed)
    u, v = rng.integers(0, n, m), rng.integers(0, n, m)
    hu = np.zeros(hub_deg, np.int64)
    hv = rng.choice(np.arange(1, n), hub_deg, replace=False)
    w = rng.integers(1, 4, m + hub_deg)
    A = _sym_csr(n, np.r_[u, hu], np.r_[v, hv], w)
    assert np.diff(A.indptr)[0] > 256                     # the hub path is exercised
    return A


def test_cluster_and_refine_subrounds_match_the_oracle():
    A = _hub_graph()
    n = A.shape[0]
    rng = np.random.default_rng(5)
    vw = rng.integers(1, 3, n).astype(np.int32)
    g = gp.Graph.from_csr(A.indptr, A.indices, DEV, ew=A.data, vw=vw)
    # clustering: start from a random labelling over 300 clusters, cap 9
    label0 = rng.integers(0, 300, n).astype(np.int32)
    lw0 = np.bincount(label0, weights=vw, minlength=n).astype(np.int64)
    for seed, r, s in [(0, 0, 0), (7, 3, 1), (123456789, 2, 0)]:
        lab, lw = torch.from_numpy(label0).to(DEV), torch.from_numpy(lw0).to(DEV)
        moved = gp.cluster_subround(g, lab, lw, 9, seed, r, s)
        want_l, want_w = PO.lp_subround(A.indptr, A.indices, A.data, vw, label0, lw0, 9, seed, r, s)
        assert moved > 0
        assert np.array_equal(lab.cpu().numpy(), want_l), (seed, r, s)
        assert np.array_equal(lw.cpu().numpy(), want_w), (seed, r, s)
    # refinement: k = 5 blocks
    k = 5
    part0 = rng.integers(0, k, n).astype(np.int32)
    bw0 = np.bincount(part0, weights=vw, minlength=k).astype(np.int64)
    cap = int(bw0.max()) + 12
    for seed, r, s in [(0, 0, 0), (9, 1, 1)]:
        part, bw = torch.from_numpy(part0).to(DEV), torch.from_numpy(bw0).to(DEV)
        moved = gp.refine_subround(g, part, bw, k, cap, seed, r, s)
        want_p, want_b = PO.lp_subround(A.indptr, A.indices, A.data, vw, part0, bw0, cap, seed, r, s)
        assert moved > 0
        assert np.array_equal(part.cpu().numpy(), want_p), (seed, r, s)
        assert np.array_equal(bw.cpu().numpy(), want_b), (seed, r, s)


def _check_valid(indptr, part, k):
    n = indptr.size - 1
    assert part.dtype == np.int32 and part.shape == (n,)
    sizes = np.bincount(part, minlength=k)
    assert sizes.size == k and sizes.min() >= 1, sizes
    assert sizes.max() <= gp.max_block_weight(n, k), (sizes.max(), gp.max_block_weight(n, k))


@pytest.fixture(scope="module")
def products():
    """Products-config synthetic graphs at scale 0.05 (122 451 nodes) per W, node ids shuffled, and planted cuts."""
    import yaml
    from adaqp_b200.manager.partition_synth import global_graph, spec_from_config
    with open(os.path.join(ROOT, "adaqp_b200", "config", "ogbn-products.yaml")) as f:
        cfg = yaml.safe_load(f)
    out = {}
    for W in (2, 4, 8):
        g, planted = global_graph(spec_from_config(cfg, W, 0.05))
        perm = np.random.default_rng(W).permutation(g.num_nodes)
        out[W] = (g.permuted(perm), gp.edge_cut(g.indptr, g.indices, planted))
    return out


def test_determinism_and_other_seed(products):
    g, _ = products[4]
    a = gp.partition(g.indptr, g.indices, 4, seed=0)
    b = gp.partition(g.indptr, g.indices, 4, seed=0)
    assert np.array_equal(a, b)
    c = gp.partition(g.indptr, g.indices, 4, seed=1)
    _check_valid(g.indptr, c, 4)


@pytest.mark.parametrize("W", [2, 4, 8])
def test_quality_on_shuffled_products(products, W):
    g, planted = products[W]
    info = {}
    part = gp.partition(g.indptr, g.indices, W, seed=0, info=info)
    _check_valid(g.indptr, part, W)
    cut = gp.edge_cut(g.indptr, g.indices, part)
    assert cut == info["edge_cut"]
    n = g.num_nodes
    contiguous = gp.edge_cut(g.indptr, g.indices, (np.arange(n) * W // n).astype(np.int32))
    m = (g.indices.size - n) // 2
    print(f"\nW={W}: cut {cut} ({cut / m:.4f}), planted {planted} ({planted / m:.4f}), "
          f"ratio {cut / planted:.3f}, contiguous {contiguous / m:.4f}, levels {info['levels']}, "
          f"times {json.dumps({k: round(v, 3) for k, v in info['times'].items()})}")
    assert cut < 0.5 * contiguous
    assert cut <= 1.15 * planted, f"cut / planted = {cut / planted:.3f}"


def test_isolated_vertices_and_components():
    # 3000 isolated vertices next to a 3000-vertex ring
    n = 6000
    ring = np.arange(3000)
    A = _sym_csr(n, ring, (ring + 1) % 3000)
    for k in (2, 5):
        _check_valid(A.indptr, gp.partition(A.indptr, A.indices, k, seed=2), k)
    # three components (cliques of 40, 30, 30), k = 8 > components
    off, us, vs = 0, [], []
    for m in (40, 30, 30):
        iu = np.triu_indices(m, 1)
        us.append(iu[0] + off)
        vs.append(iu[1] + off)
        off += m
    A = _sym_csr(off, np.concatenate(us), np.concatenate(vs))
    _check_valid(A.indptr, gp.partition(A.indptr, A.indices, 8, seed=0), 8)


def test_star_with_100k_leaves():
    n = 100_001
    A = _sym_csr(n, np.zeros(n - 1, np.int64), np.arange(1, n))
    for k in (2, 7):
        part = gp.partition(A.indptr, A.indices, k, seed=0)
        _check_valid(A.indptr, part, k)


@pytest.mark.parametrize("k", [1, 3, 64])
def test_k_edge_values(products, k):
    g, _ = products[4]
    part = gp.partition(g.indptr, g.indices, k, seed=0)
    _check_valid(g.indptr, part, k)
    if k == 1:
        assert not part.any()


# ----------------------------------------------------------------------------- end to end
def _write_ogbn_fixture(root, g):
    d = os.path.join(root, "ogbn_products")
    os.makedirs(os.path.join(d, "raw"))
    os.makedirs(os.path.join(d, "split", "sales_ranking"))
    rows = np.repeat(np.arange(g.num_nodes), np.diff(g.indptr))
    keep = rows < g.indices                                   # each undirected edge once; OGB adds the inverse
    def w(name, arr, fmt):
        with gzip.open(os.path.join(d, name), "wb") as f:
            np.savetxt(f, arr, fmt=fmt, delimiter=",")
    w("raw/edge.csv.gz", np.stack([rows[keep], g.indices[keep]], 1), "%d")
    w("raw/node-feat.csv.gz", g.feat, "%.9g")
    w("raw/node-label.csv.gz", g.label[:, None], "%d")
    for name, m in (("train", g.train_mask), ("valid", g.val_mask), ("test", g.test_mask)):
        w(f"split/sales_ranking/{name}.csv.gz", np.nonzero(m)[0][:, None], "%d")


def _worker(rank, world, port, tmp, mode, model_name, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank),
                       "WORLD_SIZE": str(world), "LOCAL_RANK": str(rank % max(torch.cuda.device_count(), 1)),
                       "ADAQP_SEED": "11"})
    os.environ.pop("ADAQP_SYNTHETIC", None)
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    from adaqp_b200.communicator import Communicator as comm
    from adaqp_b200.manager import GraphEngine as engine
    from test_gpu_trainer import _oracle_forward
    args = Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                     model_name=model_name, mode=mode, assign_scheme="uniform", logger_level="WARNING",
                     num_epoches=8, exp_path=f"{tmp}/exp")
    tr = Trainer(args)
    eng = engine.ctx
    from adaqp_b200.trainer.runtime_util import sync_seed, sync_model
    sync_seed()
    tr.model.reset_parameters()
    sync_model(tr.model)
    tr.model.eval()
    with torch.no_grad():
        logits = tr.model(eng.graph, eng.feats)
    eng.timer.clear(is_train=False)
    torch.cuda.synchronize()
    comm.ctx.comm_buffer.p2p.check_status()
    layouts = comm.gather_all(eng.layout)
    err = 0.0
    if rank == 0:
        state = {k: v.detach().cpu().numpy() for k, v in tr.model.state_dict().items()}
        want = _oracle_forward(layouts, state, model_name)[0]
        err = float(np.abs(logits.cpu().numpy().astype(np.float64) - want).max() / (np.abs(want).max() + 1e-12))
    rec = tr.train()
    acc = eng.recorder.epoches_metrics[:8, 0]
    out.put((rank, err, bool(torch.isfinite(rec).all()), float(acc[0]), float(acc.max())))


def test_graph_partition_then_train():
    import yaml
    from adaqp_b200.manager.partition_synth import global_graph, spec_from_config
    from adaqp_b200.manager.graphEngine import read_rank_layout
    from adaqp_b200.manager.layout import read_partition_book
    from test_gpu_trainer import _free_port
    with open(os.path.join(ROOT, "adaqp_b200", "config", "ogbn-products.yaml")) as f:
        cfg = yaml.safe_load(f)
    g, _ = global_graph(spec_from_config(cfg, 2, 20000 / 2449029))
    g = g.permuted(np.random.default_rng(3).permutation(g.num_nodes))
    with tempfile.TemporaryDirectory() as tmp:
        _write_ogbn_fixture(os.path.join(tmp, "data", "dataset"), g)
        env = {k: v for k, v in os.environ.items() if k != "ADAQP_SYNTHETIC"}
        r = subprocess.run([sys.executable, os.path.join(ROOT, "graph_partition.py"), "--dataset", "ogbn-products",
                            "--partition_size", "2"], cwd=tmp, env=env, capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stdout + r.stderr
        print(r.stdout)
        assert "edge cut" in r.stdout and "halo rows per rank" in r.stdout and "marginal share" in r.stdout
        d = os.path.join(tmp, "data", "part_data", "ogbn-products", "2part")
        part, header = read_partition_book(os.path.join(d, "partition_book.npz"))
        assert header["k"] == 2 and header["edge_cut"] == gp.edge_cut(g.indptr, g.indices, part)
        lays = [read_rank_layout(os.path.join(d, f"part{r}.npz")) for r in range(2)]
        assert [L.n_inner for L in lays] == np.bincount(part).tolist()
        for mode in ("AdaQP", "Vanilla"):
            ctx = mp.get_context("spawn")
            out = ctx.Queue()
            port = _free_port()
            procs = [ctx.Process(target=_worker, args=(rk, 2, port, tmp, mode, "gcn", out)) for rk in range(2)]
            for p in procs:
                p.start()
            for p in procs:
                p.join(timeout=900)
            assert all(p.exitcode == 0 for p in procs), (mode, [p.exitcode for p in procs])
            res = sorted(out.get(timeout=5) for _ in procs)
            assert res[0][1] < 2e-4, f"{mode}: eval logits vs float64 oracle: rel err {res[0][1]}"
            assert all(x[2] for x in res)
            assert res[0][4] > res[0][3] or res[0][4] > 0.5

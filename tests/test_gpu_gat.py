"""GAT on the GPU: the three kernels of csrc/gat.cu against the float64 oracle (oracle/gat_oracle.py), one two-rank
training step against the monolithic float64 model, bitwise determinism, the CLI and partition-then-train.

Stated bounds:
  * kernels: |got - oracle| <= 2e-5 * (per-row L1 mass + 1e-30) for out, dz, del, der (the mass of out[v] is
    sum_u alpha |z[u]|, of dz / del / der the sum of the absolute terms before cancellation, each alpha weighted by
    1 + |its exponent|; gat_oracle.masses), with 5e-4 for the hub row (degree > 100 000: fp32 sequential
    accumulation); |lse - oracle| <= 1e-5 * (1 + |lse|);
  * fp32 training step (Vanilla, AdaQP-p) vs float64: logits max error <= 2e-4 of max |logit|, loss <= 1e-4
    relative, every parameter gradient <= 1e-3 of its max magnitude;
  * 8-bit training step (AdaQP, AdaQP-q): attention scalars received bit-identical to what their owner computed;
    logits within 5e-2 of max |logit| of the float64 step.
"""
import hashlib
import os
import socket
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gat_oracle as G  # noqa: E402


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


# ----------------------------------------------------------------------------- kernels
def _graph(n, deg, seed, hub=False):
    import scipy.sparse as sp
    rng = np.random.RandomState(seed)
    m = n * deg // 2
    a, b = rng.randint(0, n, m), rng.randint(0, n, m)
    if hub:                                    # node 0 is adjacent to every other node
        a, b = np.r_[a, np.zeros(n - 1, np.int64)], np.r_[b, np.arange(1, n)]
    A = sp.coo_matrix((np.ones(a.size * 2), (np.r_[a, b], np.r_[b, a])), shape=(n, n)).tocsr()
    A.setdiag(0)
    A.eliminate_zeros()
    A = (A + sp.eye(n)).tocsr()
    A.sort_indices()
    return A.indptr.astype(np.int64), A.indices.astype(np.int64)


def _check_kernels(n, n_in, deg, F, H, seed, hub=False, hub_tol=5e-4):
    from adaqp_b200 import gat
    from adaqp_b200.manager.graph import LocalGraph
    dev = torch.device("cuda:0")
    indptr, indices = _graph(n, deg, seed, hub)
    rng = np.random.RandomState(seed)
    z = rng.randn(n, F).astype(np.float32)
    a_l, a_r = (rng.randn(H, F // H) * 0.3).astype(np.float32), (rng.randn(H, F // H) * 0.3).astype(np.float32)
    g = rng.randn(n, F).astype(np.float32)
    z64, g64 = z.astype(np.float64), g.astype(np.float64)
    # el / er from the kernel (compared with float64), then fed to both sides so that both see identical logits
    zt = torch.from_numpy(z).to(dev)
    el_t, er_t = gat.scores(zt, torch.from_numpy(a_l).to(dev), torch.from_numpy(a_r).to(dev), H)
    el, er = el_t.cpu().numpy().astype(np.float64), er_t.cpu().numpy().astype(np.float64)
    el_ref, er_ref = G.scores(z64, a_l.astype(np.float64), a_r.astype(np.float64), H)
    scale = np.abs(z64).reshape(n, H, -1).sum(-1) * np.abs(a_l).max() + 1e-30
    assert np.all(np.abs(el - el_ref) <= 1e-5 * scale) and np.all(np.abs(er - er_ref) <= 1e-5 * scale)
    out_all, lse_all = G.forward(indptr, indices, z64, el, er, H)      # every node is a destination somewhere
    s_all = (g64.reshape(n, H, -1) * out_all.reshape(n, H, -1)).sum(-1)
    # local graph of the first n_in rows; ids >= n_in are halo rows
    ip = indptr[:n_in + 1]
    ix = indices[:ip[-1]]
    L = LocalGraph(ip, ix.astype(np.int32), np.diff(indptr), np.diff(indptr), n_in, n - n_in, dev)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)  # noqa: E731
    el32, er32 = T(el), T(er)
    aux = T(np.concatenate([er, lse_all, s_all], 1))
    args_f = (L, T(z[:n_in]), T(z[n_in:]), el32[:n_in].contiguous(), el32[n_in:].contiguous(), er32[:n_in].contiguous(), H)
    out, lse = gat.forward(*args_f)
    # central / marginal style split: two row ranges of the one CSR equal the full launch bit for bit
    k = n_in // 3
    o1, l1 = gat.forward(*args_f, row_begin=0, row_end=k)
    o2, l2 = gat.forward(*args_f, row_begin=k, row_end=n_in)
    out_b, lse_b = gat.forward(*args_f)
    assert torch.equal(torch.cat([o1, o2]), out) and torch.equal(torch.cat([l1, l2]), lse)
    assert torch.equal(out_b, out) and torch.equal(lse_b, lse)
    args_b = (L, T(g[:n_in]), T(g[n_in:]), T(z[:n_in]), T(z[n_in:]), el32[:n_in].contiguous(), el32[n_in:].contiguous(),
              aux[:n_in].contiguous(), aux[n_in:].contiguous(), T(a_l), T(a_r), H)
    dz, dl, dr = gat.backward(*args_b)
    d1 = gat.backward(*args_b, row_begin=0, row_end=k)
    d2 = gat.backward(*args_b, row_begin=k, row_end=n_in)
    dz_b, dl_b, dr_b = gat.backward(*args_b)
    assert torch.equal(torch.cat([d1[0], d2[0]]), dz) and torch.equal(torch.cat([d1[1], d2[1]]), dl)
    assert torch.equal(torch.cat([d1[2], d2[2]]), dr)
    assert torch.equal(dz_b, dz) and torch.equal(dl_b, dl) and torch.equal(dr_b, dr)
    dz_ref, dl_ref, dr_ref = G.backward(ip, ix, g64, z64, el, er, lse_all, s_all, a_l.astype(np.float64),
                                        a_r.astype(np.float64), H)
    fm, bm, m1, m2 = G.masses(ip, ix, g64, z64, el, er, lse_all, s_all, a_l.astype(np.float64), a_r.astype(np.float64), H)
    tol = np.full((n_in, 1), 2e-5)
    if hub:
        tol[0] = hub_tol
    worst = {}
    for name, got, ref, mass in (("out", out, out_all[:n_in], fm), ("dz", dz, dz_ref, bm), ("del", dl, dl_ref, m1),
                                 ("der", dr, dr_ref, m2)):
        ratio = np.abs(got.cpu().numpy() - ref) / (mass + 1e-30)
        worst[name] = float(ratio.max())
        assert np.all(ratio <= tol), (name, F, H, float(ratio.max()), np.unravel_index(ratio.argmax(), ratio.shape))
    lerr = np.abs(lse.cpu().numpy() - lse_all[:n_in]) / (1 + np.abs(lse_all[:n_in]))
    worst["lse"] = float(lerr.max())
    assert lerr.max() <= 1e-5, lerr.max()
    print(f"GAT kernels F={F} H={H} hub={hub}: worst error / mass {worst}")


@pytest.mark.parametrize("F,H", [(256, 4), (256, 1), (256, 16), (128, 2), (128, 128), (47, 1), (47, 47), (41, 1),
                                 (41, 41), (107, 1)])
def test_kernels_match_oracle(F, H):
    _check_kernels(3000, 2000, 8, F, H, seed=F + H)


def test_kernels_hub_above_100k():
    """A node adjacent to all of 101 000 others (halo neighbours included) is exact at its full degree."""
    _check_kernels(101_001, 60_000, 2, 47, 1, seed=5, hub=True)


# ----------------------------------------------------------------------------- two-rank training step
def _mono_step(layouts, state, heads, n_layers):
    """float64 torch model on the unpartitioned graph (dropout off): logits, loss and parameter gradients."""
    import torch.nn.functional as F
    indptr, indices, base = G.global_from_layouts(layouts)
    N = int(base[-1])
    dst = torch.from_numpy(np.repeat(np.arange(N), np.diff(indptr)))
    src = torch.from_numpy(indices)
    x = torch.from_numpy(np.concatenate([L.feat for L in layouts]).astype(np.float64))
    y = torch.from_numpy(np.concatenate([L.label for L in layouts]).astype(np.int64))
    train = torch.from_numpy(np.concatenate([L.train_mask for L in layouts]).astype(bool))
    P = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in state.items()}
    h = x
    for i in range(n_layers):
        h = G.torch_gat_layer(src, dst, h, P[f"convs.{i}.weight"], P[f"convs.{i}.attn_l"], P[f"convs.{i}.attn_r"],
                              P[f"convs.{i}.bias"], heads[i])
        if i < n_layers - 1:
            h = F.relu(F.layer_norm(h, (h.shape[1],), P[f"norms.{i}.weight"], P[f"norms.{i}.bias"], 1e-5))
    loss = F.cross_entropy(h[train], y[train], reduction="sum") / int(train.sum())
    loss.backward()
    return h.detach().numpy(), float(loss), {k: v.grad.numpy() for k, v in P.items()}, base


def _step_worker(rank, world, port, tmp, mode, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": str(rank % torch.cuda.device_count()), "ADAQP_SYNTH_SCALE": "0.002",
                       "ADAQP_SEED": "11", "ADAQP_SYNTHETIC": "1"})
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    from adaqp_b200.communicator import Communicator as comm
    from adaqp_b200.manager import GraphEngine as engine
    from adaqp_b200.model import ops
    from adaqp_b200.trainer import runtime_util as ru
    tr = Trainer(Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                           model_name="gat", mode=mode, assign_scheme="uniform", logger_level="WARNING", num_epoches=1,
                           exp_path=f"{tmp}/exp"))
    eng, ex = engine.ctx, comm.ctx.comm_buffer.p2p
    ru.sync_seed()
    tr.model.reset_parameters()
    ru.sync_model(tr.model)
    tr.model.drop_rate = 0.0
    sent = {}
    real = ops._gat_exchange

    def spy(rows, name, is_train, scalars, aux_key, stream=None):
        sent[aux_key] = scalars.clone()
        return real(rows, name, is_train, scalars, aux_key, stream)

    ops._gat_exchange = spy
    tr.model.train()
    logits = tr.model(eng.graph, eng.feats)
    n_train = torch.LongTensor([eng.train_mask.numel()])
    comm.all_reduce_sum(n_train)
    loss = torch.nn.functional.cross_entropy(logits[eng.train_mask], eng.labels[eng.train_mask], reduction="sum") / int(n_train)
    tr.model.zero_grad()
    loss.backward()
    ru.average_gradients(tr.model)
    torch.cuda.synchronize()
    ex.check_status()
    ops._gat_exchange = real
    recv = {k: ex.halo(k).cpu().numpy().copy() for k in sent}
    sent_rows = {k: v.cpu().numpy() for k, v in sent.items()}
    eng.timer.clear()
    # the layer-0 evaluation cache never applies to GAT: every evaluation pass exchanges test0
    tr.model.eval()
    s0 = ex.seq["test0"]
    with torch.no_grad():
        e1 = tr.model(eng.graph, eng.feats)
        eng.timer.clear(is_train=False)
        e2 = tr.model(eng.graph, eng.feats)
        eng.timer.clear(is_train=False)
    torch.cuda.synchronize()
    ex.check_status()
    eval_ok = ex.seq["test0"] == s0 + 2 and torch.equal(e1, e2) and not hasattr(eng, "_eval_layer0_cache")
    layouts = comm.gather_all(eng.layout)
    mine = {"logits": logits.detach().cpu().numpy(), "loss": float(loss.detach()), "sent": sent_rows, "recv": recv}
    allr = comm.gather_all(mine)
    res = {"eval_ok": eval_ok}
    if rank == 0:
        state = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in tr.model.state_dict().items()}
        heads = [c._num_heads for c in tr.model.convs]
        want, want_loss, want_grads, base = _mono_step(layouts, state, heads, len(heads))
        got = np.concatenate([a["logits"] for a in allr]).astype(np.float64)
        res["logit_err"] = float(np.abs(got - want).max() / np.abs(want).max())
        res["loss_err"] = abs(sum(a["loss"] for a in allr) - want_loss) / abs(want_loss)
        grads = {k: p.grad.detach().cpu().numpy().astype(np.float64) for k, p in tr.model.named_parameters()}
        res["grad_err"] = {k: float(np.abs(grads[k] - want_grads[k]).max() / (np.abs(want_grads[k]).max() + 1e-30))
                           for k in grads}
        # attention scalars: what each rank received at halo position j == its owner's row, bit for bit
        mism = compared = 0
        for r, L in enumerate(layouts):
            for key, h in allr[r]["recv"].items():
                for p, pos in L.recv_idx.items():
                    lo, hi = layouts[p].send_idx[r]
                    want_rows = allr[p]["sent"][key][layouts[p].total_send_idx[lo:hi]]
                    mism += int((h[pos].view(np.uint32) != want_rows.view(np.uint32)).sum())
                    compared += want_rows.size
        res["aux_mismatches"], res["aux_compared"], res["aux_keys"] = mism, compared, sorted(allr[0]["recv"])
    comm.ctx.delete_buffer()
    out.put((rank, res))


def _spawn(target, world, *args, timeout=900):
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    with tempfile.TemporaryDirectory() as tmp:
        procs = [ctx.Process(target=target, args=(r, world, port, tmp) + args + (out,)) for r in range(world)]
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=timeout)
        assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
        return dict(out.get(timeout=5) for _ in procs)


@pytest.mark.parametrize("mode", ["Vanilla", "AdaQP-p", "AdaQP", "AdaQP-q"])
def test_two_rank_training_step(mode):
    res = _spawn(_step_worker, 2, mode)
    r = res[0]
    print("GAT step", mode, r)
    assert res[0]["eval_ok"] and res[1]["eval_ok"]
    assert r["aux_keys"] == ["attn_bwd0", "attn_bwd1", "attn_bwd2", "attn_fwd0", "attn_fwd1", "attn_fwd2"]
    assert r["aux_compared"] > 0 and r["aux_mismatches"] == 0
    if mode in ("Vanilla", "AdaQP-p"):
        assert r["logit_err"] <= 2e-4 and r["loss_err"] <= 1e-4, r
        assert all(v <= 1e-3 for v in r["grad_err"].values()), r["grad_err"]
    else:
        assert r["logit_err"] <= 5e-2, r


# ----------------------------------------------------------------------------- determinism
def _train_worker(rank, world, port, tmp, mode, scheme, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": str(rank % torch.cuda.device_count()), "ADAQP_SYNTH_SCALE": "0.004",
                       "ADAQP_SEED": "23", "ADAQP_SYNTHETIC": "1"})
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    # the Trainer draws the first random bit assignment while it is built, before train() seeds the run
    torch.manual_seed(23)
    tr = Trainer(Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                           model_name="gat", mode=mode, assign_scheme=scheme, logger_level="WARNING", num_epoches=3,
                           exp_path=f"{tmp}/exp", assign_cycle=2))
    rec = tr.train()
    h = hashlib.sha256()
    for k, v in tr.model.state_dict().items():
        h.update(k.encode())
        h.update(v.detach().cpu().numpy().tobytes())
    out.put((rank, (h.hexdigest(), bool(torch.isfinite(rec).all()))))


def test_determinism_adaqp_random():
    a = _spawn(_train_worker, 2, "AdaQP", "random")
    b = _spawn(_train_worker, 2, "AdaQP", "random")
    assert all(a[r][1] for r in a)
    assert a == b, (a, b)


# ----------------------------------------------------------------------------- CLI and partition files
def test_main_cli_gat_adaptive(tmp_path):
    port = _free_port()
    procs = []
    for r in range(2):
        env = dict(os.environ)
        env.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(r), "WORLD_SIZE": "2",
                    "LOCAL_RANK": str(r % torch.cuda.device_count()), "ADAQP_SYNTHETIC": "1",
                    "ADAQP_SYNTH_SCALE": "0.004", "ADAQP_NUM_EPOCHES": "3", "ADAQP_SEED": "5", "PYTHONPATH": ROOT})
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "main.py"), "--dataset", "ogbn-products",
                                       "--num_parts", "2", "--model_name", "gat", "--mode", "AdaQP", "--assign_scheme",
                                       "adaptive", "--logger_level", "WARNING"], cwd=str(tmp_path), env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=900)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), [o[-3000:] for o in outs]
    csv = tmp_path / "exp" / "ogbn-products" / "2part" / "gat" / "time" / "AdaQP_adaptive.csv"
    assert csv.exists()
    assert len(csv.read_text().strip().splitlines()) == 3


def _files_worker(rank, world, port, tmp, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": str(rank % torch.cuda.device_count()), "ADAQP_SEED": "11"})
    os.environ.pop("ADAQP_SYNTHETIC", None)
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    from adaqp_b200.manager import GraphEngine as engine
    tr = Trainer(Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                           model_name="gat", mode="AdaQP", assign_scheme="uniform", logger_level="WARNING",
                           num_epoches=4, exp_path=f"{tmp}/exp"))
    rec = tr.train()
    acc = engine.ctx.recorder.epoches_metrics[:4, 0]
    out.put((rank, (bool(torch.isfinite(rec).all()), float(acc.max()))))


def test_graph_partition_gat_then_train():
    import yaml
    from adaqp_b200.manager.partition_synth import global_graph, spec_from_config
    from test_gpu_partition import _write_ogbn_fixture
    with open(os.path.join(ROOT, "adaqp_b200", "config", "ogbn-products.yaml")) as f:
        cfg = yaml.safe_load(f)
    g, _ = global_graph(spec_from_config(cfg, 2, 20000 / 2449029))
    g = g.permuted(np.random.default_rng(3).permutation(g.num_nodes))
    with tempfile.TemporaryDirectory() as tmp:
        _write_ogbn_fixture(os.path.join(tmp, "data", "dataset"), g)
        env = {k: v for k, v in os.environ.items() if k != "ADAQP_SYNTHETIC"}
        r = subprocess.run([sys.executable, os.path.join(ROOT, "graph_partition.py"), "--dataset", "ogbn-products",
                            "--partition_size", "2", "--model_name", "gat"], cwd=tmp, env=env, capture_output=True,
                           text=True, timeout=900)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "files written for model gat" in r.stdout
        ctx = mp.get_context("spawn")
        out = ctx.Queue()
        port = _free_port()
        procs = [ctx.Process(target=_files_worker, args=(rk, 2, port, tmp, out)) for rk in range(2)]
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=900)
        assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
        res = dict(out.get(timeout=5) for _ in procs)
    assert all(v[0] for v in res.values())
    print("GAT from partition files: best train accuracy", res[0][1])

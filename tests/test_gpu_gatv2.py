"""GATv2 on the GPU: the three kernels of csrc/gatv2.cu against the float64 oracle (oracle/gatv2_oracle.py), the push
of halo gradients between in-process ranks, two-rank training steps against float64 models, bitwise determinism,
bit-exact resume, the CLI and partition-then-train.

Stated bounds:
  * kernels: |got - oracle| <= 2e-5 * (per-row L1 mass + 1e-30) for out, dzs (inner and halo), dzd and the per-row
    da shares (the mass of every term taken before cancellation, each alpha weighted by 1 + the magnitude of its
    exponent; gatv2_oracle.masses), 5e-4 for the hub row (degree > 100 000: fp32 sequential accumulation);
    |lse - oracle| <= 1e-5 * (1 + |lse|);
  * fp32 training step (Vanilla, AdaQP-p) vs the float64 model of the whole graph: GAT's bounds, logits <= 2e-4 of
    max |logit|, loss <= 1e-4 relative, every parameter gradient <= 1e-3 of its max magnitude;
  * every mode: the float64 protocol fed with the halo rows each rank received reproduces every layer's dzs, dzd
    and da within 1e-4 of their max magnitude (fp32 rounding only: this checks the push under quantisation).
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

from oracle import gatv2_oracle as G  # noqa: E402


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
    from adaqp_b200 import gatv2
    from adaqp_b200.manager.graph import LocalGraph
    dev = torch.device("cuda:0")
    indptr, indices = _graph(n, deg, seed, hub)
    rng = np.random.RandomState(seed)
    zs = rng.randn(n, F).astype(np.float32)
    zd = rng.randn(n_in, F).astype(np.float32)
    g = rng.randn(n_in, F).astype(np.float32)
    attn = (rng.randn(H, F // H) * 0.3).astype(np.float32)
    zs64, zd64, g64, a64 = (x.astype(np.float64) for x in (zs, zd, g, attn))
    ip = indptr[:n_in + 1]
    ix = indices[:ip[-1]]
    L = LocalGraph(ip, ix.astype(np.int32), np.diff(indptr), np.diff(indptr), n_in, n - n_in, dev)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)  # noqa: E731
    zs_t, zh_t, zd_t, g_t, a_t = T(zs[:n_in]), T(zs[n_in:]), T(zd), T(g), T(attn)
    # forward
    out_ref, lse_ref = G.forward(ip, ix, zs64, zd64, a64, H)
    args_f = (L, zs_t, zh_t, zd_t, a_t, H)
    out, lse = gatv2.forward(*args_f)
    k = n_in // 3
    o1, l1 = gatv2.forward(*args_f, row_begin=0, row_end=k)
    o2, l2 = gatv2.forward(*args_f, row_begin=k, row_end=n_in)
    out_b, lse_b = gatv2.forward(*args_f)
    assert torch.equal(torch.cat([o1, o2]), out) and torch.equal(torch.cat([l1, l2]), lse)
    assert torch.equal(out_b, out) and torch.equal(lse_b, lse)
    # backward: both sides read the same fp32 lse and S
    lse32 = lse_ref.astype(np.float32)
    S32 = (g64.reshape(n_in, H, -1) * out_ref.reshape(n_in, H, -1)).sum(-1).astype(np.float32)
    lse_t, S_t = T(lse32), T(S32)
    ref_s, ref_h, ref_d, ref_a = G.backward(ip, ix, zs64, zd64, g64, lse32.astype(np.float64),
                                            S32.astype(np.float64), a64, H)
    fm, sm, hm, dm, am = G.masses(ip, ix, zs64, zd64, g64, lse32.astype(np.float64), S32.astype(np.float64), a64, H)
    hp, hd = gatv2.halo_table(ip, ix, n_in, n - n_in)
    hp_t, hd_t = torch.from_numpy(hp).to(dev), torch.from_numpy(hd).to(dev)
    dh = gatv2.backward_halo(hp_t, hd_t, zh_t, zd_t, g_t, lse_t, S_t, a_t, H)
    m = (n - n_in) // 2
    dh1 = gatv2.backward_halo(hp_t, hd_t, zh_t, zd_t, g_t, lse_t, S_t, a_t, H, 0, m)
    dh2 = gatv2.backward_halo(hp_t, hd_t, zh_t, zd_t, g_t, lse_t, S_t, a_t, H, m, n - n_in)
    assert torch.equal(torch.cat([dh1, dh2]), dh)
    assert torch.equal(gatv2.backward_halo(hp_t, hd_t, zh_t, zd_t, g_t, lse_t, S_t, a_t, H), dh)
    # a push region and a fold table of two fictitious peers over a third of the inner rows
    sent = np.sort(rng.choice(n_in, size=max(n_in // 3, 1), replace=False))
    tsi = np.concatenate([sent, sent[::2]])
    send_idx = {1: (0, sent.size), 2: (sent.size, tsi.size)}
    fi, fp = gatv2.fold_table(n_in, [1, 2], send_idx, tsi)
    push = rng.randn(tsi.size, F).astype(np.float32)
    fold = (torch.from_numpy(fi).to(dev), torch.from_numpy(fp).to(dev))
    args_b = (L, zs_t, zh_t, zd_t, g_t, lse_t, S_t, a_t, H, T(push), fold)
    ds, dd, da = gatv2.backward_inner(*args_b)
    p1 = gatv2.backward_inner(*args_b, row_begin=0, row_end=k)
    p2 = gatv2.backward_inner(*args_b, row_begin=k, row_end=n_in)
    rep = gatv2.backward_inner(*args_b)
    for i, t in enumerate((ds, dd, da)):
        assert torch.equal(torch.cat([p1[i], p2[i]]), t) and torch.equal(rep[i], t)
    ref_sf = G.fold(ref_s, push.astype(np.float64), fi, fp)
    fold_mass = G.fold(sm, np.abs(push).astype(np.float64), fi, fp)
    tol = np.full((n_in, 1), 2e-5)
    if hub:
        tol[0] = hub_tol
    worst = {}
    for name, got, ref, mass, tl in (("out", out, out_ref, fm, tol), ("dzs", ds, ref_sf, fold_mass, tol),
                                     ("dzd", dd, ref_d, dm, tol), ("da", da, ref_a, am, tol),
                                     ("dzs_halo", dh, ref_h, hm, 2e-5)):
        ratio = np.abs(got.cpu().numpy() - ref) / (mass + 1e-30)
        worst[name] = float(ratio.max())
        assert np.all(ratio <= tl), (name, F, H, float(ratio.max()), np.unravel_index(ratio.argmax(), ratio.shape))
    lerr = np.abs(lse.cpu().numpy() - lse_ref) / (1 + np.abs(lse_ref))
    worst["lse"] = float(lerr.max())
    assert lerr.max() <= 1e-5, lerr.max()
    print(f"GATv2 kernels F={F} H={H} hub={hub}: worst error / mass {worst}")


@pytest.mark.parametrize("F,H", [(256, 4), (256, 1), (128, 2), (47, 1), (41, 1), (107, 1)])
def test_kernels_match_oracle(F, H):
    _check_kernels(3000, 2000, 8, F, H, seed=F + H)


def test_kernels_hub_above_100k():
    """A node adjacent to all of 101 000 others (halo neighbours included) is exact at its full degree, and the halo
    rows (each a neighbour of the hub) reduce over their inner destinations."""
    _check_kernels(101_001, 60_000, 2, 47, 1, seed=5, hub=True)


# ----------------------------------------------------------------------------- in-process push
def test_push_in_process_w3():
    """Three ranks on one device, several rounds: each owner's push region holds, bit for bit, the rows its holders
    pushed, and the fold kernel adds them as a brute-force sum does."""
    from adaqp_b200 import gatv2
    from adaqp_b200.communicator.p2p import PeerExchange, gatv2_key_dims, push_key, wire_in_process
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.graph import LocalGraph
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    W, F = 3, 48
    spec = SynthSpec(name="push", num_nodes=3000, num_edges=30000, num_parts=W, num_feats=F, num_classes=5,
                     cross_fraction=0.3, community_size=64, seed=4)
    lays = prepare_all_in_process(spec, DistGNNType.DistGATv2)
    dev = torch.device("cuda:0")
    dims = gatv2_key_dims([F, 16])
    exs = [PeerExchange(L.rank, W, dev, [F, 16], L.send_idx, {p: torch.from_numpy(v) for p, v in L.recv_idx.items()},
                        torch.from_numpy(L.total_send_idx), L.n_halo, timeout_ns=5_000_000_000, key_dims=dims)
           for L in lays]
    wire_in_process(exs)
    try:
        rng = np.random.RandomState(0)
        for rnd in range(4):
            key = push_key(rnd % 2)
            Fk = dims[key]
            rows = [torch.from_numpy(rng.randn(L.n_halo, Fk).astype(np.float32)).to(dev) for L in lays]
            for ex, r in zip(exs, rows):
                ex.post_send_fp(key, r)
            regions = [ex.complete_recv_fp(key).clone() for ex in exs]
            torch.cuda.synchronize()
            for ex in exs:
                ex.check_status()
            want = G.push([r.cpu().numpy() for r in rows], lays)
            for r, L in enumerate(lays):
                got = regions[r].cpu().numpy()
                assert got.shape == (len(L.total_send_idx), Fk)
                assert np.array_equal(got.view(np.uint32), want[r].astype(np.float32).view(np.uint32)), (rnd, r)
            # the fold of the inner backward adds every pushed row of an inner row, in send-peer order
            r = rnd % W
            L, ex = lays[r], exs[r]
            lg = LocalGraph(L.indptr, L.indices.astype(np.int32), np.diff(L.indptr), np.diff(L.indptr), L.n_inner,
                            L.n_halo, dev)
            fi, fp = gatv2.fold_table(L.n_inner, ex.send_peers, ex.send_idx, ex.total_send_idx)
            zeros = torch.zeros((L.n_inner, Fk), device=dev)
            lse = torch.zeros((L.n_inner, 1), device=dev)
            ds, _, _ = gatv2.backward_inner(lg, zeros, torch.zeros((L.n_halo, Fk), device=dev), zeros, zeros, lse,
                                            lse, torch.zeros(Fk, device=dev), 1, regions[r],
                                            (torch.from_numpy(fi).to(dev), torch.from_numpy(fp).to(dev)))
            brute = np.zeros((L.n_inner, Fk))
            for p in ex.send_peers:
                lo, hi = ex.send_idx[p]
                for i in range(lo, hi):
                    brute[L.total_send_idx[i]] += want[r][i]
            assert np.abs(ds.cpu().numpy() - brute).max() <= 1e-5 * max(np.abs(brute).max(), 1.0)
            for ex in exs:
                ex.release_fp(key)
        torch.cuda.synchronize()
    finally:
        for ex in exs:
            ex.close()


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
        c = f"convs.{i}."
        h = G.torch_gatv2_layer(src, dst, h, P[c + "W_s"], P[c + "b_s"], P[c + "W_d"], P[c + "b_d"], P[c + "attn"],
                                heads[i])
        if i < n_layers - 1:
            h = F.relu(F.layer_norm(h, (h.shape[1],), P[f"norms.{i}.weight"], P[f"norms.{i}.bias"], 1e-5))
    loss = F.cross_entropy(h[train], y[train], reduction="sum") / int(train.sum())
    loss.backward()
    return h.detach().numpy(), float(loss), {k: v.grad.numpy() for k, v in P.items()}


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
                           model_name="gatv2", mode=mode, assign_scheme="uniform", logger_level="WARNING",
                           num_epoches=1, exp_path=f"{tmp}/exp"))
    eng, ex = engine.ctx, comm.ctx.comm_buffer.p2p
    ru.sync_seed()
    tr.model.reset_parameters()
    ru.sync_model(tr.model)
    tr.model.drop_rate = 0.0
    # record every layer's inputs, received halo rows, upstream gradient and results
    seen = {}
    real_fwd, real_bwd = ops.DistAggGATv2.forward, ops.DistAggGATv2.backward

    def fwd(ctx, zs, zd, attn, graph, layer, is_train, heads):
        out_ = real_fwd(ctx, zs, zd, attn, graph, layer, is_train, heads)
        if is_train:
            seen[layer] = {"zs": zs.detach().cpu().numpy().copy(), "zd": zd.detach().cpu().numpy().copy(),
                           "attn": attn.detach().cpu().numpy().copy(), "heads": heads}
        return out_

    def bwd(ctx, grad):
        res_ = real_bwd(ctx, grad)
        seen[ctx.layer].update({"zs_halo": ctx.saved_tensors[1].cpu().numpy().copy(),
                                "g": grad.detach().cpu().numpy().copy(), "dzs": res_[0].cpu().numpy(),
                                "dzd": res_[1].cpu().numpy(), "da": res_[2].cpu().numpy()})
        return res_

    ops.DistAggGATv2.forward, ops.DistAggGATv2.backward = staticmethod(fwd), staticmethod(bwd)
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
    ops.DistAggGATv2.forward, ops.DistAggGATv2.backward = staticmethod(real_fwd), staticmethod(real_bwd)
    eng.timer.clear()
    # the layer-0 evaluation cache never applies: every evaluation pass exchanges test0
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
    allr = comm.gather_all({"logits": logits.detach().cpu().numpy(), "loss": float(loss.detach()), "seen": seen})
    res = {"eval_ok": eval_ok, "keys": sorted(ex.keys)}
    if rank == 0:
        state = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in tr.model.state_dict().items()}
        heads = [c._num_heads for c in tr.model.convs]
        want, want_loss, want_grads = _mono_step(layouts, state, heads, len(heads))
        got = np.concatenate([a["logits"] for a in allr]).astype(np.float64)
        res["logit_err"] = float(np.abs(got - want).max() / np.abs(want).max())
        res["loss_err"] = abs(sum(a["loss"] for a in allr) - want_loss) / abs(want_loss)
        grads = {k: p.grad.detach().cpu().numpy().astype(np.float64) for k, p in tr.model.named_parameters()}
        res["grad_err"] = {k: float(np.abs(grads[k] - want_grads[k]).max() / (np.abs(want_grads[k]).max() + 1e-30))
                           for k in grads}
        # the float64 protocol on the rows each rank actually used (its own zs / zd, the halo rows it received)
        proto = {}
        for layer in sorted(allr[0]["seen"]):
            per = [a["seen"][layer] for a in allr]
            H = per[0]["heads"]
            attn = per[0]["attn"].astype(np.float64)
            f64 = lambda a: np.asarray(a, np.float64)  # noqa: E731
            halo_grads, inner = [], []
            for r, L in enumerate(layouts):
                d = per[r]
                zs_all = np.concatenate([f64(d["zs"]), f64(d["zs_halo"])])
                o, lse = G.forward(L.indptr, L.indices, zs_all, f64(d["zd"]), attn, H)
                n = o.shape[0]
                S = (f64(d["g"]).reshape(n, H, -1) * o.reshape(n, H, -1)).sum(-1)
                ds, dh, dd, da = G.backward(L.indptr, L.indices, zs_all, f64(d["zd"]), f64(d["g"]), lse, S, attn, H)
                halo_grads.append(dh)
                inner.append((ds, dd, da))
            regions = G.push(halo_grads, layouts)
            errs = {"dzs": 0.0, "dzd": 0.0, "da": 0.0}
            for r, L in enumerate(layouts):
                fi, fp = G.fold_table(L)
                ds = G.fold(inner[r][0], regions[r], fi, fp)
                for name, ref in (("dzs", ds), ("dzd", inner[r][1]), ("da", inner[r][2].sum(0).reshape(H, -1))):
                    err = np.abs(per[r][name] - ref).max() / (np.abs(ref).max() + 1e-30)
                    errs[name] = max(errs[name], float(err))
            proto[layer] = errs
        res["proto_err"] = proto
        res["pushed_rows"] = int(sum(len(L.total_send_idx) for L in layouts))
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
    print("GATv2 step", mode, r)
    assert res[0]["eval_ok"] and res[1]["eval_ok"]
    assert r["keys"] == ["forward0", "forward1", "forward2", "push0", "push1", "push2", "test0", "test1", "test2"]
    assert r["pushed_rows"] > 0 and sorted(r["proto_err"]) == [0, 1, 2]
    for layer, errs in r["proto_err"].items():
        assert all(v <= 1e-4 for v in errs.values()), (layer, errs)
    if mode in ("Vanilla", "AdaQP-p"):
        assert r["logit_err"] <= 2e-4 and r["loss_err"] <= 1e-4, r
        assert all(v <= 1e-3 for v in r["grad_err"].values()), r["grad_err"]
    else:
        assert r["logit_err"] <= 5e-2, r


# ----------------------------------------------------------------------------- determinism, resume
def _train_worker(rank, world, port, tmp, mode, scheme, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": str(rank % torch.cuda.device_count()), "ADAQP_SYNTH_SCALE": "0.004",
                       "ADAQP_SEED": "23", "ADAQP_SYNTHETIC": "1"})
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    torch.manual_seed(23)
    tr = Trainer(Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                           model_name="gatv2", mode=mode, assign_scheme=scheme, logger_level="WARNING", num_epoches=3,
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


def test_resume_is_bit_exact():
    from test_gpu_checkpoint import _resume_worker, _spawn as spawn_ckpt
    with tempfile.TemporaryDirectory() as tmp:
        a = spawn_ckpt(_resume_worker, 2, tmp, "gatv2", "AdaQP", "random", None, "straight")
        spawn_ckpt(_resume_worker, 2, tmp, "gatv2", "AdaQP", "random", None, "first")
        b = spawn_ckpt(_resume_worker, 2, tmp, "gatv2", "AdaQP", "random", None, "resume")
    for r in (0, 1):
        ra, rb = a[r], b[r]
        assert ra["finite"] and rb["finite"]
        for key in ra["model"]:
            assert np.array_equal(ra["model"][key].view(np.uint32), rb["model"][key].view(np.uint32)), (r, key)
        for key in ra["adam"]:
            assert np.array_equal(ra["adam"][key], rb["adam"][key]), (r, key)
        assert len(rb["losses"]) == 6 and ra["losses"][3:] == rb["losses"][3:], (ra["losses"], rb["losses"])


# ----------------------------------------------------------------------------- CLI and partition files
def test_main_cli_gatv2_adaptive(tmp_path):
    port = _free_port()
    procs = []
    for r in range(2):
        env = dict(os.environ)
        env.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(r), "WORLD_SIZE": "2",
                    "LOCAL_RANK": str(r % torch.cuda.device_count()), "ADAQP_SYNTHETIC": "1",
                    "ADAQP_SYNTH_SCALE": "0.004", "ADAQP_NUM_EPOCHES": "3", "ADAQP_SEED": "5", "PYTHONPATH": ROOT})
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "main.py"), "--dataset", "ogbn-products",
                                       "--num_parts", "2", "--model_name", "gatv2", "--mode", "AdaQP", "--assign_scheme",
                                       "adaptive", "--logger_level", "WARNING"], cwd=str(tmp_path), env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=900)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), [o[-3000:] for o in outs]
    csv = tmp_path / "exp" / "ogbn-products" / "2part" / "gatv2" / "time" / "AdaQP_adaptive.csv"
    assert csv.exists()
    rows = csv.read_text().strip().splitlines()
    assert len(rows) == 3
    comm_col = [float(x.split(",")[4]) for x in rows[1:]]             # the push is timed as communication
    assert all(c > 0 for c in comm_col), rows


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
                           model_name="gatv2", mode="AdaQP", assign_scheme="uniform", logger_level="WARNING",
                           num_epoches=4, exp_path=f"{tmp}/exp"))
    rec = tr.train()
    acc = engine.ctx.recorder.epoches_metrics[:4, 0]
    out.put((rank, (bool(torch.isfinite(rec).all()), float(acc.max()))))


def test_graph_partition_gatv2_then_train():
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
                            "--partition_size", "2", "--model_name", "gatv2"], cwd=tmp, env=env, capture_output=True,
                           text=True, timeout=900)
        assert r.returncode == 0, r.stdout + r.stderr
        assert "files written for model gatv2" in r.stdout
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
    print("GATv2 from partition files: best train accuracy", res[0][1])

"""GraphSAGE max-pool on the GPU: the two kernels of csrc/sage_pool.cu against the float64 oracle
(oracle/sage_pool_oracle.py), the arg rows on the fp32 send path, one two-rank training step per mode, bitwise
determinism and the CLI.

Stated bounds:
  * kernels: m and arg bit-identical to the oracle (a max is an exact copy of one input); |dp - oracle| <=
    1e-5 * (sum of |routed terms|) per element, 5e-4 for the hub row (degree > 100 000: fp32 sequential sum);
  * training step, every mode: each layer's m / arg bit-identical to the oracle fed the rows this rank received,
    dp within the kernel bound, and the received pool_arg rows bit-identical to the sender's saved rows;
  * fp32 training step (Vanilla, AdaQP-p) vs a float64 monolithic model: logits within 2e-4 of max |logit|, loss
    within 1e-4 relative, every parameter gradient within 2e-3 of its max magnitude (an fp32 near-tie can pick a
    different arg than float64 and route one gradient term elsewhere).
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

from oracle import sage_pool_oracle as P  # noqa: E402


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


def _check_kernels(n, n_in, deg, F, seed, hub=False, ties=False, hub_tol=5e-4):
    from adaqp_b200 import sage_pool
    from adaqp_b200.manager.graph import LocalGraph
    dev = torch.device("cuda:0")
    indptr, indices = _graph(n, deg, seed, hub)
    rng = np.random.RandomState(seed)
    p = np.maximum(rng.randn(n, F), 0).astype(np.float32)
    if ties:                                   # a handful of levels: most maxima are attained several times
        p = (np.floor(p * 2) / 2).astype(np.float32)
    g = rng.randn(n, F).astype(np.float32)
    # every node is a destination somewhere: arg of all n rows, in the encoding of a rank whose inner rows are < n_in
    m_all, arg_all = P.forward(indptr, indices, p, n_in)
    ip = indptr[:n_in + 1]
    ix = indices[:ip[-1]]
    L = LocalGraph(ip, ix.astype(np.int32), np.diff(indptr), np.diff(indptr), n_in, n - n_in, dev)
    T = lambda a, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(a)).to(dev, dt)  # noqa: E731
    x0, x1 = T(p[:n_in]), T(p[n_in:])
    m, arg = sage_pool.forward(L, x0, x1)
    assert np.array_equal(m.cpu().numpy(), m_all[:n_in].astype(np.float32)), F
    assert np.array_equal(arg.cpu().numpy().astype(np.int64), arg_all[:n_in]), F
    # local / halo two-pass form == one pass, bit for bit; row-range split and repeated launches too
    m2, a2 = sage_pool.forward(L, x0, None, part="local")
    sage_pool.forward(L, x0, x1, out=m2, arg=a2, part="halo")
    assert torch.equal(m2, m) and torch.equal(a2, arg)
    k = n_in // 3
    r1 = sage_pool.forward(L, x0, x1, 0, k)
    r2 = sage_pool.forward(L, x0, x1, k, n_in)
    rb = sage_pool.forward(L, x0, x1)
    assert torch.equal(torch.cat([r1[0], r2[0]]), m) and torch.equal(torch.cat([r1[1], r2[1]]), arg)
    assert torch.equal(rb[0], m) and torch.equal(rb[1], arg)
    # backward: local rows u, want[e] = u - n_in (one numbering), arg rows of every destination
    want = (np.repeat(np.arange(n_in), np.diff(ip)) - n_in).astype(np.int32)
    wt = T(want, torch.int32)
    ga, gb = T(g[:n_in]), T(g[n_in:])
    aa, ab = T(arg_all[:n_in].astype(np.int32), torch.int32), T(arg_all[n_in:].astype(np.int32), torch.int32)
    dp = sage_pool.backward(L, wt, ga, gb, aa, ab)
    d2 = sage_pool.backward(L, wt, ga, None, aa, None, part="local")
    sage_pool.backward(L, wt, ga, gb, aa, ab, dp=d2, part="halo")
    assert torch.equal(d2, dp)
    s1 = sage_pool.backward(L, wt, ga, gb, aa, ab, 0, k)
    s2 = sage_pool.backward(L, wt, ga, gb, aa, ab, k, n_in)
    assert torch.equal(torch.cat([s1, s2]), dp) and torch.equal(sage_pool.backward(L, wt, ga, gb, aa, ab), dp)
    g64 = g.astype(np.float64)
    ref = P.backward(ip, ix, want, g64, arg_all)
    mass = P.backward(ip, ix, want, np.abs(g64), arg_all)
    tol = np.full((n_in, 1), 1e-5)
    if hub:
        tol[0] = hub_tol
    ratio = np.abs(dp.cpu().numpy() - ref) / (mass + 1e-30)
    assert np.all(ratio <= tol), (F, float(ratio.max()), np.unravel_index(ratio.argmax(), ratio.shape))
    hits = int((mass > 0).sum())
    assert hits > 0
    print(f"SAGE-pool kernels F={F} hub={hub} ties={ties}: worst dp error / mass {float(ratio.max()):.3g}, "
          f"routed columns {hits}")


@pytest.mark.parametrize("F", [602, 256, 100, 47, 41])
def test_kernels_match_oracle(F):
    _check_kernels(3000, 2000, 8, F, seed=F)


@pytest.mark.parametrize("F", [256, 41])
def test_kernels_exact_ties(F):
    """Values on a coarse grid, so most maxima are attained several times: arg is the first maximum in CSR order."""
    _check_kernels(3000, 2000, 8, F, seed=F + 1, ties=True)


@pytest.mark.parametrize("F,ties", [(47, False), (602, True)])
def test_kernels_hub_above_100k(F, ties):
    """A node adjacent to all of 101 000 others (halo neighbours included) is exact at its full degree."""
    _check_kernels(101_001, 60_000, 2, F, seed=5, hub=True, ties=ties)


# ----------------------------------------------------------------------------- transport
def test_arg_bit_patterns_survive_fp32_send():
    """int32 arg rows travel through the fp32 path; patterns that are NaN as floats arrive unchanged."""
    from adaqp_b200.communicator.p2p import PeerExchange, sage_pool_key_dims, wire_in_process
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    dev = torch.device("cuda:0")
    W, F = 2, 41
    spec = SynthSpec(name="pool", num_nodes=2000, num_edges=2000 * 10, num_parts=W, num_feats=F, num_classes=5,
                     cross_fraction=0.2, community_size=64, seed=4)
    lays = prepare_all_in_process(spec)
    dims = sage_pool_key_dims([F, 16])
    exs = [PeerExchange(L.rank, W, dev, [F, 16], L.send_idx, {p: torch.from_numpy(v) for p, v in L.recv_idx.items()},
                        torch.from_numpy(L.total_send_idx), L.n_halo, timeout_ns=5_000_000_000, key_dims=dims)
           for L in lays]
    wire_in_process(exs)
    rng = np.random.RandomState(0)
    special = np.array([0x7FC00001, 0x7F800001, -1, -2 ** 31, 0x7FFFFFFF, -4194305], np.int64).astype(np.int32)
    args = []
    for L in lays:
        a = rng.randint(-2 ** 31, 2 ** 31 - 1, size=(L.n_inner, F), dtype=np.int64).astype(np.int32)
        a.reshape(-1)[::7] = special[np.arange(a.size // 7 + 1) % special.size][:a.reshape(-1)[::7].size]
        args.append(a)
    for e, a in zip(exs, args):
        e.post_send_fp("pool_arg0", torch.from_numpy(a).to(dev).view(torch.float32))
    got = [e.complete_recv_fp("pool_arg0").view(torch.int32).cpu().numpy().copy() for e in exs]
    for e in exs:
        e.release_fp("pool_arg0")
    torch.cuda.synchronize()
    for e in exs:
        e.check_status()
    for r, L in enumerate(lays):
        for p, pos in L.recv_idx.items():
            lo, hi = lays[p].send_idx[r]
            assert np.array_equal(got[r][pos], args[p][lays[p].total_send_idx[lo:hi]])
    for e in exs:
        e.close()


# ----------------------------------------------------------------------------- two-rank training step
def _mono_step(layouts, state, n_layers):
    """float64 torch model on the unpartitioned graph (dropout off): logits, loss and parameter gradients."""
    import torch.nn.functional as F
    indptr, indices, base = P.global_from_layouts(layouts)
    N = int(base[-1])
    dst = torch.from_numpy(np.repeat(np.arange(N), np.diff(indptr)))
    src = torch.from_numpy(indices)
    x = torch.from_numpy(np.concatenate([L.feat for L in layouts]).astype(np.float64))
    y = torch.from_numpy(np.concatenate([L.label for L in layouts]).astype(np.int64))
    train = torch.from_numpy(np.concatenate([L.train_mask for L in layouts]).astype(bool))
    Pm = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in state.items()}
    h = x
    for i in range(n_layers):
        s = f"sages.{i}."
        h = P.torch_pool_layer(src, dst, h, Pm[s + "fc_pool.weight"], Pm[s + "fc_pool.bias"], Pm[s + "fc_self.weight"],
                               Pm[s + "fc_neigh.weight"], Pm[s + "bias"])
        if i < n_layers - 1:
            h = F.relu(F.layer_norm(h, (h.shape[1],), Pm[f"norms.{i}.weight"], Pm[f"norms.{i}.bias"], 1e-5))
    loss = F.cross_entropy(h[train], y[train], reduction="sum") / int(train.sum())
    loss.backward()
    return h.detach().numpy(), float(loss), {k: v.grad.numpy() for k, v in Pm.items()}


def _layer_checks(rec, recv, g, want, n_inner):
    """Per layer: m / arg bit-identical to the oracle fed the received p rows, dp within the kernel bound of the
    oracle fed the received gm and arg rows.  Returns (bit mismatches, worst dp error / mass)."""
    ip, ix = g
    bad, worst = 0, 0.0
    for l, d in sorted(rec.items()):
        p_all = np.concatenate([d["p"], recv[f"forward{l}"]]).astype(np.float64)
        m_ref, a_ref = P.forward(ip, ix, p_all, n_inner)
        bad += int((d["m"] != m_ref.astype(np.float32)).sum()) + int((d["arg"] != a_ref).sum())
        g_all = np.concatenate([d["gm"], recv[f"backward{l}"]]).astype(np.float64)
        a_all = np.concatenate([d["arg"], recv[f"pool_arg{l}"]]).astype(np.int64)
        ref = P.backward(ip, ix, want, g_all, a_all)
        mass = P.backward(ip, ix, want, np.abs(g_all), a_all)
        worst = max(worst, float((np.abs(d["dp"] - ref) / (mass + 1e-30)).max()))
    return bad, worst


def _step_worker(rank, world, port, tmp, mode, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": str(rank % torch.cuda.device_count()), "ADAQP_SYNTH_SCALE": "0.002",
                       "ADAQP_SEED": "11", "ADAQP_SYNTHETIC": "1"})
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    from adaqp_b200.communicator import Communicator as comm
    from adaqp_b200.manager import DecompGraph
    from adaqp_b200.manager import GraphEngine as engine
    from adaqp_b200.model import ops
    from adaqp_b200.trainer import runtime_util as ru
    tr = Trainer(Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                           model_name="sage", mode=mode, assign_scheme="uniform", logger_level="WARNING", num_epoches=1,
                           exp_path=f"{tmp}/exp", aggregator_type="pool"))
    eng, ex = engine.ctx, comm.ctx.comm_buffer.p2p
    ru.sync_seed()
    tr.model.reset_parameters()
    ru.sync_model(tr.model)
    tr.model.drop_rate = 0.0
    rec = {}
    real_f, real_b = ops.DistAggSAGEPool.forward, ops.DistAggSAGEPool.backward

    def spy_f(ctx, p, graph, layer, is_train):
        m = real_f(ctx, p, graph, layer, is_train)
        rec[layer] = {"p": p.detach().cpu().numpy().copy(), "m": m.detach().cpu().numpy().copy()}
        return m

    def spy_b(ctx, *grads):
        rec[ctx.layer]["arg"] = ctx.saved_tensors[0].cpu().numpy().copy()
        out = real_b(ctx, *grads)
        rec[ctx.layer].update(gm=grads[0].cpu().numpy().copy(), dp=out[0].cpu().numpy().copy())
        return out

    ops.DistAggSAGEPool.forward, ops.DistAggSAGEPool.backward = staticmethod(spy_f), staticmethod(spy_b)
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
    ops.DistAggSAGEPool.forward, ops.DistAggSAGEPool.backward = staticmethod(real_f), staticmethod(real_b)
    L = len(rec)
    recv = {}
    for l in range(L):
        for k in (f"forward{l}", f"backward{l}"):
            recv[k] = ex.halo(k).cpu().numpy().copy()
        recv[f"pool_arg{l}"] = ex.halo(f"pool_arg{l}").view(torch.int32).cpu().numpy().copy()
    g = eng.graph.full if isinstance(eng.graph, DecompGraph) else eng.graph
    bad, worst = _layer_checks(rec, recv, (g.indptr.cpu().numpy(), g.indices.cpu().numpy().astype(np.int64)),
                               eng.pool_want.cpu().numpy().astype(np.int64), g.n_inner)
    eng.timer.clear()
    # the layer-0 evaluation cache never applies to pool: every evaluation pass exchanges test0
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
    mine = {"logits": logits.detach().cpu().numpy(), "loss": float(loss.detach()),
            "args": {l: rec[l]["arg"] for l in rec}, "recv_args": {l: recv[f"pool_arg{l}"] for l in rec}}
    allr = comm.gather_all(mine)
    res = {"eval_ok": eval_ok, "layer_bit_mismatches": bad, "dp_worst": worst, "layers": L}
    if rank == 0:
        state = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in tr.model.state_dict().items()}
        want, want_loss, want_grads = _mono_step(layouts, state, L)
        got = np.concatenate([a["logits"] for a in allr]).astype(np.float64)
        res["logit_err"] = float(np.abs(got - want).max() / np.abs(want).max())
        res["loss_err"] = abs(sum(a["loss"] for a in allr) - want_loss) / abs(want_loss)
        grads = {k: p.grad.detach().cpu().numpy().astype(np.float64) for k, p in tr.model.named_parameters()}
        res["grad_err"] = {k: float(np.abs(grads[k] - want_grads[k]).max() / (np.abs(want_grads[k]).max() + 1e-30))
                           for k in grads}
        # pool_arg rows: what each rank received at halo position j == its owner's saved arg row, bit for bit
        mism = compared = 0
        for r, Lr in enumerate(layouts):
            for l, h in allr[r]["recv_args"].items():
                for p, pos in Lr.recv_idx.items():
                    lo, hi = layouts[p].send_idx[r]
                    rows = allr[p]["args"][l][layouts[p].total_send_idx[lo:hi]]
                    mism += int((h[pos] != rows).sum())
                    compared += rows.size
        res["arg_mismatches"], res["arg_compared"] = mism, compared
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
    print("SAGE-pool step", mode, r, res[1])
    for q in res.values():
        assert q["eval_ok"] and q["layers"] == 3
        assert q["layer_bit_mismatches"] == 0 and q["dp_worst"] <= 1e-5, q
    assert r["arg_compared"] > 0 and r["arg_mismatches"] == 0
    if mode in ("Vanilla", "AdaQP-p"):
        assert r["logit_err"] <= 2e-4 and r["loss_err"] <= 1e-4, r
        assert all(v <= 2e-3 for v in r["grad_err"].values()), r["grad_err"]


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
                           model_name="sage", mode=mode, assign_scheme=scheme, logger_level="WARNING", num_epoches=3,
                           exp_path=f"{tmp}/exp", assign_cycle=2, aggregator_type="pool"))
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


# ----------------------------------------------------------------------------- CLI
def test_main_cli_pool_adaptive(tmp_path):
    port = _free_port()
    procs = []
    for r in range(2):
        env = dict(os.environ)
        env.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(r), "WORLD_SIZE": "2",
                    "LOCAL_RANK": str(r % torch.cuda.device_count()), "ADAQP_SYNTHETIC": "1",
                    "ADAQP_SYNTH_SCALE": "0.004", "ADAQP_NUM_EPOCHES": "3", "ADAQP_SEED": "5", "PYTHONPATH": ROOT})
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "main.py"), "--dataset", "ogbn-products",
                                       "--num_parts", "2", "--model_name", "sage", "--aggregator_type", "pool",
                                       "--mode", "AdaQP", "--assign_scheme", "adaptive", "--logger_level", "WARNING"],
                                      cwd=str(tmp_path), env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                                      text=True))
    outs = [p.communicate(timeout=900)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), [o[-3000:] for o in outs]
    csv = tmp_path / "exp" / "ogbn-products" / "2part" / "sage" / "time" / "AdaQP_adaptive.csv"
    assert csv.exists()
    assert len(csv.read_text().strip().splitlines()) == 3

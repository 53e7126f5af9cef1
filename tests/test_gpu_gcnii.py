"""GCNII on the GPU: the column-sliced propagation kernel (csrc/spmm.cu appnp_prop_sliced_kernel) bitwise against the
unsliced appnp_prop_kernel and within the float64 oracle's bound, training steps against a float64 model of the
unpartitioned graph (oracle/gcnii_oracle.py), L >= 10 exchange keys, bitwise determinism, bit-exact resume and the CLI
from training through resume to predictions.

Stated bounds:
  * kernel: sliced output (and acc) torch.equal to the unsliced kernel's; |got - oracle| <= 4e-6 * (per-row L1 mass),
    the mass being every term of the step before cancellation (test_gpu_spmm_shapes.py's bound);
  * fp32 training step (Vanilla, AdaQP-p): logits <= 2e-5 of max |logit|, loss <= 1e-5 relative, every parameter
    gradient <= 1e-3 of its max magnitude (test_gpu_gnn_step.py's bounds), halo rows bit-identical to the owners' rows;
  * 8-bit training step (AdaQP, AdaQP-q): logits <= 1e-2 of max |logit|; every received row within one 8-bit
    quantisation step of its owner's row plus the bf16 rounding of the wire's scale and row minimum.
"""
import contextlib
import hashlib
import json
import os
import socket
import sys
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import gcnii_oracle as G  # noqa: E402

ALPHA = 0.1


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


@contextlib.contextmanager
def slice_cols(w):
    from adaqp_b200 import _lib
    old = _lib.get_option("spmm_slice_cols")
    _lib.set_option("spmm_slice_cols", w)
    try:
        yield
    finally:
        _lib.set_option("spmm_slice_cols", old)


# ----------------------------------------------------------------------------- kernel
def _hub_graph(n, deg, seed):
    """Random symmetric graph with one self-loop per node; node 0 is adjacent to every other node."""
    import scipy.sparse as sp
    rng = np.random.RandomState(seed)
    m = n * deg // 2
    a, b = rng.randint(0, n, m), rng.randint(0, n, m)
    a, b = np.r_[a, np.zeros(n - 1, np.int64)], np.r_[b, np.arange(1, n)]
    A = sp.coo_matrix((np.ones(a.size * 2), (np.r_[a, b], np.r_[b, a])), shape=(n, n)).tocsr()
    A.setdiag(0)
    A.eliminate_zeros()
    A = (A + sp.eye(n)).tocsr()
    A.sort_indices()
    return A.indptr.astype(np.int64), A.indices.astype(np.int64)


def _check_kernel(L, x, F, widths, seed, ranges):
    """Every form of the step on LocalGraph L with sources x ([n_inner + n_halo, F]): the automatic choice and each
    forced width in `widths` against the forced-unsliced kernel (torch.equal), the unsliced result against the float64
    oracle (<= 4e-6 of the L1 mass), over the row ranges `ranges`, the two-pass local + halo form and an output view."""
    from adaqp_b200.manager.graph import ACC_FOLD, ACC_ON, ACC_READ, appnp_prop
    dev = L.device
    n_in = L.n_inner
    rng = np.random.RandomState(seed)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)  # noqa: E731
    xl, xh = T(x[:n_in]), (T(x[n_in:]) if L.n_halo else None)
    z = rng.randn(n_in, F).astype(np.float32)
    acc0 = rng.randn(n_in, F).astype(np.float32)
    zt = T(z)
    ip, ix = L.indptr.cpu().numpy(), L.indices.cpu().numpy().astype(np.int64)
    worst = 0.0
    for fwd in (True, False):
        pre, post = (L.norm["out_-0.5"], L.norm["in_-0.5"]) if fwd else (L.norm["in_-0.5"], L.norm["out_-0.5"])
        A = G.matrix(ip, ix, x.shape[0], pre.cpu().numpy(), post.cpu().numpy())
        base = (1 - ALPHA) * (A @ x.astype(np.float64))
        m_base = (1 - ALPHA) * (abs(A) @ np.abs(x).astype(np.float64))
        own = ALPHA * x[:n_in].astype(np.float64)
        if fwd:
            cases = {"teleport": ({}, base + ALPHA * z, m_base + ALPHA * np.abs(z))}
        else:
            cases = {"on": ({"acc_mode": ACC_ON}, base, m_base),
                     "on_read": ({"acc_mode": ACC_ON | ACC_READ}, base, m_base),
                     "on_fold": ({"acc_mode": ACC_ON | ACC_FOLD}, base + own, m_base + np.abs(own)),
                     "on_read_fold": ({"acc_mode": ACC_ON | ACC_READ | ACC_FOLD}, base + acc0 + own,
                                      m_base + np.abs(acc0) + np.abs(own))}
        for name, (kw, ref, mass) in cases.items():
            def launch(lo, hi, out=None, part=None):
                kw2 = dict(kw)
                a = None
                if "acc_mode" in kw:
                    a = kw2["acc"] = T(acc0[lo:hi])
                else:
                    kw2["tele"] = zt[lo:hi]
                o = appnp_prop(L, xl, xh, pre, post, 1 - ALPHA, ALPHA, row_begin=lo, row_end=hi, out=out, part=part,
                               **kw2)
                return o, a

            def forms(lo, hi):
                res = {"one": launch(lo, hi)}
                if xh is not None:
                    o, a = launch(lo, hi, part="local")
                    appnp_prop(L, xl, xh, pre, post, 1 - ALPHA, ALPHA, row_begin=lo, row_end=hi, out=o, part="halo")
                    res["two_pass"] = (o, a)
                sentinel = -12345.5
                buf = torch.full((hi - lo + 6, F), sentinel, dtype=torch.float32, device=dev)
                o, a = launch(lo, hi, out=buf[3:3 + hi - lo])
                assert bool((buf[:3] == sentinel).all()) and bool((buf[3 + hi - lo:] == sentinel).all()), name
                res["view"] = (buf[3:3 + hi - lo].clone(), a)
                return res

            for lo, hi in ranges:
                if hi <= lo:
                    continue
                with slice_cols(F):
                    want = forms(lo, hi)
                out = want["one"][0].cpu().numpy().astype(np.float64)
                ratio = np.abs(out - ref[lo:hi]) / (mass[lo:hi] + 1e-30)
                worst = max(worst, float(ratio.max()))
                assert ratio.max() <= 4e-6, (name, F, float(ratio.max()))
                for w in widths:
                    ctx = slice_cols(w) if w else contextlib.nullcontext()
                    with ctx:
                        got = forms(lo, hi)
                    for form in want:
                        assert torch.equal(got[form][0], want[form][0]), (name, F, w, form, lo, hi)
                        if want[form][1] is not None:
                            assert torch.equal(got[form][1], want[form][1]), (name, F, w, form, "acc")
    return worst


def _layouts(W, F, seed):
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    spec = SynthSpec(name="gcnii", num_nodes=6000, num_edges=6000 * 12, num_parts=W, num_feats=F, num_classes=5,
                     cross_fraction=0.25, community_size=128, seed=seed)
    return prepare_all_in_process(spec, DistGNNType.DistGCNII)


@pytest.mark.parametrize("F,widths", [(256, [0, 128, 64]), (384, [0]), (512, [0])])
def test_sliced_kernel_bitwise_w3(F, widths):
    """Rank 1 of three: central rows, marginal rows, both, in one pass and as local + halo passes."""
    from adaqp_b200.manager.graph import LocalGraph
    lay = _layouts(3, 4, seed=F)[1]
    assert lay.n_halo > 0 and 0 < lay.n_central < lay.n_inner
    L = LocalGraph(lay.indptr, lay.indices, lay.in_degrees, lay.out_degrees, lay.n_inner, lay.n_halo, torch.device("cuda:0"))
    x = np.random.RandomState(F).randn(lay.n_inner + lay.n_halo, F).astype(np.float32)
    ranges = [(0, lay.n_central), (lay.n_central, lay.n_inner), (0, lay.n_inner), (lay.n_inner // 3, lay.n_inner // 2)]
    worst = _check_kernel(L, x, F, widths, F + 1, ranges)
    print(f"sliced propagation F={F}: bitwise equal to unsliced; worst error / mass {worst:.2e}")


def test_sliced_kernel_hub_above_100k():
    """A node adjacent to all of 101 000 others (halo neighbours included), F = 256."""
    from adaqp_b200.manager.graph import LocalGraph
    n, n_in, F = 101_001, 60_000, 256
    indptr, indices = _hub_graph(n, 2, seed=5)
    ip = indptr[:n_in + 1]
    ix = indices[:ip[-1]]
    deg = np.diff(indptr)
    assert deg[0] > 100_000
    L = LocalGraph(ip, ix.astype(np.int32), deg, deg, n_in, n - n_in, torch.device("cuda:0"))
    x = np.random.RandomState(5).randn(n, F).astype(np.float32)
    worst = _check_kernel(L, x, F, [0], 6, [(0, n_in), (0, 1)])
    print(f"sliced propagation hub: worst error / mass {worst:.2e}")


def test_slice_width_refused():
    from adaqp_b200.manager.graph import LocalGraph, appnp_prop
    lay = _layouts(2, 4, seed=1)[0]
    L = LocalGraph(lay.indptr, lay.indices, lay.in_degrees, lay.out_degrees, lay.n_inner, lay.n_halo, torch.device("cuda:0"))
    x = torch.randn(lay.n_inner, 256, device="cuda:0")
    for w in (6, 132):
        with slice_cols(w), pytest.raises(RuntimeError, match="slice width"):
            appnp_prop(L, x, None, None, None, 0.9, 0.1, tele=x)


# ----------------------------------------------------------------------------- training steps
def _mono_step(layouts, state, L, alpha, theta):
    """float64 torch model on the unpartitioned graph (dropout off): logits, loss and parameter gradients."""
    import torch.nn.functional as F
    indptr, indices, base = G.global_from_layouts(layouts)
    N = int(base[-1])
    dst = torch.from_numpy(np.repeat(np.arange(N), np.diff(indptr)))
    src = torch.from_numpy(indices)
    x = torch.from_numpy(np.concatenate([Lr.feat for Lr in layouts]).astype(np.float64))
    y = torch.from_numpy(np.concatenate([Lr.label for Lr in layouts]).astype(np.int64))
    train = torch.from_numpy(np.concatenate([Lr.train_mask for Lr in layouts]).astype(bool))
    Pm = {key: torch.tensor(v, dtype=torch.float64, requires_grad=True) for key, v in state.items()}
    h = G.torch_gcnii(src, dst, x, Pm, L, alpha, theta)
    loss = F.cross_entropy(h[train], y[train], reduction="sum") / int(train.sum())
    loss.backward()
    return h.detach().numpy(), float(loss.detach()), {key: v.grad.numpy() for key, v in Pm.items()}


def _step_worker(rank, world, port, tmp, mode, split, layers, out):
    try:
        _step(rank, world, port, tmp, mode, split, layers, out)
    except Exception:                           # noqa: BLE001 - reported to the parent instead of a timeout
        import traceback
        out.put((rank, {"error": traceback.format_exc()}))
        raise


def _step(rank, world, port, tmp, mode, split, layers, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": str(rank % torch.cuda.device_count()), "ADAQP_SYNTH_SCALE": "0.002",
                       "ADAQP_SEED": "11", "ADAQP_SYNTHETIC": "1", "ADAQP_MARGINAL_SPLIT": "1" if split else "0"})
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    from adaqp_b200 import _lib
    from adaqp_b200.communicator import Communicator as comm
    from adaqp_b200.manager import GraphEngine as engine
    from adaqp_b200.model import ops
    from adaqp_b200.trainer import runtime_util as ru
    tr = Trainer(Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                           model_name="gcnii", mode=mode, assign_scheme="uniform", logger_level="WARNING", num_epoches=1,
                           exp_path=f"{tmp}/exp", gcnii_layers=layers))
    eng, ex = engine.ctx, comm.ctx.comm_buffer.p2p
    Lc, alpha, theta = tr.model.layers, tr.model.alpha, tr.model.theta
    H = tr.model.convs[0].weight.shape[0]
    ru.sync_seed()
    tr.model.reset_parameters()
    ru.sync_model(tr.model)
    tr.model.drop_rate = 0.0
    sent, recv = {}, {}
    real = ops.halo_exchange

    def spy(messages, name, is_train, gathered=False, stream=None):
        sent[name] = messages.clone()
        pend = real(messages, name, is_train, gathered=gathered, stream=stream)
        with torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream()):
            recv[name] = pend.halo.clone()
        return pend

    ops.halo_exchange = spy
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
    ops.halo_exchange = real
    eng.timer.clear()
    keys = sorted(sent)
    # evaluation exchanges test0 .. test{L-1} once per pass, fp32, and is deterministic
    tr.model.eval()
    s0 = {f"test{i}": ex.seq[f"test{i}"] for i in range(Lc)}
    with torch.no_grad():
        e1 = tr.model(eng.graph, eng.feats)
        eng.timer.clear(is_train=False)
        e2 = tr.model(eng.graph, eng.feats)
        eng.timer.clear(is_train=False)
    torch.cuda.synchronize()
    ex.check_status()
    eval_ok = all(ex.seq[key] == s0[key] + 2 for key in s0) and torch.equal(e1, e2)
    layouts = comm.gather_all(eng.layout)
    mine = {"logits": logits.detach().cpu().numpy(), "loss": float(loss.detach()),
            "sent": {key: v.cpu().numpy() for key, v in sent.items()},
            "recv": {key: v.cpu().numpy() for key, v in recv.items()}}
    allr = comm.gather_all(mine)
    res = {"eval_ok": eval_ok, "keys": keys, "H": int(H), "L": int(Lc),
           "sliced": _lib.get_option("spmm_slice_cols") == 0 and H > 128 and H % 128 == 0}
    if rank == 0:
        state = {key: v.detach().cpu().numpy().astype(np.float64) for key, v in tr.model.state_dict().items()}
        want, want_loss, want_grads = _mono_step(layouts, state, Lc, alpha, theta)
        got = np.concatenate([a["logits"] for a in allr]).astype(np.float64)
        res["logit_err"] = float(np.abs(got - want).max() / np.abs(want).max())
        res["loss_err"] = abs(sum(a["loss"] for a in allr) - want_loss) / abs(want_loss)
        grads = {key: p.grad.detach().cpu().numpy().astype(np.float64) for key, p in tr.model.named_parameters()}
        res["grad_err"] = {key: float(np.abs(grads[key] - want_grads[key]).max() / (np.abs(want_grads[key]).max() + 1e-30))
                           for key in grads}
        q_err, fp_mism = 0.0, 0
        for key in keys:
            rows = [a["sent"][key].astype(np.float64) for a in allr]
            want_halo = G.exchange(rows, layouts)
            for r, Lr in enumerate(layouts):
                got_h = allr[r]["recv"][key].astype(np.float64)
                if mode in ("Vanilla", "AdaQP-p"):
                    fp_mism += int((got_h != want_halo[r]).sum())
                else:
                    lo_ = want_halo[r].min(1, keepdims=True)
                    span = want_halo[r].max(1, keepdims=True) - lo_
                    bound = span / 255 + (span + np.abs(lo_)) * 2.0 ** -8 + 1e-30
                    q_err = max(q_err, float((np.abs(got_h - want_halo[r]) / bound).max(initial=0)))
        res["fp_mismatches"], res["quant_steps"] = fp_mism, q_err
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
        res = dict(out.get(timeout=timeout) for _ in procs)
        for p in procs:
            p.join(timeout=120)
        assert all(p.exitcode == 0 for p in procs) or any("error" in v for v in res.values() if isinstance(v, dict)), \
            [p.exitcode for p in procs]
        return res


@pytest.mark.parametrize("world,mode,split,layers", [(2, "Vanilla", True, None), (2, "AdaQP-p", True, None),
                                                     (2, "AdaQP-p", False, None), (2, "AdaQP", True, None),
                                                     (2, "AdaQP-q", True, None), (3, "AdaQP-p", True, None),
                                                     (1, "Vanilla", True, None), (2, "AdaQP-p", True, 11)])
def test_training_step(world, mode, split, layers):
    res = _spawn(_step_worker, world, mode, split, layers, timeout=600)
    assert not any("error" in v for v in res.values()), [v.get("error") for v in res.values()]
    r = res[0]
    print("GCNII step", world, mode, split, layers, {key: v for key, v in r.items() if key != "keys"})
    assert all(res[i]["eval_ok"] for i in res)
    L = layers or 8
    assert r["L"] == L and r["H"] == 256 and r["sliced"]            # the sliced kernel runs inside the step
    if world > 1:
        assert r["keys"] == sorted([f"forward{i}" for i in range(L)] + [f"backward{i}" for i in range(L)])
    if mode in ("Vanilla", "AdaQP-p"):
        assert r["logit_err"] <= 2e-5 and r["loss_err"] <= 1e-5, r
        assert all(v <= 1e-3 for v in r["grad_err"].values()), r["grad_err"]
        assert r["fp_mismatches"] == 0, r
    else:
        assert r["logit_err"] <= 1e-2, r
        assert r["quant_steps"] <= 1.0, r


# ----------------------------------------------------------------------------- determinism, resume, CLI
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
                           model_name="gcnii", mode=mode, assign_scheme=scheme, logger_level="WARNING", num_epoches=3,
                           exp_path=f"{tmp}/exp", assign_cycle=2))
    rec = tr.train()
    h = hashlib.sha256()
    for key, v in tr.model.state_dict().items():
        h.update(key.encode())
        h.update(v.detach().cpu().numpy().tobytes())
    out.put((rank, (h.hexdigest(), bool(torch.isfinite(rec).all()), list(tr.losses))))


def test_determinism_adaqp_random():
    a = _spawn(_train_worker, 2, "AdaQP", "random")
    b = _spawn(_train_worker, 2, "AdaQP", "random")
    assert all(a[r][1] for r in a)
    assert a == b, (a, b)


def test_resume_is_bit_exact():
    from test_gpu_checkpoint import _resume_worker, _spawn as spawn_ckpt
    with tempfile.TemporaryDirectory() as tmp:
        a = spawn_ckpt(_resume_worker, 2, tmp, "gcnii", "AdaQP", "random", None, "straight")
        spawn_ckpt(_resume_worker, 2, tmp, "gcnii", "AdaQP", "random", None, "first")
        b = spawn_ckpt(_resume_worker, 2, tmp, "gcnii", "AdaQP", "random", None, "resume")
        with open(f"{tmp}/ckpt/epoch00003/manifest.json") as f:
            assert json.load(f)["run"]["propagation"] == {"layers": 8, "alpha": 0.1, "theta": 0.5}
    for r in (0, 1):
        ra, rb = a[r], b[r]
        assert ra["finite"] and rb["finite"]
        for key in ra["model"]:
            assert np.array_equal(ra["model"][key].view(np.uint32), rb["model"][key].view(np.uint32)), (r, key)
        assert set(ra["adam"]) == set(rb["adam"])
        for key in ra["adam"]:
            assert np.array_equal(ra["adam"][key], rb["adam"][key]), (r, key)
        assert len(rb["losses"]) == 6 and ra["losses"][3:] == rb["losses"][3:], (ra["losses"], rb["losses"])
        assert np.array_equal(ra["recorder"].view(np.uint32), rb["recorder"].view(np.uint32))


def test_main_cli_train_resume_predict(tmp_path):
    from test_gpu_checkpoint import _launch, _predictions
    ck = str(tmp_path / "ckpt")
    argv = ["--dataset", "ogbn-products", "--num_parts", "2", "--model_name", "gcnii", "--mode", "AdaQP",
            "--assign_scheme", "adaptive", "--gcnii_layers", "4", "--gcnii_alpha", "0.2", "--gcnii_theta", "1.0",
            "--checkpoint_dir", ck, "--checkpoint_every", "1"]
    env = {"ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": "0.004"}
    runs = []
    for name, extra in (("first", ["--num_epoches", "2"]), ("resumed", ["--num_epoches", "4", "--resume", "auto"]),
                        ("predict", ["--predict_out", str(tmp_path / "pred")])):
        cwd = tmp_path / name
        cwd.mkdir()
        _launch(2, argv + extra, str(cwd), env)
        runs.append(cwd)
    for cwd in runs[:2]:
        csv = cwd / "exp" / "ogbn-products" / "2part" / "gcnii" / "time" / "AdaQP_adaptive.csv"
        assert len(csv.read_text().strip().splitlines()) == 3
    assert (tmp_path / "ckpt" / "latest").read_text().strip() == "epoch00004"
    with open(os.path.join(ck, "epoch00004", "manifest.json")) as f:
        assert json.load(f)["run"]["propagation"] == {"layers": 4, "alpha": 0.2, "theta": 1.0}
    node_id, logits, header = _predictions(str(tmp_path / "pred" / "predictions.npz"))
    assert np.array_equal(node_id, np.arange(node_id.size)) and logits.shape[0] == node_id.size
    assert np.isfinite(logits).all() and 0.0 <= header["test"] <= 1.0

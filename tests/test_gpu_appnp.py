"""APPNP on the GPU: the propagation kernel (csrc/spmm.cu appnp_prop_kernel) against the float64 oracle
(oracle/appnp_oracle.py), training steps against a float64 model of the unpartitioned graph, K >= 10 exchange keys,
bitwise determinism, bit-exact resume and the CLI with the adaptive scheme.

Stated bounds:
  * kernel: |got - oracle| <= 1e-5 * (per-row L1 mass) (test_gpu_spmm.py's bound), the mass being every term of the
    step before cancellation: (1 - alpha) |A| |x| plus |alpha z| (forward) or |acc| + |alpha g| (backward);
  * fp32 training step (Vanilla, AdaQP-p): logits <= 2e-5 of max |logit|, loss <= 1e-5 relative, every parameter
    gradient <= 1e-3 of its max magnitude (test_gpu_gnn_step.py's bounds); each step's h_k within 1e-5 of the
    distributed oracle fed with the step's own z;
  * 8-bit training step (AdaQP, AdaQP-q): logits <= 1e-2 of max |logit|; every received row within one 8-bit
    quantisation step of its owner's row plus the bf16 rounding of the wire's scale and row minimum (fp32 modes:
    bit-identical).
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import appnp_oracle as P  # noqa: E402

ALPHA = 0.1


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


# ----------------------------------------------------------------------------- kernel
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


def _check_kernel(n, n_in, deg, C, seed, hub=False):
    from adaqp_b200.manager.graph import ACC_FOLD, ACC_ON, ACC_READ, LocalGraph, appnp_prop
    dev = torch.device("cuda:0")
    indptr, indices = _graph(n, deg, seed, hub)
    rng = np.random.RandomState(seed)
    x = rng.randn(n, C).astype(np.float32)
    z = rng.randn(n_in, C).astype(np.float32)
    acc0 = rng.randn(n_in, C).astype(np.float32)
    ip = indptr[:n_in + 1]
    ix = indices[:ip[-1]]
    deg_all = np.diff(indptr)
    L = LocalGraph(ip, ix.astype(np.int32), deg_all, deg_all, n_in, n - n_in, dev)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(dev)  # noqa: E731
    # halo rows as the exchange leaves them: [num_remote, C] contiguous (4-byte aligned rows for odd C)
    xl, xh = T(x[:n_in]), (T(x[n_in:]) if n > n_in else None)
    zt = T(z)
    worst = {}

    def check(name, got, ref, mass):
        ratio = np.abs(got.cpu().numpy().astype(np.float64) - ref) / (mass + 1e-30)
        worst[name] = float(ratio.max())
        assert ratio.max() <= 1e-5, (name, C, hub, float(ratio.max()))

    for fwd in (True, False):
        pre, post = (L.norm["out_-0.5"], L.norm["in_-0.5"]) if fwd else (L.norm["in_-0.5"], L.norm["out_-0.5"])
        A = P.matrix(ip, ix, n, pre.cpu().numpy(), post.cpu().numpy())
        Aabs = abs(A)
        base = (1 - ALPHA) * (A @ x.astype(np.float64))
        m_base = (1 - ALPHA) * (Aabs @ np.abs(x).astype(np.float64))
        run = lambda **kw: appnp_prop(L, xl, xh, pre, post, 1 - ALPHA, ALPHA, **kw)  # noqa: E731
        if fwd:
            cases = {"fwd": (dict(tele=zt), base + ALPHA * z, m_base + ALPHA * np.abs(z), None)}
        else:
            own = ALPHA * x[:n_in].astype(np.float64)
            cases = {"bwd_store": (dict(acc_mode=ACC_ON), base, m_base, (own, np.abs(own))),
                     "bwd_read": (dict(acc_mode=ACC_ON | ACC_READ), base, m_base,
                                  (acc0 + own, np.abs(acc0) + np.abs(own))),
                     "bwd_fold": (dict(acc_mode=ACC_ON | ACC_READ | ACC_FOLD), base + acc0 + own,
                                  m_base + np.abs(acc0) + np.abs(own), None)}
        for name, (kw, ref, mass, acc_ref) in cases.items():
            def launch(lo=0, hi=n_in, out=None, part=None):
                a = T(acc0[lo:hi]) if "acc_mode" in kw else None
                kw2 = dict(kw, acc=a) if a is not None else dict(kw)
                if "tele" in kw2:
                    kw2["tele"] = zt[lo:hi]
                return run(row_begin=lo, row_end=hi, out=out, part=part, **kw2), a
            out, acc = launch()
            check(name, out, ref, mass)
            if acc_ref is not None:
                check(name + "_acc", acc, acc_ref[0], acc_ref[1])
            # repeated launches and two row ranges of the one CSR are bitwise equal to the one launch
            out_b, acc_b = launch()
            assert torch.equal(out_b, out) and (acc is None or torch.equal(acc_b, acc)), name
            k = n_in // 3
            o1, a1 = launch(0, k)
            o2, a2 = launch(k, n_in)
            assert torch.equal(torch.cat([o1, o2]), out), name
            assert acc is None or torch.equal(torch.cat([a1, a2]), acc), name
            # local + halo two passes against the one pass and the oracle
            if xh is not None:
                o_two, a_two = launch(part="local")
                run(row_begin=0, row_end=n_in, out=o_two, part="halo")
                check(name + "_two_pass", o_two, ref, mass)
                assert acc is None or torch.equal(a_two, acc), name
            # rows outside the launched range are left untouched
            sentinel = -12345.5
            buf = torch.full((n_in + 6, C), sentinel, dtype=torch.float32, device=dev)
            lo, hi = n_in // 4, n_in // 2
            launch(lo, hi, out=buf[3:3 + hi - lo])
            assert bool((buf[:3] == sentinel).all()) and bool((buf[3 + hi - lo:] == sentinel).all()), name
            assert torch.equal(buf[3:3 + hi - lo], out[lo:hi]), name
    print(f"APPNP kernel C={C} hub={hub} halo={n > n_in}: worst error / mass {worst}")


@pytest.mark.parametrize("C", [41, 47, 100, 107, 256])
@pytest.mark.parametrize("halo", [True, False])
def test_kernel_matches_oracle(C, halo):
    _check_kernel(3000, 2000 if halo else 3000, 8, C, seed=C + halo)


def test_kernel_hub_above_100k():
    """A node adjacent to all of 101 000 others (halo neighbours included) stays within the bound at full degree."""
    _check_kernel(101_001, 60_000, 2, 47, seed=5, hub=True)


# ----------------------------------------------------------------------------- training steps
def _mono_step(layouts, state, n_layers, k, alpha):
    """float64 torch model on the unpartitioned graph (dropout off): logits, loss and parameter gradients."""
    import torch.nn.functional as F
    indptr, indices, base = P.global_from_layouts(layouts)
    N = int(base[-1])
    dst = torch.from_numpy(np.repeat(np.arange(N), np.diff(indptr)))
    src = torch.from_numpy(indices)
    x = torch.from_numpy(np.concatenate([L.feat for L in layouts]).astype(np.float64))
    y = torch.from_numpy(np.concatenate([L.label for L in layouts]).astype(np.int64))
    train = torch.from_numpy(np.concatenate([L.train_mask for L in layouts]).astype(bool))
    Pm = {key: torch.tensor(v, dtype=torch.float64, requires_grad=True) for key, v in state.items()}
    h = x
    for i in range(n_layers):
        h = h @ Pm[f"lins.{i}.weight"] + Pm[f"lins.{i}.bias"]
        if i < n_layers - 1:
            h = F.relu(F.layer_norm(h, (h.shape[1],), Pm[f"norms.{i}.weight"], Pm[f"norms.{i}.bias"], 1e-5))
    h = P.torch_appnp(src, dst, h, k, alpha)
    loss = F.cross_entropy(h[train], y[train], reduction="sum") / int(train.sum())
    loss.backward()
    return h.detach().numpy(), float(loss), {key: v.grad.numpy() for key, v in Pm.items()}


def _step_worker(rank, world, port, tmp, mode, split, k, out):
    try:
        _step(rank, world, port, tmp, mode, split, k, out)
    except Exception:                           # noqa: BLE001 - reported to the parent instead of a timeout
        import traceback
        out.put((rank, {"error": traceback.format_exc()}))
        raise


def _step(rank, world, port, tmp, mode, split, k, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": str(rank % torch.cuda.device_count()), "ADAQP_SYNTH_SCALE": "0.002",
                       "ADAQP_SEED": "11", "ADAQP_SYNTHETIC": "1", "ADAQP_MARGINAL_SPLIT": "1" if split else "0"})
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    from adaqp_b200.communicator import Communicator as comm
    from adaqp_b200.manager import GraphEngine as engine
    from adaqp_b200.model import ops
    from adaqp_b200.trainer import runtime_util as ru
    tr = Trainer(Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                           model_name="appnp", mode=mode, assign_scheme="uniform", logger_level="WARNING", num_epoches=1,
                           exp_path=f"{tmp}/exp", appnp_k=k))
    eng, ex = engine.ctx, comm.ctx.comm_buffer.p2p
    K, alpha = tr.model.k, tr.model.alpha
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
    # evaluation exchanges test0 .. test{K-1} once per pass, fp32
    tr.model.eval()
    s0 = {f"test{i}": ex.seq[f"test{i}"] for i in range(K)}
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
    res = {"eval_ok": eval_ok, "keys": keys}
    if rank == 0:
        state = {key: v.detach().cpu().numpy().astype(np.float64) for key, v in tr.model.state_dict().items()}
        want, want_loss, want_grads = _mono_step(layouts, state, len(tr.model.lins), K, alpha)
        got = np.concatenate([a["logits"] for a in allr]).astype(np.float64)
        res["logit_err"] = float(np.abs(got - want).max() / np.abs(want).max())
        res["loss_err"] = abs(sum(a["loss"] for a in allr) - want_loss) / abs(want_loss)
        grads = {key: p.grad.detach().cpu().numpy().astype(np.float64) for key, p in tr.model.named_parameters()}
        res["grad_err"] = {key: float(np.abs(grads[key] - want_grads[key]).max() / (np.abs(want_grads[key]).max() + 1e-30))
                           for key in grads}
        # per step: what each rank received at halo position j against its owner's row (the exchange oracle)
        q_err, fp_mism = 0.0, 0
        for key in keys:
            rows = [a["sent"][key].astype(np.float64) for a in allr]
            want_halo = P.exchange(rows, layouts)
            for r, L in enumerate(layouts):
                got_h = allr[r]["recv"][key].astype(np.float64)
                if mode in ("Vanilla", "AdaQP-p"):
                    fp_mism += int((got_h != want_halo[r]).sum())
                else:
                    # one 8-bit step of stochastic rounding, plus the bf16 rounding (2^-9 relative) of the wire's
                    # scale and row minimum: |q / scale - q / scale_bf16| <= span 2^-8, |rmin - rmin_bf16| <= |rmin| 2^-8
                    lo_ = want_halo[r].min(1, keepdims=True)
                    span = want_halo[r].max(1, keepdims=True) - lo_
                    bound = span / 255 + (span + np.abs(lo_)) * 2.0 ** -8 + 1e-30
                    q_err = max(q_err, float((np.abs(got_h - want_halo[r]) / bound).max(initial=0)))
        res["fp_mismatches"], res["quant_steps"] = fp_mism, q_err
        # per step h_k against the distributed oracle fed with this step's z (fp32 modes)
        if mode in ("Vanilla", "AdaQP-p"):
            zs = [a["sent"]["forward0"].astype(np.float64) for a in allr]
            hs, _ = P.dist_forward(layouts, zs, K, alpha)
            res["h_err"] = max(float(np.abs(allr[r]["sent"][f"forward{s}"] - hs[r][s - 1]).max() /
                                     np.abs(hs[r][s - 1]).max()) for r in range(world) for s in range(1, K))
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


@pytest.mark.parametrize("world,mode,split,k", [(2, "Vanilla", True, None), (2, "AdaQP-p", True, None),
                                                (2, "AdaQP-p", False, None), (2, "AdaQP", True, None),
                                                (2, "AdaQP-q", True, None), (3, "AdaQP-p", True, None),
                                                (1, "Vanilla", True, None), (2, "AdaQP-p", True, 12)])
def test_training_step(world, mode, split, k):
    res = _spawn(_step_worker, world, mode, split, k, timeout=400)
    assert not any("error" in v for v in res.values()), [v.get("error") for v in res.values()]
    r = res[0]
    print("APPNP step", world, mode, split, k, {key: v for key, v in r.items() if key != "keys"})
    assert all(res[i]["eval_ok"] for i in res)
    K = k or 10
    if world > 1:
        assert r["keys"] == sorted([f"forward{i}" for i in range(K)] + [f"backward{i}" for i in range(K)])
    if mode in ("Vanilla", "AdaQP-p"):
        assert r["logit_err"] <= 2e-5 and r["loss_err"] <= 1e-5, r
        assert all(v <= 1e-3 for v in r["grad_err"].values()), r["grad_err"]
        assert r["fp_mismatches"] == 0 and r["h_err"] <= 1e-5, r
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
                           model_name="appnp", mode=mode, assign_scheme=scheme, logger_level="WARNING", num_epoches=3,
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
        a = spawn_ckpt(_resume_worker, 2, tmp, "appnp", "AdaQP", "random", None, "straight")
        spawn_ckpt(_resume_worker, 2, tmp, "appnp", "AdaQP", "random", None, "first")
        b = spawn_ckpt(_resume_worker, 2, tmp, "appnp", "AdaQP", "random", None, "resume")
        with open(f"{tmp}/ckpt/epoch00003/manifest.json") as f:
            import json
            assert json.load(f)["run"]["propagation"] == {"k": 10, "alpha": 0.1}
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


def test_main_cli_appnp_adaptive(tmp_path):
    port = _free_port()
    procs = []
    for r in range(2):
        env = dict(os.environ)
        env.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(r), "WORLD_SIZE": "2",
                    "LOCAL_RANK": str(r % torch.cuda.device_count()), "ADAQP_SYNTHETIC": "1",
                    "ADAQP_SYNTH_SCALE": "0.004", "ADAQP_NUM_EPOCHES": "3", "ADAQP_SEED": "5", "PYTHONPATH": ROOT})
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "main.py"), "--dataset", "ogbn-products",
                                       "--num_parts", "2", "--model_name", "appnp", "--mode", "AdaQP", "--assign_scheme",
                                       "adaptive", "--appnp_k", "4", "--appnp_alpha", "0.2", "--logger_level",
                                       "WARNING"], cwd=str(tmp_path), env=env,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=900)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), [o[-3000:] for o in outs]
    csv = tmp_path / "exp" / "ogbn-products" / "2part" / "appnp" / "time" / "AdaQP_adaptive.csv"
    assert csv.exists()
    assert len(csv.read_text().strip().splitlines()) == 3

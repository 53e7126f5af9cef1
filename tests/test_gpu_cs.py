"""Correct & Smooth on the GPU: its three kernels against float64 (csrc/cs.cu, csrc/spmm.cu cs_prop_kernel), the clamp
step bitwise against APPNP's teleport step, and the distributed pass of two ranks sharing one GPU against the float64
oracle (oracle/cs_oracle.py), in the overlapped (AdaQP) and the plain (Vanilla) schedule, and one rank from the same
weights: repeatable bit for bit and blind to val / test labels.  main.py end to end with and without the flag.

Stated bounds:
  * cs_prop: |got - float64| <= 1e-5 * (per-row L1 mass of the step) (test_gpu_appnp.py's bound); fixed rows bitwise;
  * cs_init: yhat and e0 within 1e-6, the L1 sum within 1e-6 relative; cs_combine within 1e-6 of float64 on the same
    fp32 inputs, labelled rows bitwise one-hot;
  * the whole pass: 1e-4 absolute on the probabilities against the oracle fed the same base logits, over the rows whose
    float64 autoscale is not within 1e-3 relative of the 1000 cut-off (a discontinuity); those rows are counted and
    must be under 1 % of the rows.
"""
import json
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
from oracle import cs_oracle as CS  # noqa: E402

PROB_TOL = 1e-4


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _graph(n, deg, seed):
    import scipy.sparse as sp
    rng = np.random.RandomState(seed)
    m = n * deg // 2
    a, b = rng.randint(0, n, m), rng.randint(0, n, m)
    A = sp.coo_matrix((np.ones(a.size * 2), (np.r_[a, b], np.r_[b, a])), shape=(n, n)).tocsr()
    A.setdiag(0)
    A.eliminate_zeros()
    A = (A + sp.eye(n)).tocsr()
    A.sort_indices()
    return A.indptr.astype(np.int64), A.indices.astype(np.int64)


# ----------------------------------------------------------------------------- kernels
# every rung of the width ladder: contiguous rows of these widths take <VEC, CHUNKS> = <1,1> (1, 3, 7), <1,2> (41, 47),
# <4,1> (100, 128), <2,1> (34), <2,2> (66), <2,4> (130), <2,8> (450), <2,16> (514), <1,4> (97), <1,8> (129),
# <1,16> (257), <1,32> (1023), <4,2> (200), <4,4> (300), <4,8> (1000)
WIDTHS = [1, 3, 7, 41, 47, 100, 128, 34, 66, 130, 450, 514, 97, 129, 257, 1023, 200, 300, 1000]


@pytest.mark.parametrize("C", WIDTHS)
def test_prop_kernel(C):
    from adaqp_b200 import cs
    from adaqp_b200.manager.graph import LocalGraph, appnp_prop
    dev = torch.device("cuda:0")
    n, n_in = 3000, 2000
    indptr, indices = _graph(n, 8, seed=C)
    rng = np.random.RandomState(C)
    x = (rng.randn(n, C) * 1.5).astype(np.float32)
    tele = rng.randn(n_in, C).astype(np.float32)
    fix = rng.randn(n_in, C).astype(np.float32)
    y = np.where(rng.rand(n_in) < 0.3, rng.randint(0, C, n_in), -1).astype(np.int32)
    ip, deg = indptr[:n_in + 1], np.diff(indptr)
    ix = indices[:ip[-1]]
    L = LocalGraph(ip, ix.astype(np.int32), deg, deg, n_in, n - n_in, dev)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    xl, xh, tt, ft, yt = T(x[:n_in]), T(x[n_in:]), T(tele), T(fix), T(y)
    pre, post = L.norm["out_-0.5"], L.norm["in_-0.5"]
    A = P.matrix(ip, ix, n, pre.cpu().numpy(), post.cpu().numpy())
    a = 0.8
    ax, mass = a * (A @ x.astype(np.float64)), a * (abs(A) @ np.abs(x).astype(np.float64))
    worst = 0.0
    for mode in ("clamp", "fix"):
        if mode == "clamp":
            kw = dict(tele=tt, lo=-1.0, hi=1.0)
            ref = np.clip(ax + (1 - a) * tele, -1.0, 1.0)
            m = mass + (1 - a) * np.abs(tele)
        else:
            kw = dict(y=yt, fix=ft)
            ref = np.where((y >= 0)[:, None], fix, ax)
            m = mass

        def run(lo=0, hi=n_in, out=None):
            sub = {k: (v[lo:hi] if isinstance(v, torch.Tensor) else v) for k, v in kw.items()}
            return cs.prop(L, xl, xh, pre, post, a, 1 - a, lo, hi, out=out, **sub)

        got = run()
        ratio = np.abs(got.cpu().numpy() - ref) / (m + 1e-30)
        worst = max(worst, float(ratio.max()))
        assert ratio.max() <= 1e-5, (mode, C, float(ratio.max()))
        if mode == "fix":
            lab = y >= 0
            assert np.array_equal(got.cpu().numpy()[lab], fix[lab])
        # a repeat and two row ranges are bitwise the one launch; rows outside the range are untouched
        assert torch.equal(run(), got)
        k = n_in // 3
        assert torch.equal(torch.cat([run(0, k), run(k, n_in)]), got)
        buf = torch.full((n_in + 6, C), -12345.5, dtype=torch.float32, device=dev)
        lo, hi = n_in // 4, n_in // 2
        run(lo, hi, out=buf[3:3 + hi - lo])
        assert bool((buf[:3] == -12345.5).all()) and bool((buf[3 + hi - lo:] == -12345.5).all())
        assert torch.equal(buf[3:3 + hi - lo], got[lo:hi])
    # unbounded clamp = APPNP's teleport step, bit for bit
    want = appnp_prop(L, xl, xh, pre, post, a, 1 - a, tele=tt)
    assert torch.equal(cs.prop(L, xl, xh, pre, post, a, 1 - a, tele=tt), want)
    print(f"cs_prop C={C}: worst error / mass {worst:.2e}")


@pytest.mark.parametrize("C", [1, 7, 47, 100, 1024])
def test_init_kernel(C):
    from adaqp_b200 import cs
    dev = torch.device("cuda:0")
    n = 5000
    rng = np.random.RandomState(C)
    z = (rng.randn(n, C) * 4).astype(np.float32)
    z[:10] += 80.0                            # large logits: the row maximum is subtracted
    y = np.where(rng.rand(n) < 0.4, rng.randint(0, C, n), -1).astype(np.int32)
    zt, yt = torch.from_numpy(z).to(dev), torch.from_numpy(y).to(dev)
    yhat, e0, l1 = cs.init(zt, yt)
    want_p = CS.softmax(z)
    want_e = np.where((y >= 0)[:, None], CS.onehot(y, C) - want_p, 0.0)
    assert np.abs(yhat.cpu().numpy() - want_p).max() <= 1e-6
    assert np.abs(e0.cpu().numpy() - want_e).max() <= 1e-6
    assert (e0.cpu().numpy()[y < 0] == 0).all()
    assert abs(l1 - np.abs(want_e).sum()) <= 1e-6 * np.abs(want_e).sum()
    # the partials do not depend on scheduling
    _, _, l1b = cs.init(zt, yt)
    assert l1b == l1


@pytest.mark.parametrize("auto", [True, False])
def test_combine_kernel(auto):
    from adaqp_b200 import cs
    dev = torch.device("cuda:0")
    n, C = 4000, 47
    rng = np.random.RandomState(3)
    yhat = CS.softmax(rng.randn(n, C)).astype(np.float32)
    e = (rng.randn(n, C) * 0.1).astype(np.float32)
    e[:20] = 0.0                                          # zero L1: scale 1
    e[20:40] *= 1e-6                                      # ratio far above 1000: scale 1
    y = np.where(rng.rand(n) < 0.2, rng.randint(0, C, n), -1).astype(np.int32)
    y[:40] = -1
    sigma, scale = 0.37, 1.7
    T = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
    got = cs.combine(T(yhat), T(e), T(y), **(dict(sigma=sigma) if auto else dict(scale=scale))).cpu().numpy()
    e64 = e.astype(np.float64)
    s = CS.autoscale(sigma, e64) if auto else np.full(n, scale)
    if auto:
        assert (s[:40] == 1.0).all() and (CS.autoscale_ratio(sigma, e64)[20:40] > 1000).all()
    want = np.where((y >= 0)[:, None], CS.onehot(y, C), yhat + s[:, None] * e64)
    assert np.abs(got - want).max() <= 1e-6 * max(1.0, float(np.abs(want).max()))
    lab = y >= 0
    assert np.array_equal(got[lab], CS.onehot(y, C)[lab].astype(np.float32))


# ----------------------------------------------------------------------------- two ranks on one GPU
def _env(rank, world, port, tmp):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": str(rank % torch.cuda.device_count()), "ADAQP_SYNTH_SCALE": "0.004",
                       "ADAQP_SEED": "17", "ADAQP_SYNTHETIC": "1"})
    sys.path.insert(0, ROOT)
    os.chdir(tmp)


def _args(world, tmp, mode, **kw):
    from argparse import Namespace
    return Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://", model_name="gcn",
                     mode=mode, assign_scheme="uniform", logger_level="WARNING", num_epoches=5, exp_path=f"{tmp}/exp",
                     checkpoint_dir=f"{tmp}/ckpt", **kw)


def _pass_worker(rank, world, port, tmp, train, modes, out):
    try:
        _env(rank, world, port, tmp)
        from adaqp_b200 import Trainer
        if train:
            Trainer(_args(world, tmp, "AdaQP")).train()
        out.put((rank, {mode: _cs_check(rank, tmp, world, mode) for mode in modes}))
    except Exception:                           # noqa: BLE001 - reported to the parent instead of a timeout
        import traceback
        out.put((rank, {"error": traceback.format_exc()}))
        raise


def _cs_check(rank, tmp, world, mode):
    """Predict from the trained weights, run C&S (autoscale: twice, then with val / test labels permuted; fixed scale
    once) and compare with the float64 oracle fed the same logits on rank 0."""
    from adaqp_b200 import Trainer
    from adaqp_b200.communicator import Communicator as comm
    from adaqp_b200.cs import cs_params
    from adaqp_b200.manager import GraphEngine as engine
    tr = Trainer(_args(world, tmp, mode, correct_and_smooth=True))
    eng = engine.ctx
    logits = tr.predict(f"{tmp}/ckpt/best")
    p1 = tr.correct_and_smooth(logits)
    metrics = list(tr.cs_metrics)
    p2 = tr.correct_and_smooth(logits)
    # val / test labels are never read: permuting them leaves the result bit for bit
    hidden = torch.cat([eng.val_mask, eng.test_mask])
    g = torch.Generator().manual_seed(rank)
    perm = hidden[torch.randperm(hidden.numel(), generator=g).to(hidden.device)]
    eng.labels[hidden] = eng.labels[perm].clone()
    p3 = tr.correct_and_smooth(logits)
    tr.cs = cs_params(scale=1.3)
    pf = tr.correct_and_smooth(logits)
    torch.cuda.synchronize()
    comm.ctx.comm_buffer.p2p.check_status()
    y = np.full(eng.num_inner, -1, np.int64)
    tm = eng.train_mask.cpu().numpy()
    y[tm] = eng.labels.cpu().numpy()[tm]
    mine = {"logits": logits.cpu().numpy().astype(np.float64), "y": y, "auto": p1.cpu().numpy(),
            "fixed": pf.cpu().numpy()}
    allr = comm.gather_all(mine)
    layouts = comm.gather_all(eng.layout)
    res = {"repeat": torch.equal(p1, p2), "blind": torch.equal(p1, p3), "metrics": metrics}
    if rank == 0:
        zs, ys = [a["logits"] for a in allr], [a["y"] for a in allr]
        for name, scale in (("auto", None), ("fixed", 1.3)):
            want = CS.distributed(layouts, zs, ys, 50, 0.8, 50, 0.8, scale)
            got = np.concatenate([a[name] for a in allr]).astype(np.float64)
            ref = np.concatenate(want["g"])
            keep = np.ones(got.shape[0], bool)
            if scale is None:
                ratio = np.concatenate(want["ratio"])
                keep = ~(np.abs(ratio / CS.CUTOFF - 1.0) <= 1e-3)
            res[name] = {"err": float(np.abs(got - ref)[keep].max()), "excluded": int((~keep).sum()),
                         "rows": int(keep.size)}
    comm.ctx.delete_buffer()
    return res


def _spawn(world, tmp, *args, timeout=600):
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_pass_worker, args=(r, world, port, tmp) + args + (out,)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        res = dict(out.get(timeout=timeout) for _ in procs)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.kill()
                p.join()
    assert not any("error" in v for v in res.values()), [v.get("error") for v in res.values()]
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return res


def _check(res, world, mode):
    print(f"C&S W={world} {mode}: {res[0][mode]['auto']} (auto), {res[0][mode]['fixed']} (fixed); "
          f"accuracy {res[0][mode]['metrics']}")
    assert all(res[r][mode]["repeat"] and res[r][mode]["blind"] for r in res), res
    for name in ("auto", "fixed"):
        r = res[0][mode][name]
        assert r["err"] <= PROB_TOL, (world, mode, name, r)
        assert r["excluded"] <= 0.01 * r["rows"], (world, mode, name, r)
    assert all(0.0 <= m <= 1.0 for m in res[0][mode]["metrics"])


# ----------------------------------------------------------------------------- main.py
def _launch(world, argv, cwd, extra_env, timeout=600):
    port = _free_port()
    procs = []
    for r in range(world):
        env = dict(os.environ)
        env.pop("ADAQP_NUM_EPOCHES", None)
        env.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(r), "WORLD_SIZE": str(world),
                    "LOCAL_RANK": str(r % torch.cuda.device_count()), "PYTHONPATH": ROOT})
        env.update(extra_env)
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "main.py"), "--logger_level", "WARNING"] + argv,
                                      cwd=cwd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    try:
        outs = [p.communicate(timeout=timeout)[0] for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    assert all(p.returncode == 0 for p in procs), [o[-3000:] for o in outs]
    return outs


def _npz(path):
    z = np.load(path, allow_pickle=False)
    return {k: z[k] for k in z.files}, json.loads(bytes(z["header_json"]).decode("utf-8"))


def test_distributed_pass_and_cli():
    """A GCN trained for 5 epochs at W = 2 (AdaQP), then C&S of its predictions: two ranks sharing one GPU in the
    overlapped (AdaQP) and the plain (Vanilla) schedule, and one rank from the same weights, each against the float64
    oracle fed the same logits; then main.py --predict_out with and without --correct_and_smooth."""
    with tempfile.TemporaryDirectory() as tmp:
        two = _spawn(2, tmp, True, ("AdaQP", "Vanilla"))
        for mode in ("AdaQP", "Vanilla"):
            _check(two, 2, mode)
        _check(_spawn(1, tmp, False, ("Vanilla",)), 1, "Vanilla")
        env = {"ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": "0.004", "ADAQP_SEED": "17"}
        common = ["--dataset", "ogbn-products", "--num_parts", "2", "--model_name", "gcn", "--mode", "AdaQP",
                  "--assign_scheme", "uniform", "--checkpoint_dir", os.path.join(tmp, "ckpt")]
        _launch(2, common + ["--predict_out", os.path.join(tmp, "plain")], tmp, env)
        _launch(2, common + ["--predict_out", os.path.join(tmp, "cs"), "--correct_and_smooth", "--cs_scale", "auto"],
                tmp, env)
        plain, hp = _npz(os.path.join(tmp, "plain", "predictions.npz"))
        z, h = _npz(os.path.join(tmp, "cs", "predictions.npz"))
    # without the flag: today's keys and header; with it: cs_probs and the C&S header fields on top
    assert sorted(plain) == ["header_json", "logits", "node_id"]
    assert sorted(hp) == ["checkpoint", "epoch", "metric", "num_parts", "test", "train", "val"]
    assert sorted(z) == ["cs_probs", "header_json", "logits", "node_id"]
    assert np.array_equal(z["logits"], plain["logits"]) and np.array_equal(z["node_id"], plain["node_id"])
    assert h["correct_and_smooth"] == {"correct_layers": 50, "correct_alpha": 0.8, "smooth_layers": 50,
                                       "smooth_alpha": 0.8, "scale": "auto"}
    assert all(0.0 <= h[k] <= 1.0 for k in ("cs_train", "cs_val", "cs_test"))
    assert set(h) - {"correct_and_smooth", "cs_train", "cs_val", "cs_test"} == set(hp)
    assert z["cs_probs"].dtype == np.float32 and z["cs_probs"].shape == z["logits"].shape
    assert np.isfinite(z["cs_probs"]).all() and (z["cs_probs"] >= 0).all() and (z["cs_probs"] <= 1).all()

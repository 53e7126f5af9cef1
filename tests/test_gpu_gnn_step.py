"""One distributed GCN / GraphSAGE (mean, gcn) training step against float64 references.

Each case spawns W ranks on synthetic partitions, takes one training step (forward, loss, backward,
average_gradients; dropout off) and checks:

  * per layer, every mode: each aggregation the step ran (DistAggConv / DistAggSAGE, forward and backward) against
    the float64 oracle (oracle.gcn_aggregation, sage_aggregation, sage_gcn_aggregation) fed this rank's local input
    and the halo rows the kernel actually read (the exchange's receive slab, dequantised in the quantised modes):
    |got - oracle| <= 1e-5 * (L1 mass of the element's terms), test_gpu_spmm.py's bound taken per element rather
    than per row, and halved (worst observed on an H100 at the default power limit: 1.8e-6).  The keys that ran are forward0..2 and backward1..2: the layer-0 input (the features)
    needs no gradient, so autograd never calls the layer-0 backward aggregation;
  * fp32 exchange (Vanilla, AdaQP-p) against the float64 model of the unpartitioned graph (oracle/gnn_oracle.py):
    logits within 2e-5 of max |logit| and loss within 1e-5 relative (worst observed 3.0e-6 and 8.0e-7), every
    parameter gradient within 1e-3 of its max magnitude (the GAT step test's bound; worst observed 3.0e-4).  The
    GEMMs are 3xTF32, about 1.3e-6 of |dy| |W| per element of dx (1e-7 for fp32), and the GCN bias-like
    gradients (convs.l.bias, norms.l.bias, and convs.l.weight through them) are sums over thousands of rows that
    largely cancel, so those reach 1e-4 - 3e-4 of their max while SAGE's stay below 5e-6; with ADAQP_GEMM=0
    (fp32 torch GEMMs) every gradient is within 3e-7;
  * 8-bit exchange (AdaQP, AdaQP-q): logits within 1e-2 of max |logit| of the float64 step (worst observed 8.9e-4).

The same worker runs on CPU/gloo in tests/test_gnn_step_cpu.py (whole-step checks only: the per-layer check reads
the p2p receive slab).
"""
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

KEYS = ["backward1", "backward2", "forward0", "forward1", "forward2"]
LAYER_TOL = 1e-5
LOGIT_TOL, LOSS_TOL, GRAD_TOL, QUANT_LOGIT_TOL = 2e-5, 1e-5, 1e-3, 1e-2


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _oracle_fn(model, agg):
    from oracle import oracle as O
    if model == "gcn":
        return O.gcn_aggregation
    return {"mean": O.sage_aggregation, "gcn": O.sage_gcn_aggregation}[agg]


def layer_checks(rec, recv, ip, ix, in_deg, out_deg, n_inner, fn):
    """Worst |got - oracle| / mass per recorded aggregation key (mass: the oracle fed |x|, every norm positive)."""
    worst = {}
    for key, (x, got) in rec.items():
        x_all = np.concatenate([x, recv[key]]).astype(np.float32)
        bwd = key.startswith("backward")
        want = fn(ip, ix, x_all, in_deg, out_deg, n_inner, backward=bwd)
        mass = fn(ip, ix, np.abs(x_all), in_deg, out_deg, n_inner, backward=bwd)
        err = np.abs(got.astype(np.float64) - want)
        assert np.all((err == 0) | (mass > 0)), key
        worst[key] = float((err / np.maximum(mass, 1e-300)).max())
    return worst


def whole_step(layouts, state, model, agg, logits, loss, grads):
    """Rank 0: the distributed step (logits gathered in rank order, summed loss, averaged gradients) against the
    float64 model.  Returns the relative errors."""
    from oracle import gnn_oracle as GO
    want, want_loss, want_grads, (in_deg, out_deg) = GO.mono_step(layouts, state, model, agg)
    base = np.concatenate([[0], np.cumsum([L.n_inner for L in layouts])])
    for r, L in enumerate(layouts):      # the layouts' global degrees are those of the edge list the model sees
        assert np.array_equal(np.asarray(L.in_degrees[:L.n_inner], np.float64), in_deg[base[r]:base[r + 1]])
        assert np.array_equal(np.asarray(L.out_degrees[:L.n_inner], np.float64), out_deg[base[r]:base[r + 1]])
    assert np.array_equal(in_deg, out_deg)                    # symmetric: see tests/test_gnn_oracle_cpu.py
    res = {"logit_err": float(np.abs(logits - want).max() / np.abs(want).max()),
           "loss_err": abs(loss - want_loss) / abs(want_loss)}
    assert set(grads) == set(want_grads), (sorted(grads), sorted(want_grads))
    res["grad_err"] = {k: float(np.abs(grads[k] - want_grads[k]).max() / (np.abs(want_grads[k]).max() + 1e-30))
                       for k in grads}
    return res


def step_worker(rank, world, port, tmp, cfg, out):
    cpu = cfg.get("device") == "cpu"
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "ADAQP_SYNTH_SCALE": cfg.get("scale", "0.002"), "ADAQP_SEED": "11", "ADAQP_SYNTHETIC": "1",
                       # read once, at the first decomposed aggregation: set before the package is imported
                       "ADAQP_MARGINAL_SPLIT": cfg.get("split", "1")})
    if cpu:
        os.environ.update({"ADAQP_DEVICE": "cpu", "OMP_NUM_THREADS": "1", "LOCAL_RANK": str(rank)})
    else:
        os.environ["LOCAL_RANK"] = str(rank % torch.cuda.device_count())
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    from adaqp_b200.communicator import Communicator as comm
    from adaqp_b200.manager import DecompGraph
    from adaqp_b200.manager import GraphEngine as engine
    from adaqp_b200.model import ops
    from adaqp_b200.trainer import runtime_util as ru
    model, agg, mode = cfg["model"], cfg.get("agg", "mean"), cfg["mode"]
    tr = Trainer(Namespace(dataset=cfg.get("dataset", "ogbn-products"), num_parts=world, backend="gloo",
                           init_method="env://", model_name=model, mode=mode, assign_scheme="uniform",
                           logger_level="WARNING", num_epoches=1, exp_path=f"{tmp}/exp", aggregator_type=agg))
    eng = engine.ctx
    ru.sync_seed()
    tr.model.reset_parameters()
    ru.sync_model(tr.model)
    tr.model.drop_rate = 0.0
    Fn = ops.DistAggConv if model == "gcn" else ops.DistAggSAGE
    real_f, real_b = Fn.forward, Fn.backward
    rec = {}

    def spy_f(ctx, x, graph, layer, is_train):
        y = real_f(ctx, x, graph, layer, is_train)
        rec[f"forward{layer}"] = (x.detach().cpu().numpy().copy(), y.detach().cpu().numpy().copy())
        return y

    def spy_b(ctx, *grads):
        res = real_b(ctx, *grads)
        rec[f"backward{ctx.saved}"] = (grads[0].detach().cpu().numpy().copy(), res[0].detach().cpu().numpy().copy())
        return res

    Fn.forward, Fn.backward = staticmethod(spy_f), staticmethod(spy_b)
    tr.model.train()
    logits = tr.model(eng.graph, eng.feats)
    n_train = torch.LongTensor([eng.train_mask.numel()])
    comm.all_reduce_sum(n_train)
    loss = torch.nn.functional.cross_entropy(logits[eng.train_mask], eng.labels[eng.train_mask], reduction="sum") / int(n_train)
    tr.model.zero_grad()
    loss.backward()
    ru.average_gradients(tr.model)
    Fn.forward, Fn.backward = staticmethod(real_f), staticmethod(real_b)
    res = {"keys": sorted(rec), "n_halo": eng.num_remove}
    if not cpu:
        ex = comm.ctx.comm_buffer.p2p
        torch.cuda.synchronize()
        ex.check_status()
        recv = {k: ex.halo(k).cpu().numpy().copy() if eng.num_remove else np.zeros((0, x.shape[1]), np.float32)
                for k, (x, _) in rec.items()}
        g = eng.graph.full if isinstance(eng.graph, DecompGraph) else eng.graph
        L = eng.layout
        res["layer_worst"] = layer_checks(rec, recv, g.indptr.cpu().numpy(), g.indices.cpu().numpy().astype(np.int64),
                                          L.in_degrees, L.out_degrees, g.n_inner, _oracle_fn(model, agg))
    layouts = comm.gather_all(eng.layout)
    allr = comm.gather_all({"logits": logits.detach().cpu().numpy(), "loss": float(loss.detach())})
    if rank == 0:
        state = {k: v.detach().cpu().numpy().astype(np.float64) for k, v in tr.model.state_dict().items()}
        grads = {k: p.grad.detach().cpu().numpy().astype(np.float64) for k, p in tr.model.named_parameters()}
        res.update(whole_step(layouts, state, model, agg, np.concatenate([a["logits"] for a in allr]).astype(np.float64),
                              sum(a["loss"] for a in allr), grads))
    if not cpu:
        comm.ctx.delete_buffer()
    out.put((rank, res))


def spawn(world, cfg, timeout=900):
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    with tempfile.TemporaryDirectory() as tmp:
        procs = [ctx.Process(target=step_worker, args=(r, world, port, tmp, cfg, out)) for r in range(world)]
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=timeout)
        assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
        return dict(out.get(timeout=5) for _ in procs)


def check_step(res, world, fp32, layer_checked=True):
    r = res[0]
    assert sorted(res) == list(range(world))
    for q in res.values():
        assert q["keys"] == KEYS, q["keys"]
        if layer_checked:
            assert all(v <= LAYER_TOL for v in q["layer_worst"].values()), q["layer_worst"]
    if world > 1:
        assert all(q["n_halo"] > 0 for q in res.values())
    if fp32:
        assert r["logit_err"] <= LOGIT_TOL and r["loss_err"] <= LOSS_TOL, r
        assert all(v <= GRAD_TOL for v in r["grad_err"].values()), r["grad_err"]
    else:
        assert r["logit_err"] <= QUANT_LOGIT_TOL, r


CASES = {
    "gcn-Vanilla": (2, dict(model="gcn", mode="Vanilla")),
    "gcn-AdaQP-p": (2, dict(model="gcn", mode="AdaQP-p")),
    "gcn-AdaQP-p-one-pass-marginal": (2, dict(model="gcn", mode="AdaQP-p", split="0")),
    "gcn-AdaQP": (2, dict(model="gcn", mode="AdaQP")),
    "gcn-AdaQP-q": (2, dict(model="gcn", mode="AdaQP-q")),
    "sage_mean-Vanilla": (2, dict(model="sage", agg="mean", mode="Vanilla")),
    "sage_mean-AdaQP-p": (2, dict(model="sage", agg="mean", mode="AdaQP-p")),
    "sage_mean-AdaQP": (2, dict(model="sage", agg="mean", mode="AdaQP")),
    "sage_gcn-Vanilla": (2, dict(model="sage", agg="gcn", mode="Vanilla")),
    "sage_gcn-AdaQP-p": (2, dict(model="sage", agg="gcn", mode="AdaQP-p")),
    "sage_gcn-AdaQP-q": (2, dict(model="sage", agg="gcn", mode="AdaQP-q")),
    # 602 input features: the vec2 aggregation kernel and the GEMM at K = 602
    "reddit-gcn-Vanilla": (2, dict(model="gcn", mode="Vanilla", dataset="reddit", scale="0.002")),
    # three ranks sharing the GPUs round-robin: every rank has two peers with halos of unequal size
    "3rank-gcn-AdaQP-p": (3, dict(model="gcn", mode="AdaQP-p")),
    # no halo at all: the bench.py --gpus 1 configuration
    "1rank-gcn-Vanilla": (1, dict(model="gcn", mode="Vanilla")),
}


@pytest.mark.parametrize("case", list(CASES))
def test_training_step(case):
    world, cfg = CASES[case]
    res = spawn(world, cfg)
    r = res[0]
    print(f"\n{case}: layer worst {max(max(q['layer_worst'].values()) for q in res.values()):.3g} "
          f"logits {r['logit_err']:.3g} loss {r['loss_err']:.3g} grad {max(r['grad_err'].values()):.3g} "
          f"({max(r['grad_err'], key=r['grad_err'].get)}) halo {[res[k]['n_halo'] for k in sorted(res)]}\n"
          f"  grad {({k: float(f'{v:.3g}') for k, v in r['grad_err'].items()})}")
    check_step(res, world, fp32=cfg["mode"] in ("Vanilla", "AdaQP-p"))

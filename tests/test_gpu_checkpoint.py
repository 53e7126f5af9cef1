"""Checkpoints on the GPU (trainer/checkpoint.py), two ranks over the P2P exchange:

* resume is bit-exact: 6 epochs straight equal 3 epochs + a checkpoint, then new processes resuming to epoch 6
  (assign_cycle = 2, so bits are re-assigned after the resume point) -- weights, Adam state, losses and Recorder
  rows bit for bit -- for GCN AdaQP / random, GCN AdaQP-q / adaptive (cost model pinned: a profiled one is timed,
  so even two straight runs would differ), SAGE-pool AdaQP / uniform and GAT AdaQP-p;
* predictions: one graph partitioned by graph_partition.py at k = 2 and k = 1; trained at W = 2, predicted from
  `best/` at W = 2 and at W = 1 (another mode, too); both list every node id once, agree per node id within 2e-4
  of the logit scale, and the W = 2 logits match a float64 forward with the weights of best/model.pt;
* main.py end to end: --checkpoint_dir, then --resume auto with a higher --num_epoches, then --predict_out.
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


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


# ----------------------------------------------------------------------------- bit-exact resume
def _pinned_cost_model(rank, send_idx):
    return {f"{rank}_{p}": np.array([0.05 + 0.01 * p, 0.002]) for p in send_idx}


def _resume_worker(rank, world, port, tmp, model_name, mode, scheme, agg, phase, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": str(rank % torch.cuda.device_count()), "ADAQP_SYNTH_SCALE": "0.004",
                       "ADAQP_SEED": "23", "ADAQP_SYNTHETIC": "1"})
    sys.path.insert(0, ROOT)
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    from adaqp_b200.manager import GraphEngine as engine
    epochs = {"straight": 6, "first": 3, "resume": 6}[phase]
    kw = dict(checkpoint_dir=f"{tmp}/ckpt", checkpoint_every=3) if phase != "straight" else {}
    if phase == "resume":
        kw["resume"] = "auto"
    # the Trainer draws a first random assignment while it is built, before train() seeds the run; a resumed run
    # draws another one (here from a different seed) that the checkpoint's assignment must replace
    torch.manual_seed(99 if phase == "resume" else 23)
    tr = Trainer(Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                           model_name=model_name, mode=mode, assign_scheme=scheme, logger_level="WARNING",
                           num_epoches=epochs, exp_path=f"{tmp}/exp", assign_cycle=2, aggregator_type=agg, **kw))
    pinned = _pinned_cost_model(rank, engine.ctx.send_idx)
    if scheme == "adaptive" and phase != "resume":
        tr.assigner.cost_model = pinned
    rec = tr.train()
    res = {"model": {k: v.detach().cpu().numpy().copy() for k, v in tr.model.state_dict().items()},
           "adam": {(i, k): v.detach().cpu().numpy().copy() for i, s in tr.optimizer.state_dict()["state"].items()
                    for k, v in s.items()},
           "losses": list(tr.losses), "recorder": engine.ctx.recorder.epoches_metrics.numpy().copy(),
           "rows": {k: len(v) for k, v in tr.epoch_records.items()}, "finite": bool(torch.isfinite(rec).all())}
    if scheme == "adaptive" and phase == "resume":
        res["cost_model_restored"] = all(np.array_equal(tr.assigner.cost_model[k], v) for k, v in pinned.items())
    out.put((rank, res))


def _spawn(target, world, tmp, *args, timeout=900):
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=target, args=(r, world, port, tmp) + args + (out,)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(out.get(timeout=timeout) for _ in procs)
    for p in procs:
        p.join(timeout=120)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return res


@pytest.mark.parametrize("model_name,mode,scheme,agg", [("gcn", "AdaQP", "random", None),
                                                        ("gcn", "AdaQP-q", "adaptive", None),
                                                        ("sage", "AdaQP", "uniform", "pool"),
                                                        ("gat", "AdaQP-p", "uniform", None)])
def test_resume_is_bit_exact(model_name, mode, scheme, agg):
    with tempfile.TemporaryDirectory() as tmp:
        a = _spawn(_resume_worker, 2, tmp, model_name, mode, scheme, agg, "straight")
        _spawn(_resume_worker, 2, tmp, model_name, mode, scheme, agg, "first")
        b = _spawn(_resume_worker, 2, tmp, model_name, mode, scheme, agg, "resume")
        with open(f"{tmp}/ckpt/latest") as f:
            assert f.read().strip() == "epoch00006"
    for r in (0, 1):
        ra, rb = a[r], b[r]
        for k in ra["model"]:
            assert np.array_equal(ra["model"][k].view(np.uint32), rb["model"][k].view(np.uint32)), (r, k)
        assert set(ra["adam"]) == set(rb["adam"])
        for k in ra["adam"]:
            assert np.array_equal(ra["adam"][k], rb["adam"][k]), (r, k)
        assert len(rb["losses"]) == 6 and ra["losses"][3:] == rb["losses"][3:], (ra["losses"], rb["losses"])
        assert np.array_equal(ra["recorder"].view(np.uint32), rb["recorder"].view(np.uint32))
        assert rb["rows"] == {"assign_time": 6, "train_time": 6, "exposed_comm_ms": 6, "loss": 6}
        assert rb["finite"]
        if scheme == "adaptive":
            assert rb["cost_model_restored"]


# ----------------------------------------------------------------------------- main.py launches
def _launch(world, argv, cwd, extra_env, timeout=900):
    port = _free_port()
    procs = []
    for r in range(world):
        env = dict(os.environ)
        env.pop("ADAQP_SYNTHETIC", None)
        env.pop("ADAQP_NUM_EPOCHES", None)
        env.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(r), "WORLD_SIZE": str(world),
                    "LOCAL_RANK": str(r % torch.cuda.device_count()), "ADAQP_SEED": "5", "PYTHONPATH": ROOT})
        env.update(extra_env)
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "main.py"), "--logger_level", "WARNING"] + argv,
                                      cwd=cwd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=timeout)[0] for p in procs]
    assert all(p.returncode == 0 for p in procs), [o[-3000:] for o in outs]
    return outs


def _predictions(path):
    z = np.load(path, allow_pickle=False)
    return z["node_id"], z["logits"], json.loads(bytes(z["header_json"]).decode("utf-8"))


def test_predictions_across_partitionings():
    import yaml
    from adaqp_b200.helper.dataset import load_dataset
    from adaqp_b200.manager.graphEngine import read_rank_layout
    from adaqp_b200.manager.partition_synth import global_graph, spec_from_config
    from test_gpu_partition import _write_ogbn_fixture
    from test_gpu_trainer import _oracle_forward
    with open(os.path.join(ROOT, "adaqp_b200", "config", "ogbn-products.yaml")) as f:
        cfg = yaml.safe_load(f)
    g, _ = global_graph(spec_from_config(cfg, 2, 20000 / 2449029))
    g = g.permuted(np.random.default_rng(3).permutation(g.num_nodes))
    with tempfile.TemporaryDirectory() as tmp:
        _write_ogbn_fixture(os.path.join(tmp, "data", "dataset"), g)
        env = {k: v for k, v in os.environ.items() if k != "ADAQP_SYNTHETIC"}
        for k in (2, 1):
            r = subprocess.run([sys.executable, os.path.join(ROOT, "graph_partition.py"), "--dataset", "ogbn-products",
                                "--partition_size", str(k)], cwd=tmp, env=env, capture_output=True, text=True, timeout=900)
            assert r.returncode == 0, r.stdout + r.stderr
        N = load_dataset("ogbn-products", os.path.join(tmp, "data", "dataset")).num_nodes
        ck = os.path.join(tmp, "ckpt")
        common = ["--dataset", "ogbn-products", "--model_name", "gcn", "--assign_scheme", "uniform", "--checkpoint_dir", ck]
        _launch(2, common + ["--num_parts", "2", "--mode", "Vanilla", "--num_epoches", "6"], tmp, {})
        _launch(2, common + ["--num_parts", "2", "--mode", "Vanilla", "--predict_out", os.path.join(tmp, "p2")], tmp, {})
        # weights do not depend on the partition: predict on one rank, in another mode
        _launch(1, common + ["--num_parts", "1", "--mode", "AdaQP", "--predict_out", os.path.join(tmp, "p1")], tmp, {})
        id2, l2, h2 = _predictions(os.path.join(tmp, "p2", "predictions.npz"))
        id1, l1, h1 = _predictions(os.path.join(tmp, "p1", "predictions.npz"))
        with open(os.path.join(ck, "best", "manifest.json")) as f:
            best = json.load(f)
        state = {k: v.numpy() for k, v in torch.load(os.path.join(ck, "best", "model.pt"), weights_only=True)["model"].items()}
        layouts = [read_rank_layout(os.path.join(tmp, "data", "part_data", "ogbn-products", "2part", f"part{r}.npz"))
                   for r in range(2)]
    assert id2.dtype == np.int64 and np.array_equal(id2, np.arange(N)) and np.array_equal(id1, np.arange(N))
    assert l2.dtype == np.float32 and l2.shape == l1.shape == (N, cfg["data"]["num_classes"])
    scale = float(np.abs(l2).max())
    err_w = float(np.abs(l2.astype(np.float64) - l1).max() / scale)
    want = np.empty(l2.shape, np.float64)
    for L, y in zip(layouts, _oracle_forward(layouts, state, "gcn")):
        want[L.inner_gid] = y
    err_o = float(np.abs(l2 - want).max() / np.abs(want).max())
    print(f"predictions: W=2 vs W=1 {err_w:.2e}, W=2 vs float64 {err_o:.2e} of the logit scale; best epoch {best['epoch']}")
    assert err_w <= 2e-4 and err_o <= 2e-4
    assert h2["epoch"] == h1["epoch"] == best["epoch"] and h2["num_parts"] == 2 and h1["num_parts"] == 1
    assert abs(h2["val"] - best["val"]) < 1e-6 and h2["metric"] == "accuracy"


def test_main_cli_checkpoint_resume_predict(tmp_path):
    ck = str(tmp_path / "ckpt")
    argv = ["--dataset", "ogbn-products", "--num_parts", "2", "--model_name", "gcn", "--mode", "AdaQP",
            "--assign_scheme", "random", "--checkpoint_dir", ck, "--checkpoint_every", "1"]
    env = {"ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": "0.004"}
    runs = []
    for name, extra in (("first", ["--num_epoches", "2"]), ("resumed", ["--num_epoches", "4", "--resume", "auto"]),
                        ("predict", ["--predict_out", str(tmp_path / "pred")])):
        cwd = tmp_path / name
        cwd.mkdir()
        _launch(2, argv + extra, str(cwd), env)
        runs.append(cwd)
    for cwd in runs[:2]:
        csv = cwd / "exp" / "ogbn-products" / "2part" / "gcn" / "time" / "AdaQP_random.csv"
        assert len(csv.read_text().strip().splitlines()) == 3          # header + one row per worker
    assert (tmp_path / "ckpt" / "latest").read_text().strip() == "epoch00004"
    node_id, logits, header = _predictions(str(tmp_path / "pred" / "predictions.npz"))
    assert np.array_equal(node_id, np.arange(node_id.size)) and logits.shape[0] == node_id.size
    assert np.isfinite(logits).all() and 0.0 <= header["test"] <= 1.0

"""Checkpoints without a GPU (trainer/checkpoint.py):

* two gloo ranks on the CPU: 4 epochs straight equal 2 epochs with a checkpoint after each, then new processes
  resuming to epoch 4 -- final weights, Adam state, the epoch 3-4 losses and every Recorder row bit for bit;
  `best/` is the Recorder's argmax; the per-epoch records cover all 4 epochs;
* refusals (a manifest field that differs, a missing rank file, no epochs left, another partition), raised on
  every rank before the exchange buffers exist, and every manifest field through `resume_error`;
* `Assigner.state_dict()` round trips for the uniform, random and adaptive schemes;
* `inner_gid` from `raw_partitions` maps every inner row back to its original node id, survives the layout file,
  and a file written without it still loads.
"""
import json
import os
import shutil
import socket
import sys
import tempfile
from argparse import Namespace
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _env(rank, world, port):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank),
                       "WORLD_SIZE": str(world), "LOCAL_RANK": str(rank), "ADAQP_DEVICE": "cpu",
                       "ADAQP_SYNTH_SCALE": "0.004", "ADAQP_SEED": "7", "OMP_NUM_THREADS": "1",
                       "ADAQP_SYNTHETIC": "1"})
    sys.path.insert(0, ROOT)


def _args(tmp, world, mode, model_name, num_epoches, **kw):
    return Namespace(dataset="reddit", num_parts=world, backend="gloo", init_method="env://", model_name=model_name,
                     mode=mode, assign_scheme="uniform", logger_level="WARNING", num_epoches=num_epoches,
                     exp_path=f"{tmp}/exp", **kw)


def _summary(tr):
    from adaqp_b200.manager import GraphEngine as engine
    adam = tr.optimizer.state_dict()["state"]
    return {"model": {k: v.detach().cpu().numpy().copy() for k, v in tr.model.state_dict().items()},
            "adam": {(i, k): v.detach().cpu().numpy().copy() for i, s in adam.items() for k, v in s.items()},
            "losses": list(tr.losses), "recorder": engine.ctx.recorder.epoches_metrics.numpy().copy(),
            "records": {k: len(v) for k, v in tr.epoch_records.items()}}


def _refusals(tmp, world, mode, model_name):
    """Each case raises on every rank while the Trainer is built, before its exchange buffers exist."""
    from adaqp_b200 import Trainer
    from adaqp_b200.communicator import Communicator as comm
    src = f"{tmp}/ckpt/epoch00002"
    if os.environ["RANK"] == "0":
        # made before the first collective: rank 1 cannot reach the second case before rank 0 finished the first
        shutil.copytree(src, f"{tmp}/missing")
        os.remove(f"{tmp}/missing/rank1.pt")
        shutil.copytree(src, f"{tmp}/otherpart")
        with open(f"{tmp}/otherpart/manifest.json") as f:
            m = json.load(f)
        m["partitions"][1]["csr_sha256"] = "0" * 64
        with open(f"{tmp}/otherpart/manifest.json", "w") as f:
            json.dump(m, f)
    cases =[(dict(mode="AdaQP-p" if mode == "Vanilla" else "Vanilla", resume=src), ValueError, "'mode'"),
             (dict(resume=f"{tmp}/missing"), FileNotFoundError, "rank1.pt"),
             (dict(resume=src, num_epoches=2), ValueError, "num_epoches"),
             (dict(resume=f"{tmp}/otherpart"), ValueError, "partitions[1].csr_sha256")]
    seen = []
    for kw, kind, text in cases:
        base = dict(mode=mode, num_epoches=4)
        base.update(kw)
        try:
            Trainer(_args(tmp, world, base.pop("mode"), model_name, base.pop("num_epoches"), **base))
            seen.append(("no error", ""))
        except Exception as e:                  # noqa: BLE001 - the type and message are what is checked
            seen.append((type(e).__name__, str(e), comm.ctx.comm_buffer is None))
            assert isinstance(e, kind) and text in str(e), (kw, type(e), str(e))
    return seen


def _worker(rank, world, port, tmp, mode, model_name, phase, out):
    _env(rank, world, port)
    os.chdir(tmp)
    from adaqp_b200 import Trainer
    if phase == "first":
        a = Trainer(_args(tmp, world, mode, model_name, 4))           # run A: 4 epochs straight
        a.train()
        res = _summary(a)
        b = Trainer(_args(tmp, world, mode, model_name, 2, checkpoint_dir=f"{tmp}/ckpt", checkpoint_every=1))
        b.train()                                                      # run B: 2 epochs, a checkpoint after each
        out.put((rank, res))
        return
    refused = _refusals(tmp, world, mode, model_name) if phase == "resume+refusals" else []
    b = Trainer(_args(tmp, world, mode, model_name, 4, checkpoint_dir=f"{tmp}/ckpt", checkpoint_every=1,
                      resume="auto"))
    assert b.resume_epoch == 2
    rec = b.train()
    res = _summary(b)
    res["refused"] = refused
    res["finite"] = bool(torch.isfinite(rec).all())
    out.put((rank, res))


def _spawn(world, tmp, *args):
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, tmp) + args + (out,)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(out.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    return res


@pytest.mark.parametrize("mode,model_name,refusals", [("Vanilla", "gcn", True), ("AdaQP-p", "sage", False)])
def test_resume_is_bit_exact(mode, model_name, refusals):
    with tempfile.TemporaryDirectory() as tmp:
        a = _spawn(2, tmp, mode, model_name, "first")
        b = _spawn(2, tmp, mode, model_name, "resume+refusals" if refusals else "resume")
        with open(f"{tmp}/ckpt/best/manifest.json") as f:
            best = json.load(f)
        with open(f"{tmp}/ckpt/latest") as f:
            latest = f.read().strip()
        assert sorted(d for d in os.listdir(f"{tmp}/ckpt") if d.startswith("epoch")) == [
            "epoch00001", "epoch00002", "epoch00003", "epoch00004"]
        assert not any(d.startswith(".") for d in os.listdir(f"{tmp}/ckpt"))
    assert latest == "epoch00004"
    for r in (0, 1):
        ra, rb = a[r], b[r]
        assert set(ra["model"]) == set(rb["model"])
        for k in ra["model"]:
            assert np.array_equal(ra["model"][k].view(np.uint32), rb["model"][k].view(np.uint32)), k
        assert set(ra["adam"]) == set(rb["adam"]) and ra["adam"]
        for k in ra["adam"]:
            assert np.array_equal(ra["adam"][k], rb["adam"][k]), k
        assert len(rb["losses"]) == 4 and ra["losses"][2:] == rb["losses"][2:]
        assert np.array_equal(ra["recorder"].view(np.uint32), rb["recorder"].view(np.uint32))
        assert rb["records"] == {"assign_time": 4, "train_time": 4, "exposed_comm_ms": 4, "loss": 4}
        assert rb["finite"]
    assert best["epoch"] == int(np.argmax(b[0]["recorder"][:4, 1])) + 1
    assert best["val"] == float(b[0]["recorder"][best["epoch"] - 1, 1])
    if refusals:
        for r in (0, 1):
            assert len(b[r]["refused"]) == 4 and all(x[2] for x in b[r]["refused"]), b[r]["refused"]


# ----------------------------------------------------------------------------- refusal rules, field by field
def _fake_checkpoint(path, fields, digests, epoch=3, ranks=(0, 1)):
    from adaqp_b200.trainer import checkpoint as ck
    os.makedirs(path)
    with open(os.path.join(path, "manifest.json"), "w") as f:
        json.dump({"format": ck.FORMAT_VERSION, "epoch": epoch, "run": fields, "partitions": digests}, f)
    for name in ["model.pt"] + [f"rank{r}.pt" for r in ranks]:
        open(os.path.join(path, name), "wb").close()


def _fields():
    from adaqp_b200.trainer import checkpoint as ck
    cfg = {"data": {"num_feats": 100, "num_classes": 47}, "model": {"num_layers": 3, "hidden_dim": 256,
           "aggregator_type": "mean", "gat_heads": 4},
           "runtime": {"dataset": "ogbn-products", "model_name": "gcn", "num_parts": 2, "mode": "AdaQP",
                       "assign_scheme": "random"}}
    return ck.run_fields(cfg, None)


def test_resume_error_names_every_field(tmp_path):
    from adaqp_b200.trainer import checkpoint as ck
    fields = _fields()
    assert fields["key_dims"] == {"forward0": 100, "forward1": 256, "forward2": 256, "backward1": 256, "backward2": 256}
    digest = {"n_inner": 10, "n_halo": 3, "send_idx": {"1": [0, 4]}, "csr_sha256": "ab"}
    _fake_checkpoint(str(tmp_path / "ok"), fields, [digest, dict(digest, n_inner=11)])
    assert ck.resume_error(str(tmp_path / "ok"), fields, digest, 0, 5) is None
    changed = {"dataset": "reddit", "model_name": "sage", "aggregator_type": "gcn", "gat_heads": 2,
               "layer_dims": [100, 128, 128, 47], "num_parts": 4, "mode": "Vanilla", "assign_scheme": "adaptive",
               "key_dims": dict(fields["key_dims"], forward0=99)}
    assert set(changed) == set(ck.RUN_FIELDS)
    for k, v in changed.items():
        err = ck.resume_error(str(tmp_path / "ok"), dict(fields, **{k: v}), digest, 0, 5)
        assert isinstance(err, ValueError) and repr(k) in str(err), (k, err)
    for k, v in (("n_inner", 9), ("n_halo", 4), ("send_idx", {"1": [0, 5]}), ("csr_sha256", "cd")):
        err = ck.resume_error(str(tmp_path / "ok"), fields, dict(digest, **{k: v}), 0, 5)
        assert isinstance(err, ValueError) and f"partitions[0].{k}" in str(err), (k, err)
    err = ck.resume_error(str(tmp_path / "ok"), fields, digest, 0, 3)
    assert isinstance(err, ValueError) and "num_epoches" in str(err)
    _fake_checkpoint(str(tmp_path / "norank"), fields, [digest, digest], ranks=(0,))
    err = ck.resume_error(str(tmp_path / "norank"), fields, digest, 0, 5)
    assert isinstance(err, FileNotFoundError) and "rank1.pt" in str(err)
    assert isinstance(ck.resume_error(str(tmp_path / "none"), fields, digest, 0, 5), FileNotFoundError)
    with pytest.raises(FileNotFoundError):
        ck.resolve("auto", str(tmp_path / "none"))


# ----------------------------------------------------------------------------- Assigner state
@pytest.fixture
def fake_engine(monkeypatch):
    from adaqp_b200.helper import BitType
    from adaqp_b200.manager import GraphEngine
    monkeypatch.setattr(GraphEngine, "ctx", SimpleNamespace(bit_type=BitType.FULL))


def _round_trip(asg, tmp_path):
    from adaqp_b200.assigner import Assigner
    path = str(tmp_path / "asg.pt")
    torch.save(asg.state_dict(), path)
    back = Assigner(100, 256, 3, 6, asg.scheme, 4, {}, group_size=50, coe_lambda=0.5, assign_cycle=2)
    back.load_state_dict(torch.load(path, weights_only=True), device=torch.device("cpu"))
    assert back.is_tracing == asg.is_tracing and torch.equal(back.sample_rate, asg.sample_rate)
    assert (back.cost_model is None) == (asg.cost_model is None)
    for k, v in (asg.cost_model or {}).items():
        assert isinstance(back.cost_model[k], np.ndarray) and np.array_equal(back.cost_model[k], v)
    assert set(back.traced_layer_data) == set(asg.traced_layer_data)
    for k, v in asg.traced_layer_data.items():
        w = back.traced_layer_data[k]
        assert (torch.equal(w, v) if isinstance(v, torch.Tensor) else (w == v and isinstance(w, float))), k
    assert set(back.assignment) == set(asg.assignment)
    for k, per in asg.assignment.items():
        assert set(back.assignment[k]) == set(per)
        assert all(torch.equal(back.assignment[k][p], b) and back.assignment[k][p].dtype == torch.int32
                   for p, b in per.items())
    return back


@pytest.mark.parametrize("scheme", ["uniform", "random"])
def test_assigner_state_round_trip(scheme, fake_engine, tmp_path):
    from adaqp_b200.assigner import Assigner
    torch.manual_seed(3)
    asg = Assigner(100, 256, 3, 6, scheme, 4, {}, group_size=50, coe_lambda=0.5, assign_cycle=2)
    asg.get_assignment({1: (0, 37), 2: (37, 90)})
    _round_trip(asg, tmp_path)


def test_assigner_state_round_trip_adaptive(fake_engine, tmp_path):
    from adaqp_b200.assigner import Assigner
    asg = Assigner(100, 256, 3, 6, "adaptive", 8, {}, group_size=50, coe_lambda=0.5, assign_cycle=2)
    send_idx = {1: (0, 37), 2: (37, 90)}
    asg.get_assignment(send_idx, runtime_scheme="uniform")
    asg.cost_model = {"0_1": np.array([0.125, 0.0375]), "0_2": np.array([0.2, 0.01])}
    asg.is_tracing = True
    asg.init_traced_data(3)
    g = torch.Generator().manual_seed(1)
    asg.traced_layer_data["forward1"] = torch.rand(90, generator=g)
    asg.traced_layer_data["backward2"] = torch.rand(90, generator=g) * 1e-3
    back = _round_trip(asg, tmp_path)
    assert back.traced_layer_data["forward0"] == 0.0
    with pytest.raises(ValueError):
        Assigner(100, 256, 3, 6, "random", 8, {}, group_size=50, coe_lambda=0.5).load_state_dict(asg.state_dict())


# ----------------------------------------------------------------------------- inner_gid
def _graph(n=60, seed=0):
    import scipy.sparse as sp
    from adaqp_b200.helper.dataset import GlobalGraph
    rng = np.random.default_rng(seed)
    u, v = rng.integers(0, n, 4 * n), rng.integers(0, n, 4 * n)
    A = sp.coo_matrix((np.ones(8 * n), (np.r_[u, v], np.r_[v, u])), shape=(n, n)).tocsr()
    A.setdiag(0)
    A.eliminate_zeros()
    A = (A + sp.eye(n)).tocsr()
    A.data[:] = 1
    A.sort_indices()
    feat = np.arange(n, dtype=np.float32)[:, None] * np.ones((1, 3), np.float32)     # row v holds v
    return GlobalGraph(name="fixture", indptr=A.indptr.astype(np.int64), indices=A.indices.astype(np.int32),
                       feat=feat, label=np.arange(n) % 4, train_mask=rng.random(n) < 0.5,
                       val_mask=np.zeros(n, bool), test_mask=np.zeros(n, bool))


def test_inner_gid_maps_rows_to_original_ids(tmp_path):
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.graphEngine import read_rank_layout, save_rank_layout
    from adaqp_b200.manager.layout import layouts_from_raw, raw_partitions
    g = _graph()
    n = g.indptr.size - 1
    part = np.random.default_rng(1).integers(0, 3, n)
    lays = layouts_from_raw(raw_partitions(g, part), DistGNNType.DistGCN)
    seen = np.concatenate([L.inner_gid for L in lays])
    assert np.array_equal(np.sort(seen), np.arange(n))
    for r, L in enumerate(lays):
        assert L.inner_gid.dtype == np.int64 and L.inner_gid.shape == (L.n_inner,)
        assert np.all(part[L.inner_gid] == r)
        assert np.array_equal(L.feat[:, 0], L.inner_gid.astype(np.float32))         # row i is node inner_gid[i]
        assert np.array_equal(L.label, g.label[L.inner_gid])
        # the in-degree of every inner row is the original node's degree
        assert np.array_equal(L.in_degrees[:L.n_inner], np.diff(g.indptr)[L.inner_gid])
        back = read_rank_layout(save_rank_layout(L, str(tmp_path), "fixture"))
        assert np.array_equal(back.inner_gid, L.inner_gid)
    # a file written before the field existed still loads, without it
    path = save_rank_layout(lays[0], str(tmp_path / "old"), "fixture")
    z = dict(np.load(path, allow_pickle=False))
    z.pop("inner_gid")
    np.savez_compressed(path, **z)
    old = read_rank_layout(path)
    assert old.inner_gid is None and np.array_equal(old.indices, lays[0].indices) and old.n_inner == lays[0].n_inner


def test_synthetic_inner_gid_is_block_order():
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec, block_starts
    spec = SynthSpec(name="fixture", num_nodes=900, num_edges=900 * 8, num_parts=3, num_feats=8, num_classes=3,
                     cross_fraction=0.2, community_size=32, seed=2)
    starts = block_starts(spec)
    for r, L in enumerate(prepare_all_in_process(spec)):
        assert np.array_equal(np.sort(L.inner_gid), np.arange(starts[r], starts[r + 1]))

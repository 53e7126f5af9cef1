"""Correct & Smooth measurements on ogbn-products-shaped synthetic graphs; prints one JSON line per result.

    python tools/bench_cs.py [--kernel-scale 1.0] [--reps 20] [--scale 0.1] [--epochs 10]

* the fused step (cs_prop_kernel, C = 47, all rows of the one-rank partition) against the composition it replaces:
  clamp mode against appnp_prop + torch clamp_, fix mode against appnp_prop + an index copy of the labelled rows;
  median of --reps event-timed launches, the two variants alternated;
* the wall time of the whole C&S pass (K1 = K2 = 50, autoscale; host clock around a synchronised call, the second
  of two calls) at one rank and at two ranks sharing cuda:0, after a short GCN training (--epochs, Vanilla) on the
  synthetic partitions at --scale, and the base and C&S train / val / test accuracy of that model (synthetic data);
* the card name, power limit and max SM clock, read in the same run.
"""
import argparse
import json
import os
import socket
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
import torch.multiprocessing as mp
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"card": torch.cuda.get_device_name(0), "nvidia_smi": r.stdout.strip()}


def _port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def kernel_times(scale, reps, C=47, alpha=0.8):
    from adaqp_b200 import build
    build.build()
    from adaqp_b200 import cs
    from adaqp_b200.manager.graph import LocalGraph, appnp_prop
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import spec_from_config
    cfg = yaml.safe_load(open(os.path.join(ROOT, "adaqp_b200", "config", "ogbn-products.yaml")))
    L = prepare_all_in_process(spec_from_config(cfg, 1, scale))[0]
    dev = torch.device("cuda:0")
    g = LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, dev)
    n, nnz = L.n_inner, int(L.indptr[-1])
    pre, post = g.norm["out_-0.5"], g.norm["in_-0.5"]
    lab = torch.from_numpy(np.asarray(L.train_mask, bool)).to(dev)
    y = torch.where(lab, torch.from_numpy(np.asarray(L.label, np.int64) % C).to(dev), -1).to(torch.int32).contiguous()
    idx = torch.nonzero(lab).squeeze(1)
    x, t = torch.randn(n, C, device=dev), torch.randn(n, C, device=dev)
    fix = torch.zeros(n, C, device=dev)
    fix[idx] = torch.randn(idx.numel(), C, device=dev)
    out = torch.empty(n, C, device=dev)
    variants = {
        "clamp_fused": lambda: cs.prop(g, x, None, pre, post, alpha, 1 - alpha, out=out, tele=t, lo=-1.0, hi=1.0),
        "clamp_unfused": lambda: appnp_prop(g, x, None, pre, post, alpha, 1 - alpha, out=out, tele=t).clamp_(-1.0, 1.0),
        "fix_fused": lambda: cs.prop(g, x, None, pre, post, alpha, 1 - alpha, out=out, y=y, fix=fix),
        "fix_unfused": lambda: appnp_prop(g, x, None, pre, post, alpha, 1 - alpha, out=out).index_copy_(0, idx, fix[idx]),
    }
    times = {name: [] for name in variants}
    for name in variants:                                # warm-up of every shape
        for _ in range(3):
            variants[name]()
    for _ in range(reps):                                # alternated: one launch of every variant per round
        for name in variants:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            variants[name]()
            b.record()
            torch.cuda.synchronize()
            times[name].append(a.elapsed_time(b))
    res = [{"kernel": name, "C": C, "rows": n, "nnz": nnz, "train_share": float(lab.float().mean()),
            "median_ms": float(np.median(ts)), "min_ms": float(np.min(ts)), "reps": reps} for name, ts in times.items()]
    for m in ("clamp", "fix"):
        f, u = float(np.median(times[f"{m}_fused"])), float(np.median(times[f"{m}_unfused"]))
        res.append({"compare": m, "C": C, "fused_ms": f, "unfused_ms": u, "speedup": u / f})
    return res


def _env(rank, world, port, scale):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": "0", "ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": str(scale), "ADAQP_SEED": "1"})


def _args(world, tmp, epochs, **kw):
    from argparse import Namespace
    return Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://", model_name="gcn",
                     mode="Vanilla", assign_scheme="uniform", logger_level="WARNING", num_epoches=epochs,
                     exp_path=f"{tmp}/exp", checkpoint_dir=f"{tmp}/ckpt", **kw)


def _train_worker(rank, world, port, tmp, scale, epochs, out):
    _env(rank, world, port, scale)
    os.chdir(tmp)
    from adaqp_b200 import Trainer
    Trainer(_args(world, tmp, epochs)).train()
    out.put((rank, None))


def _cs_worker(rank, world, port, tmp, scale, epochs, out):
    _env(rank, world, port, scale)
    os.chdir(tmp)
    from adaqp_b200 import Trainer
    from adaqp_b200.communicator import Communicator as comm
    tr = Trainer(_args(world, tmp, epochs, correct_and_smooth=True))
    logits = tr.predict(f"{tmp}/ckpt/best")
    walls = []
    for _ in range(2):
        comm.barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        tr.correct_and_smooth(logits)
        torch.cuda.synchronize()
        walls.append(time.perf_counter() - t0)
    comm.ctx.delete_buffer()
    out.put((rank, {"wall_s": walls, "base": tr.predict_metrics, "cs": tr.cs_metrics}))


def _spawn(target, world, tmp, *args):
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _port()
    procs = [ctx.Process(target=target, args=(r, world, port, tmp) + args + (out,)) for r in range(world)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=3600)
    if any(p.exitcode != 0 for p in procs):
        raise RuntimeError(f"{target.__name__} failed: {[p.exitcode for p in procs]}")
    return dict(out.get(timeout=5) for _ in procs)


def cs_pass(world, scale, epochs):
    with tempfile.TemporaryDirectory() as tmp:
        _spawn(_train_worker, world, tmp, scale, epochs)
        res = _spawn(_cs_worker, world, tmp, scale, epochs)
    return {"pass": "correct_and_smooth", "k1": 50, "k2": 50, "scale_mode": "auto", "world": world,
            "synth_scale": scale, "train_epochs": epochs,
            "wall_s_first": max(v["wall_s"][0] for v in res.values()),
            "wall_s": max(v["wall_s"][1] for v in res.values()),
            "accuracy_synthetic": {"base": dict(zip(("train", "val", "test"), res[0]["base"])),
                                   "cs": dict(zip(("train", "val", "test"), res[0]["cs"]))}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kernel-scale", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--scale", type=float, default=0.1)
    ap.add_argument("--epochs", type=int, default=10)
    ap.add_argument("--skip-pass", action="store_true")
    ap.add_argument("--skip-kernels", action="store_true")
    a = ap.parse_args()
    print(json.dumps(_card()), flush=True)
    if not a.skip_kernels:
        for r in kernel_times(a.kernel_scale, a.reps):
            print(json.dumps(r), flush=True)
    if not a.skip_pass:
        for world in (1, 2):
            print(json.dumps(cs_pass(world, a.scale, a.epochs)), flush=True)
    print(json.dumps(_card()), flush=True)


if __name__ == "__main__":
    main()

"""APPNP measurements on an ogbn-products-shaped synthetic graph; prints one JSON line per result.

    python tools/bench_appnp.py [--kernel-scale 1.0] [--widths 41,47,100,107] [--reps 10] [--scale 0.1] [--epochs 6]

* the fused propagation step (appnp_prop_kernel, forward and backward) against the unfused composition it replaces --
  the CSR SpMM with post scaled by (1 - alpha), then a torch add of alpha z (forward), or a torch scale-add of
  alpha g into the dz accumulator (backward) -- over all rows of the one-rank partition, median of --reps
  event-timed launches, the two variants alternated;
* epochs/s of APPNP (K = 10, alpha = 0.1) in Vanilla and AdaQP (uniform 8-bit) at one rank and at two ranks
  sharing cuda:0 (Trainer.train's mean epoch time, first epoch included), the exposed communication per epoch and
  the bytes each rank puts on the wire per training epoch (2K exchanges of C-wide rows; quantised rows carry
  their packed bytes plus two bf16 parameters);
* the card name and power limit, read in the same run.
"""
import argparse
import json
import os
import socket
import subprocess
import sys
import tempfile

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


def kernel_times(scale, widths, reps, alpha=0.1):
    from adaqp_b200 import build
    build.build()
    from adaqp_b200.manager.graph import ACC_ON, ACC_READ, LocalGraph, appnp_prop, spmm
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import spec_from_config
    cfg = yaml.safe_load(open(os.path.join(ROOT, "adaqp_b200", "config", "ogbn-products.yaml")))
    L = prepare_all_in_process(spec_from_config(cfg, 1, scale))[0]
    dev = torch.device("cuda:0")
    g = LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, dev)
    n, nnz = L.n_inner, int(L.indptr[-1])
    pre, post = g.norm["out_-0.5"], g.norm["in_-0.5"]
    post_s = post * (1 - alpha)                          # the unfused composition's pre-scaled post norm
    res = []
    for C in widths:
        x, z = torch.randn(n, C, device=dev), torch.randn(n, C, device=dev)
        out, acc = torch.empty(n, C, device=dev), torch.randn(n, C, device=dev)
        variants = {
            "fwd_unfused": lambda: spmm(g, x, None, pre, post_s, out=out).add_(z, alpha=alpha),
            "fwd_fused": lambda: appnp_prop(g, x, None, pre, post, 1 - alpha, alpha, out=out, tele=z),
            "bwd_unfused": lambda: (spmm(g, x, None, pre, post_s, out=out), acc.add_(x, alpha=alpha)),
            "bwd_fused": lambda: appnp_prop(g, x, None, pre, post, 1 - alpha, alpha, out=out, acc=acc,
                                            acc_mode=ACC_ON | ACC_READ),
        }
        times = {name: [] for name in variants}
        for name in variants:                            # warm-up of every shape
            for _ in range(3):
                variants[name]()
        for _ in range(reps):                            # alternated: one launch of every variant per round
            for name in variants:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                variants[name]()
                b.record()
                torch.cuda.synchronize()
                times[name].append(a.elapsed_time(b))
        no_reuse = 4 * C * nnz + 8 * (n + 1) + 4 * nnz
        for name, ts in times.items():
            res.append({"kernel": name, "C": C, "rows": n, "nnz": nnz,
                        "median_ms": float(np.median(ts)), "min_ms": float(np.min(ts)), "reps": reps,
                        "no_reuse_GBps": no_reuse / float(np.median(ts)) / 1e6})
        for d in ("fwd", "bwd"):
            f, u = float(np.median(times[f"{d}_fused"])), float(np.median(times[f"{d}_unfused"]))
            res.append({"compare": d, "C": C, "fused_ms": f, "unfused_ms": u, "speedup": u / f})
    return res


def _wire_bytes(C, keys):
    """Bytes this rank sends per training epoch over the quantisable keys (fp32 rows, or the assigned bits)."""
    from adaqp_b200.assigner import Assigner as assigner
    from adaqp_b200.communicator.p2p import qsize
    from adaqp_b200.helper import BitType
    from adaqp_b200.manager import GraphEngine as engine
    eng = engine.ctx
    if eng.bit_type == BitType.FULL:
        rows = sum(hi - lo for lo, hi in eng.send_idx.values())
        return len(keys) * rows * C * 4
    total = 0
    for key in keys:
        for bits in assigner.ctx.assignment[key].values():
            bits = torch.as_tensor(bits)
            for b in (2, 4, 8):
                nb = int((bits == b).sum())
                total += qsize(nb, b, C) + 4 * nb if nb else 0
    return total


def _train_worker(rank, world, port, tmp, mode, scale, epochs, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": "0", "ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": str(scale), "ADAQP_SEED": "1"})
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    tr = Trainer(Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                           model_name="appnp", mode=mode, assign_scheme="uniform", logger_level="WARNING",
                           num_epoches=epochs, exp_path=f"{tmp}/exp"))
    C = tr.config["data"]["num_classes"]
    keys = [k for k in tr.key_dims if k.startswith(("forward", "backward"))]
    wire = _wire_bytes(C, keys)
    rec = tr.train()
    out.put((rank, (float(rec[2]), float(np.mean(tr.exposed_comm_ms)), wire)))


def epochs_per_second(mode, world, scale, epochs):
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _port()
    with tempfile.TemporaryDirectory() as tmp:
        procs = [ctx.Process(target=_train_worker, args=(r, world, port, tmp, mode, scale, epochs, out))
                 for r in range(world)]
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=3600)
        if any(p.exitcode != 0 for p in procs):
            return {"model": "appnp", "mode": mode, "world": world, "error": [p.exitcode for p in procs]}
        vals = dict(out.get(timeout=5) for _ in procs)
    t = max(v[0] for v in vals.values())
    return {"model": "appnp", "k": 10, "alpha": 0.1, "mode": mode, "world": world, "scale": scale, "epochs": epochs,
            "mean_epoch_s": t, "epochs_per_s": 1.0 / t,
            "exposed_comm_ms_per_epoch": {r: v[1] for r, v in sorted(vals.items())},
            "wire_bytes_per_epoch": {r: v[2] for r, v in sorted(vals.items())}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kernel-scale", type=float, default=1.0)
    ap.add_argument("--widths", type=str, default="41,47,100,107")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--scale", type=float, default=0.1)
    ap.add_argument("--epochs", type=int, default=6)
    ap.add_argument("--skip-train", action="store_true")
    ap.add_argument("--skip-kernels", action="store_true")
    a = ap.parse_args()
    print(json.dumps(_card()), flush=True)
    if not a.skip_kernels:
        for r in kernel_times(a.kernel_scale, [int(w) for w in a.widths.split(",")], a.reps):
            print(json.dumps(r), flush=True)
    if not a.skip_train:
        for world in (1, 2):
            for mode in ("Vanilla", "AdaQP"):
                print(json.dumps(epochs_per_second(mode, world, a.scale, a.epochs)), flush=True)
    print(json.dumps(_card()), flush=True)


if __name__ == "__main__":
    main()

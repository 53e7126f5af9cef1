"""GraphSAGE max-pool measurements on an ogbn-products-shaped synthetic graph; prints one JSON line per result.

    python tools/bench_pool.py [--scale 0.1] [--epochs 6] [--reps 10] [--skip-train]

* event-timed sage_pool_fwd and sage_pool_bwd over all inner rows of the one-rank partition at F = 256 (median of
  --reps launches after 3 warm-up launches), with algorithmic bytes from the shapes against two bounds: compulsory
  (every array once: CSR, p / gm and arg rows, want, outputs) and no-reuse (every neighbour row gathered from HBM:
  4 F nnz forward; 4 F nnz of arg rows + the 4-byte gradient columns that match backward);
* epochs/s of SAGE-mean and SAGE-pool (Vanilla and AdaQP, uniform 8-bit) at one rank and at two ranks sharing cuda:0
  (Trainer.train's mean epoch time over --epochs epochs, the first included);
* the exchanged bytes per training step of pool's extra keys: fp32 pool_arg rows against the 8-bit backward rows
  they travel with;
* the card name and power limit, read in the same run (a time means nothing without them).
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
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"card": torch.cuda.get_device_name(0), "nvidia_smi": r.stdout.strip()}


def _port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _train_worker(rank, world, port, tmp, agg, mode, scale, epochs, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": "0", "ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": str(scale), "ADAQP_SEED": "1"})
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    from adaqp_b200.manager import GraphEngine as engine
    tr = Trainer(Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                           model_name="sage", mode=mode, assign_scheme="uniform", logger_level="WARNING",
                           num_epoches=epochs, exp_path=f"{tmp}/exp", aggregator_type=agg, assign_bits=8))
    rec = tr.train()
    rows = int(engine.ctx.total_send_idx.numel())
    out.put((rank, (float(rec[2]), rows)))


def epochs_per_second(agg, mode, world, scale, epochs):
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _port()
    with tempfile.TemporaryDirectory() as tmp:
        procs = [ctx.Process(target=_train_worker, args=(r, world, port, tmp, agg, mode, scale, epochs, out))
                 for r in range(world)]
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=3600)
        if any(p.exitcode != 0 for p in procs):
            return {"aggregator": agg, "mode": mode, "world": world, "error": [p.exitcode for p in procs]}
        got = [v for _, v in (out.get(timeout=5) for _ in procs)]
    t = max(v[0] for v in got)
    res = {"model": "sage", "aggregator": agg, "mode": mode, "world": world, "scale": scale, "epochs": epochs,
           "mean_epoch_s": t, "epochs_per_s": 1.0 / t}
    if world > 1 and agg == "pool":
        cfg = yaml.safe_load(open(os.path.join(ROOT, "adaqp_b200", "config", "ogbn-products.yaml")))
        dims = [cfg["data"]["num_feats"]] + [cfg["model"]["hidden_dim"]] * (cfg["model"]["num_layers"] - 1)
        S = sum(v[1] for v in got)                     # boundary rows sent per key, all ranks
        res["pool_arg_bytes_per_step"] = int(4 * S * sum(dims))                    # fp32 in every mode
        # backward rows: 1 byte per element at 8 bits plus two bf16 parameters per row, or 4 bytes per element in fp32
        res["backward_bytes_per_step"] = int(S * sum(dims) + 4 * S * len(dims)) if mode == "AdaQP" else int(4 * S * sum(dims))
    return res


def kernel_times(scale, reps, F=256):
    from adaqp_b200 import build, sage_pool
    build.build()
    from adaqp_b200.manager.graph import LocalGraph
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import spec_from_config
    cfg = yaml.safe_load(open(os.path.join(ROOT, "adaqp_b200", "config", "ogbn-products.yaml")))
    L = prepare_all_in_process(spec_from_config(cfg, 1, scale))[0]
    dev = torch.device("cuda:0")
    g = LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, dev)
    n, nnz = L.n_inner, int(L.indptr[-1])
    p = torch.relu(torch.randn(n, F, device=dev))
    m, arg = sage_pool.forward(g, p, None)
    grad = torch.randn(n, F, device=dev)
    want = (torch.repeat_interleave(torch.arange(n, device=dev), torch.diff(g.indptr)) - n).to(torch.int32)
    dp = sage_pool.backward(g, want, grad, None, arg, None)
    # columns routed: every destination column has exactly one arg, so the matches total n F
    routed = n * F

    def timed(fn):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return float(np.median(ts))

    res = []
    csr = 8 * (n + 1) + 4 * nnz
    ms = timed(lambda: sage_pool.forward(g, p, None, out=m, arg=arg))
    comp = csr + 4 * F * n * 3                                       # p; m, arg
    res.append({"kernel": "sage_pool_fwd", "rows": n, "nnz": nnz, "F": F, "ms": ms,
                "compulsory_GBps": comp / ms / 1e6, "no_reuse_GBps": (4 * F * nnz + csr + 8 * F * n) / ms / 1e6})
    ms = timed(lambda: sage_pool.backward(g, want, grad, None, arg, None, dp=dp))
    comp = csr + 4 * nnz + 4 * F * n * 3                             # want; gm, arg, dp
    no_reuse = csr + 4 * nnz + 4 * F * nnz + 4 * routed + 4 * F * n    # arg row of every neighbour, matched gm columns
    res.append({"kernel": "sage_pool_bwd", "rows": n, "nnz": nnz, "F": F, "ms": ms,
                "compulsory_GBps": comp / ms / 1e6, "no_reuse_GBps": no_reuse / ms / 1e6})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=0.1)
    ap.add_argument("--kernel-scale", type=float, default=1.0)
    ap.add_argument("--epochs", type=int, default=6)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--skip-train", action="store_true")
    a = ap.parse_args()
    print(json.dumps(_card()), flush=True)
    for r in kernel_times(a.kernel_scale, a.reps):
        print(json.dumps(r), flush=True)
    if not a.skip_train:
        for world in (1, 2):
            for agg in ("mean", "pool"):
                for mode in ("Vanilla", "AdaQP"):
                    print(json.dumps(epochs_per_second(agg, mode, world, a.scale, a.epochs)), flush=True)
    print(json.dumps(_card()), flush=True)


if __name__ == "__main__":
    main()

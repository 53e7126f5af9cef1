"""GAT measurements on an ogbn-products-shaped synthetic graph; prints one JSON line per result.

    python tools/bench_gat.py [--scale 0.25] [--epochs 6] [--reps 10] [--skip-train]

* epochs/s of GCN and GAT (Vanilla and AdaQP, uniform 8-bit) at one rank and at two ranks sharing cuda:0
  (Trainer.train's mean epoch time over --epochs epochs, the first included);
* event-timed gat_fwd and gat_bwd over all inner rows of the one-rank partition (H = 4 heads of 64, F = 256), with
  algorithmic bytes from the shapes against two bounds: compulsory (every array once: z / g rows, CSR, per-row
  scalars, output) and no-reuse (every neighbour row gathered from HBM: 4 F nnz forward, 8 F nnz backward);
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


def _train_worker(rank, world, port, tmp, model, mode, scale, epochs, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": "0", "ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": str(scale), "ADAQP_SEED": "1"})
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    tr = Trainer(Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                           model_name=model, mode=mode, assign_scheme="uniform", logger_level="WARNING",
                           num_epoches=epochs, exp_path=f"{tmp}/exp"))
    rec = tr.train()
    out.put((rank, float(rec[2])))


def epochs_per_second(model, mode, world, scale, epochs):
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _port()
    with tempfile.TemporaryDirectory() as tmp:
        procs = [ctx.Process(target=_train_worker, args=(r, world, port, tmp, model, mode, scale, epochs, out))
                 for r in range(world)]
        for p in procs:
            p.start()
        for p in procs:
            p.join(timeout=3600)
        if any(p.exitcode != 0 for p in procs):
            return {"model": model, "mode": mode, "world": world, "error": [p.exitcode for p in procs]}
        t = max(v for _, v in (out.get(timeout=5) for _ in procs))
    return {"model": model, "mode": mode, "world": world, "scale": scale, "epochs": epochs, "mean_epoch_s": t,
            "epochs_per_s": 1.0 / t}


def kernel_times(scale, reps, H=4, D=64):
    from adaqp_b200 import build, gat
    build.build()
    from adaqp_b200.manager.graph import LocalGraph
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import spec_from_config
    cfg = yaml.safe_load(open(os.path.join(ROOT, "adaqp_b200", "config", "ogbn-products.yaml")))
    L = prepare_all_in_process(spec_from_config(cfg, 1, scale))[0]
    dev = torch.device("cuda:0")
    g = LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, dev)
    n, F, nnz = L.n_inner, H * D, int(L.indptr[-1])
    z = torch.randn(n, F, device=dev)
    a_l, a_r = torch.randn(H, D, device=dev) * 0.1, torch.randn(H, D, device=dev) * 0.1
    el, er = gat.scores(z, a_l, a_r, H)
    out, lse = gat.forward(g, z, None, el, None, er, H)
    grad = torch.randn(n, F, device=dev)
    s = (grad.view(n, H, D) * out.view(n, H, D)).sum(-1)
    aux = torch.cat([er, lse, s], 1).contiguous()

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
    ms = timed(lambda: gat.forward(g, z, None, el, None, er, H, out=out, lse=lse))
    comp = csr + 4 * F * n * 2 + 4 * H * n * 3                       # z, out; el, er, lse
    res.append({"kernel": "gat_fwd", "rows": n, "nnz": nnz, "F": F, "H": H, "ms": ms,
                "compulsory_GBps": comp / ms / 1e6, "no_reuse_GBps": (4 * F * nnz + csr) / ms / 1e6})
    ms = timed(lambda: gat.backward(g, grad, None, z, None, el, None, aux, None, a_l, a_r, H))
    comp = csr + 4 * F * n * 3 + 4 * H * n * 6                       # g, z, dz; el, er, lse, s, del, der
    res.append({"kernel": "gat_bwd", "rows": n, "nnz": nnz, "F": F, "H": H, "ms": ms,
                "compulsory_GBps": comp / ms / 1e6, "no_reuse_GBps": (8 * F * nnz + csr) / ms / 1e6})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=0.25)
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
            for model in ("gcn", "gat"):
                for mode in ("Vanilla", "AdaQP"):
                    print(json.dumps(epochs_per_second(model, mode, world, a.scale, a.epochs)), flush=True)
    print(json.dumps(_card()), flush=True)


if __name__ == "__main__":
    main()

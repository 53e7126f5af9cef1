"""GATv2 measurements on an ogbn-products-shaped synthetic graph; prints one JSON line per result.

    python tools/bench_gatv2.py [--kernel-scale 1.0] [--scale 0.25] [--epochs 6] [--reps 10] [--skip-train]

* event-timed gatv2_fwd and gatv2_bwd_inner over all inner rows of the one-rank partition, next to gat_fwd and
  gat_bwd at the same F and H (H = 4 heads of 64, F = 256): the price of the per-edge head reduction against GAT's
  per-row scalar logits;
* event-timed gatv2_bwd_halo over the halo rows of rank 0 of a two-rank partition at --scale;
* epochs/s of GAT and GATv2 (Vanilla and AdaQP, uniform 8-bit) at two ranks sharing cuda:0 (Trainer.train's mean
  epoch time over --epochs epochs, the first included), with the wire bytes per rank per training step and per
  evaluation pass, computed from the exchange tables (GATv2's push rows travel in fp32 in every mode);
* the card name, power limit and SM clocks, read in the same run (a time means nothing without them).
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
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"card": torch.cuda.get_device_name(0), "nvidia_smi": r.stdout.strip()}


def _port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def wire_bytes(ex, quant: bool, bits: int = 8):
    """Bytes this rank puts on the wire per training step and per evaluation pass: fp32 keys send 4 F bytes a row,
    quantised keys (training forward / backward rows in AdaQP) the packed rows plus two bf16 parameters a row."""
    from adaqp_b200.communicator.p2p import is_push, qsize, quantisable
    sent = sum(hi - lo for lo, hi in ex.send_idx.values())
    pushed = sum(v.size for v in ex.recv_idx.values())
    train = evalb = 0
    for key, F in ex.dims.items():
        if key.startswith("test"):
            evalb += 4 * F * sent
        elif is_push(key):
            train += 4 * F * pushed
        elif quant and quantisable(key):
            train += sum(qsize(hi - lo, bits, F) + 4 * (hi - lo) for lo, hi in ex.send_idx.values())
        else:
            train += 4 * F * sent
            if key.startswith("attn_fwd"):
                evalb += 4 * F * sent
    return train, evalb


def _train_worker(rank, world, port, tmp, model, mode, scale, epochs, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": "0", "ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": str(scale), "ADAQP_SEED": "1"})
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    from adaqp_b200.communicator import Communicator as comm
    tr = Trainer(Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                           model_name=model, mode=mode, assign_scheme="uniform", logger_level="WARNING",
                           num_epoches=epochs, exp_path=f"{tmp}/exp"))
    train_b, eval_b = wire_bytes(comm.ctx.comm_buffer.p2p, mode in ("AdaQP", "AdaQP-q"))
    torch.cuda.reset_peak_memory_stats()
    rec = tr.train()
    out.put((rank, (float(rec[2]), float(rec[3]), train_b, eval_b, torch.cuda.max_memory_allocated())))


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
        res = dict(out.get(timeout=5) for _ in procs)
    t = max(v[0] for v in res.values())
    return {"model": model, "mode": mode, "world": world, "scale": scale, "epochs": epochs, "mean_epoch_s": t,
            "epochs_per_s": 1.0 / t, "comm_s_per_epoch": [res[r][1] for r in sorted(res)],
            "train_wire_bytes_per_rank": [res[r][2] for r in sorted(res)],
            "eval_wire_bytes_per_rank": [res[r][3] for r in sorted(res)],
            "peak_mem_bytes": [res[r][4] for r in sorted(res)]}


def _timed(fn, reps):
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


def kernel_times(kernel_scale, halo_scale, reps, H=4, D=64):
    from adaqp_b200 import build, gat, gatv2
    build.build()
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.graph import LocalGraph
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import spec_from_config
    cfg = yaml.safe_load(open(os.path.join(ROOT, "adaqp_b200", "config", "ogbn-products.yaml")))
    L = prepare_all_in_process(spec_from_config(cfg, 1, kernel_scale))[0]
    dev = torch.device("cuda:0")
    g = LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, dev)
    n, F, nnz = L.n_inner, H * D, int(L.indptr[-1])
    gen = torch.Generator(device=dev).manual_seed(0)
    z = torch.randn(n, F, device=dev, generator=gen)
    zd = torch.randn(n, F, device=dev, generator=gen)
    grad = torch.randn(n, F, device=dev, generator=gen)
    a_l, a_r = torch.randn(H, D, device=dev, generator=gen) * 0.1, torch.randn(H, D, device=dev, generator=gen) * 0.1
    el, er = gat.scores(z, a_l, a_r, H)
    out, lse = gat.forward(g, z, None, el, None, er, H)
    s = (grad.view(n, H, D) * out.view(n, H, D)).sum(-1)
    aux = torch.cat([er, lse, s], 1).contiguous()
    out2, lse2 = gatv2.forward(g, z, None, zd, a_l, H)
    S2 = (grad.view(n, H, D) * out2.view(n, H, D)).sum(-1).contiguous()
    res = []
    base = {"rows": n, "nnz": nnz, "F": F, "H": H, "scale": kernel_scale}
    res.append({"kernel": "gat_fwd", **base, "ms": _timed(lambda: gat.forward(g, z, None, el, None, er, H, out=out,
                                                                               lse=lse), reps)})
    res.append({"kernel": "gatv2_fwd", **base, "ms": _timed(lambda: gatv2.forward(g, z, None, zd, a_l, H, out=out2,
                                                                                   lse=lse2), reps)})
    res.append({"kernel": "gat_bwd", **base,
                "ms": _timed(lambda: gat.backward(g, grad, None, z, None, el, None, aux, None, a_l, a_r, H), reps)})
    res.append({"kernel": "gatv2_bwd_inner", **base,
                "ms": _timed(lambda: gatv2.backward_inner(g, z, None, zd, grad, lse2, S2, a_l, H), reps)})
    del z, zd, grad, out, out2, aux
    torch.cuda.empty_cache()
    # halo rows exist only with more than one part
    L = prepare_all_in_process(spec_from_config(cfg, 2, halo_scale), DistGNNType.DistGATv2)[0]
    n, nh = L.n_inner, L.n_halo
    hp, hd = gatv2.halo_table(L.indptr, L.indices, n, nh)
    hp, hd = torch.from_numpy(hp).to(dev), torch.from_numpy(hd).to(dev)
    zh = torch.randn(nh, F, device=dev, generator=gen)
    zd = torch.randn(n, F, device=dev, generator=gen)
    grad = torch.randn(n, F, device=dev, generator=gen)
    lse = torch.randn(n, H, device=dev, generator=gen).abs() + 2.0
    S = torch.randn(n, H, device=dev, generator=gen)
    res.append({"kernel": "gatv2_bwd_halo", "rows": nh, "edges": int(hp[-1]), "F": F, "H": H, "scale": halo_scale,
                "ms": _timed(lambda: gatv2.backward_halo(hp, hd, zh, zd, grad, lse, S, a_l, H), reps)})
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
    for r in kernel_times(a.kernel_scale, a.scale, a.reps):
        print(json.dumps(r), flush=True)
    if not a.skip_train:
        for model in ("gat", "gatv2"):
            for mode in ("Vanilla", "AdaQP"):
                print(json.dumps(epochs_per_second(model, mode, 2, a.scale, a.epochs)), flush=True)
    print(json.dumps(_card()), flush=True)


if __name__ == "__main__":
    main()

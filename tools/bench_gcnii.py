"""GCNII measurements on an ogbn-products-shaped synthetic graph; prints one JSON line per result.

    python tools/bench_gcnii.py [--kernel-scale 1.0] [--widths 256] [--reps 10] [--scale 0.1] [--epochs 6] [--full]

* the hidden-width propagation step three ways, alternated, median of --reps event-timed launches over all rows of the
  one-rank partition: the column-sliced kernel (appnp_prop_sliced_kernel, the default at F = 256), the forced-unsliced
  appnp_prop_kernel (option spmm_slice_cols = F), and the CSR SpMM (post scaled by 1 - alpha) followed by the
  elementwise ops it replaces (a torch add of alpha h0 forward; a torch mul into dh0 backward); forward (teleport) and
  backward (accumulate), with a bitwise check of sliced against unsliced;
* epochs/s of GCNII (L = 8, H = 256, alpha = 0.1, theta = 0.5) in Vanilla and AdaQP (uniform 8-bit) at one rank and at
  two ranks sharing cuda:0 (Trainer.train's mean epoch time, first epoch included), the exposed communication per
  epoch, the bytes each rank puts on the wire per training epoch (quantised and as fp32) and each rank's peak
  allocated memory; with --full also one rank at the full shape;
* the card name, power limit and max SM clock, read in the same run.
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np
import torch
import torch.multiprocessing as mp
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.bench_appnp import _card, _port  # noqa: E402


def kernel_times(scale, widths, reps, alpha=0.1):
    from adaqp_b200 import _lib, build
    build.build()
    from adaqp_b200.manager.graph import ACC_ON, LocalGraph, appnp_prop, spmm
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import spec_from_config
    cfg = yaml.safe_load(open(os.path.join(ROOT, "adaqp_b200", "config", "ogbn-products.yaml")))
    L = prepare_all_in_process(spec_from_config(cfg, 1, scale))[0]
    dev = torch.device("cuda:0")
    g = LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, dev)
    n, nnz = L.n_inner, int(L.indptr[-1])
    fpre, fpost = g.norm["out_-0.5"], g.norm["in_-0.5"]
    bpre, bpost = g.norm["in_-0.5"], g.norm["out_-0.5"]
    fpost_s, bpost_s = fpost * (1 - alpha), bpost * (1 - alpha)
    old = _lib.get_option("spmm_slice_cols")
    res = []
    for F in widths:
        x, z = torch.randn(n, F, device=dev), torch.randn(n, F, device=dev)
        outs = {k: torch.empty(n, F, device=dev) for k in ("sliced", "unsliced", "spmm")}
        accs = {k: torch.empty(n, F, device=dev) for k in ("sliced", "unsliced", "spmm")}

        def prop(kind, fwd, forced):
            _lib.set_option("spmm_slice_cols", forced)
            if fwd:
                appnp_prop(g, x, None, fpre, fpost, 1 - alpha, alpha, out=outs[kind], tele=z)
            else:
                appnp_prop(g, x, None, bpre, bpost, 1 - alpha, alpha, out=outs[kind], acc=accs[kind], acc_mode=ACC_ON)

        def composed(fwd):
            _lib.set_option("spmm_slice_cols", old)
            if fwd:
                spmm(g, x, None, fpre, fpost_s, out=outs["spmm"]).add_(z, alpha=alpha)
            else:
                spmm(g, x, None, bpre, bpost_s, out=outs["spmm"])
                torch.mul(x, alpha, out=accs["spmm"])

        for d, fwd in (("fwd", True), ("bwd", False)):
            variants = {f"{d}_sliced": lambda fwd=fwd: prop("sliced", fwd, old),
                        f"{d}_unsliced": lambda fwd=fwd: prop("unsliced", fwd, F),
                        f"{d}_spmm_elementwise": lambda fwd=fwd: composed(fwd)}
            times = {name: [] for name in variants}
            for name in variants:                        # warm-up of every shape
                for _ in range(3):
                    variants[name]()
            for _ in range(reps):                        # alternated: one launch of every variant per round
                for name in variants:
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    variants[name]()
                    b.record()
                    torch.cuda.synchronize()
                    times[name].append(a.elapsed_time(b))
            _lib.set_option("spmm_slice_cols", old)
            bitwise = torch.equal(outs["sliced"], outs["unsliced"]) and (fwd or torch.equal(accs["sliced"], accs["unsliced"]))
            no_reuse = 4 * F * nnz + 8 * (n + 1) + 4 * nnz
            for name, ts in times.items():
                res.append({"kernel": name, "F": F, "rows": n, "nnz": nnz, "median_ms": float(np.median(ts)),
                            "min_ms": float(np.min(ts)), "reps": reps, "no_reuse_GBps": no_reuse / float(np.median(ts)) / 1e6})
            s, u, c = (float(np.median(times[f"{d}_{k}"])) for k in ("sliced", "unsliced", "spmm_elementwise"))
            res.append({"compare": d, "F": F, "sliced_ms": s, "unsliced_ms": u, "spmm_elementwise_ms": c,
                        "sliced_vs_unsliced": u / s, "sliced_vs_spmm_elementwise": c / s,
                        "bitwise_equal_sliced_unsliced": bool(bitwise)})
    return res


def _wire_bytes(H, keys):
    """Bytes this rank sends per training epoch over the quantisable keys: (as sent, as fp32 rows)."""
    from adaqp_b200.assigner import Assigner as assigner
    from adaqp_b200.communicator.p2p import qsize
    from adaqp_b200.helper import BitType
    from adaqp_b200.manager import GraphEngine as engine
    eng = engine.ctx
    rows = sum(hi - lo for lo, hi in eng.send_idx.values())
    fp32 = len(keys) * rows * H * 4
    if eng.bit_type == BitType.FULL:
        return fp32, fp32
    total = 0
    for key in keys:
        for bits in assigner.ctx.assignment[key].values():
            bits = torch.as_tensor(bits)
            for b in (2, 4, 8):
                nb = int((bits == b).sum())
                total += qsize(nb, b, H) + 4 * nb if nb else 0
    return total, fp32


def _train_worker(rank, world, port, tmp, mode, scale, epochs, out):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world),
                       "LOCAL_RANK": "0", "ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": str(scale), "ADAQP_SEED": "1"})
    os.chdir(tmp)
    from argparse import Namespace
    from adaqp_b200 import Trainer
    try:
        tr = Trainer(Namespace(dataset="ogbn-products", num_parts=world, backend="gloo", init_method="env://",
                               model_name="gcnii", mode=mode, assign_scheme="uniform", logger_level="WARNING",
                               num_epoches=epochs, exp_path=f"{tmp}/exp"))
        H = tr.config["model"]["hidden_dim"]
        keys = [k for k in tr.key_dims if k.startswith(("forward", "backward"))]
        wire = _wire_bytes(H, keys)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        rec = tr.train()
        peak = torch.cuda.max_memory_allocated()
        out.put((rank, (float(rec[2]), float(np.mean(tr.exposed_comm_ms)), wire, peak)))
    except torch.cuda.OutOfMemoryError as e:
        out.put((rank, ("oom", str(e)[:300])))


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
            return {"model": "gcnii", "mode": mode, "world": world, "scale": scale, "error": [p.exitcode for p in procs]}
        vals = dict(out.get(timeout=5) for _ in procs)
    if any(v[0] == "oom" for v in vals.values()):
        return {"model": "gcnii", "mode": mode, "world": world, "scale": scale, "oom": {r: v[1] for r, v in vals.items()}}
    t = max(v[0] for v in vals.values())
    return {"model": "gcnii", "layers": 8, "hidden": 256, "alpha": 0.1, "theta": 0.5, "mode": mode, "world": world,
            "scale": scale, "epochs": epochs, "mean_epoch_s": t, "epochs_per_s": 1.0 / t,
            "exposed_comm_ms_per_epoch": {r: v[1] for r, v in sorted(vals.items())},
            "wire_bytes_per_epoch": {r: v[2][0] for r, v in sorted(vals.items())},
            "wire_bytes_per_epoch_fp32": {r: v[2][1] for r, v in sorted(vals.items())},
            "peak_allocated_GB": {r: v[3] / 1e9 for r, v in sorted(vals.items())}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kernel-scale", type=float, default=1.0)
    ap.add_argument("--widths", type=str, default="256")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--scale", type=float, default=0.1)
    ap.add_argument("--epochs", type=int, default=6)
    ap.add_argument("--full", action="store_true", help="also one rank at the full shape (Vanilla, 2 epochs)")
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
    if a.full:
        print(json.dumps(epochs_per_second("Vanilla", 1, 1.0, 2)), flush=True)
    print(json.dumps(_card()), flush=True)


if __name__ == "__main__":
    main()

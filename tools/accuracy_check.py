"""Validation accuracy of the quantised exchange vs fp32 (north star: within 0.3 % of Vanilla) on a task
that is hard enough to discriminate.

The synthetic ogbn-products-shaped task (labels = community class, features = class centroid * signal +
unit noise, 60 % homophilous edges) is first CALIBRATED: `--calibrate s1,s2,...` trains Vanilla for each
feature-signal strength and keeps the one whose best validation accuracy is closest to `--target` (default
0.80, i.e. far from the label-noise ceiling where every method scores the same).  Then every mode is trained
from the same seeds: Vanilla (fp32), uniform 8 / 4 / 2 bits (2 bits is the CONTROL that should degrade),
random {2,4,8} and adaptive, `--seeds` times each; the report is best-validation accuracy per run and the
mean / min / max of the difference to Vanilla of the same seed.

    python tools/accuracy_check.py --spawn 8 --scale 0.05 --epochs 80 --json accuracy_gcn_w8.json
    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 tools/accuracy_check.py ...      (one GPU per rank)
`--spawn W` self-launches W ranks, rank r on cuda:(r % #GPUs): accuracy does not depend on how many physical
GPUs carry the 8 partitions, so the experiment runs on one H100."""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODES = [("Vanilla", "uniform", None), ("AdaQP", "uniform", 8), ("AdaQP", "uniform", 4), ("AdaQP", "uniform", 2),
         ("AdaQP", "random", None), ("AdaQP", "adaptive", None)]


def run(mode, scheme, bits, seed, args, world):
    from argparse import Namespace
    from adaqp_b200 import Trainer
    from adaqp_b200.manager import GraphEngine as engine
    os.environ["ADAQP_SEED"] = str(seed)
    t = Trainer(Namespace(dataset=args.dataset, num_parts=world, backend="gloo", init_method="env://",
                          model_name=args.model_name, mode=mode, assign_scheme=scheme, logger_level="WARNING",
                          num_epoches=args.epochs, exp_path="/tmp/adaqp_acc_exp", assign_bits=bits,
                          aggregator_type=args.aggregator_type, appnp_k=args.appnp_k, appnp_alpha=args.appnp_alpha,
                          gcnii_layers=args.gcnii_layers, gcnii_alpha=args.gcnii_alpha, gcnii_theta=args.gcnii_theta))
    if scheme == "adaptive":
        t.assigner.assign_cycle = args.assign_cycle
    t.train()
    m = engine.ctx.recorder.epoches_metrics[:args.epochs]
    best = int(m[:, 1].argmax())
    name = mode if mode == "Vanilla" else f"{scheme}{bits if scheme == 'uniform' else ''}"
    return {"name": name, "seed": seed, "best_val": float(m[best, 1]), "test_at_best": float(m[best, 2]),
            "final_val": float(m[-1, 1]), "final_train": float(m[-1, 0])}


def worker(args):
    import numpy as np
    os.environ["ADAQP_SYNTH_SCALE"] = str(args.scale)
    os.environ.setdefault("ADAQP_SYNTHETIC", "1")
    os.environ["ADAQP_SYNTH_LABEL_NOISE"] = str(args.label_noise)
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    import __graft_entry__ as entry
    if rank == 0:
        entry.build()
    signal = args.signal
    calib = []
    if args.calibrate:
        for s in [float(x) for x in args.calibrate.split(",")]:
            os.environ["ADAQP_SYNTH_SIGNAL"] = str(s)
            r = run("Vanilla", "uniform", None, args.seed0, args, world)
            calib.append({"feature_signal": s, "vanilla_best_val": r["best_val"]})
            if rank == 0:
                print(json.dumps(calib[-1]), flush=True)
        signal = min(calib, key=lambda c: abs(c["vanilla_best_val"] - args.target))["feature_signal"]
    os.environ["ADAQP_SYNTH_SIGNAL"] = str(signal)
    runs = []
    for k in range(args.seeds):
        for mode, scheme, bits in MODES:
            runs.append(run(mode, scheme, bits, args.seed0 + k, args, world))
            if rank == 0:
                print(json.dumps(runs[-1]), flush=True)
    if rank == 0:
        base = {r["seed"]: r["best_val"] for r in runs if r["name"] == "Vanilla"}
        delta = {}
        for r in runs:
            if r["name"] != "Vanilla":
                delta.setdefault(r["name"], []).append(100 * (r["best_val"] - base[r["seed"]]))
        summary = {"world": world, "epochs": args.epochs, "scale": args.scale, "model": args.model_name,
                   "aggregator_type": args.aggregator_type, "appnp_k": args.appnp_k, "appnp_alpha": args.appnp_alpha,
                   "gcnii_layers": args.gcnii_layers, "gcnii_alpha": args.gcnii_alpha, "gcnii_theta": args.gcnii_theta,
                   "dataset": args.dataset,
                   "feature_signal": signal, "label_noise": args.label_noise, "calibration": calib, "runs": runs,
                   "vanilla_best_val_mean": float(np.mean(list(base.values()))),
                   "delta_best_val_vs_vanilla_pp": {k: {"mean": float(np.mean(v)), "min": float(np.min(v)), "max": float(np.max(v)), "n": len(v)}
                                                    for k, v in delta.items()}}
        print(json.dumps(summary), flush=True)
        if args.json:
            os.makedirs(os.path.dirname(args.json) or ".", exist_ok=True)
            with open(args.json, "w") as f:
                json.dump(summary, f, indent=1)


def _spawn_entry(r, args, port, ngpu):
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(r),
                       "WORLD_SIZE": str(args.spawn), "LOCAL_RANK": str(r % ngpu)})
    worker(args)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=80)
    ap.add_argument("--scale", type=float, default=0.05)
    ap.add_argument("--dataset", type=str, default="ogbn-products")
    ap.add_argument("--model_name", type=str, default="gcn")
    ap.add_argument("--aggregator_type", type=str, default=None, help="GraphSAGE aggregator (default: the config's)")
    ap.add_argument("--appnp_k", type=int, default=None, help="APPNP propagation steps (default: the config's)")
    ap.add_argument("--appnp_alpha", type=float, default=None, help="APPNP teleport probability (default: the config's)")
    ap.add_argument("--gcnii_layers", type=int, default=None, help="GCNII layers (default: the config's)")
    ap.add_argument("--gcnii_alpha", type=float, default=None, help="GCNII initial-residual weight (default: the config's)")
    ap.add_argument("--gcnii_theta", type=float, default=None, help="GCNII identity-mapping strength (default: the config's)")
    ap.add_argument("--assign_cycle", type=int, default=20)
    ap.add_argument("--seeds", type=int, default=3)
    ap.add_argument("--seed0", type=int, default=123)
    ap.add_argument("--json", type=str, default=None)
    ap.add_argument("--feature-signal", dest="signal", type=float, default=0.05, help="class-centroid strength of the synthetic features")
    ap.add_argument("--label-noise", type=float, default=0.05)
    ap.add_argument("--calibrate", type=str, default=None, help="comma separated feature signals to try with Vanilla first")
    ap.add_argument("--target", type=float, default=0.80)
    ap.add_argument("--spawn", type=int, default=0)
    args = ap.parse_args()
    if args.spawn:
        import socket
        import torch
        import torch.multiprocessing as mp
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
        s.close()
        ngpu = max(torch.cuda.device_count(), 1)
        ctx = mp.get_context("spawn")
        procs = [ctx.Process(target=_spawn_entry, args=(r, args, port, ngpu)) for r in range(args.spawn)]
        for p in procs:
            p.start()
        for p in procs:
            p.join()
        sys.exit(max(p.exitcode or 0 for p in procs))
    worker(args)


if __name__ == "__main__":
    main()

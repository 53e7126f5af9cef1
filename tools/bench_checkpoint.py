"""Cost of one checkpoint and of one prediction on an ogbn-products-shaped synthetic graph; prints one JSON line.

    python tools/bench_checkpoint.py [--scale 1.0] [--mode AdaQP] [--assign_scheme random]

One rank on cuda:0, GCN 3x256.  The Trainer trains one epoch (keeping `best/`), then, timed on the host around work
that ends in a device synchronise:
* the partition digest (SHA-256 of the rank's CSR), computed once per run;
* one `checkpoint.save` (model + Adam state, RNG, Assigner, Recorder, manifest; rename; `latest`) and its bytes;
* one `Trainer.save_predictions` from that checkpoint in a fresh Trainer (load weights, evaluation forward, shard,
  merge into predictions.npz) and its bytes.
Everything is written under a temporary directory that is removed afterwards.  The card name and power limit are
read in the same run.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _du(path):
    return sum(os.path.getsize(os.path.join(d, f)) for d, _, fs in os.walk(path) for f in fs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--mode", default="AdaQP")
    ap.add_argument("--assign_scheme", default="random")
    a = ap.parse_args()
    os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": os.environ.get("MASTER_PORT", "29531"), "RANK": "0",
                       "WORLD_SIZE": "1", "LOCAL_RANK": "0", "ADAQP_SYNTHETIC": "1", "ADAQP_SYNTH_SCALE": str(a.scale),
                       "ADAQP_SEED": "1"})
    import torch
    import __graft_entry__ as entry
    entry.build()
    from argparse import Namespace
    from adaqp_b200 import Trainer
    from adaqp_b200.manager import GraphEngine as engine
    from adaqp_b200.trainer import checkpoint as ckpt
    tmp = tempfile.mkdtemp(prefix="adaqp_ckpt_bench_")
    try:
        os.chdir(tmp)
        args = dict(dataset="ogbn-products", num_parts=1, backend="gloo", init_method="env://", model_name="gcn",
                    mode=a.mode, assign_scheme=a.assign_scheme, logger_level="WARNING", num_epoches=1,
                    exp_path=f"{tmp}/exp", checkpoint_dir=f"{tmp}/ckpt")
        tr = Trainer(Namespace(**args))
        tr.train()
        layout = engine.ctx.layout
        t0 = time.perf_counter()
        digest = ckpt.partition_digest(layout)
        t_digest = time.perf_counter() - t0
        if torch.cuda.is_available():
            torch.cuda.synchronize()
        t0 = time.perf_counter()
        path = ckpt.save(f"{tmp}/ckpt", 1, tr.model, tr.optimizer, tr.run_fields(), digest, tr.epoch_records)
        t_save = time.perf_counter() - t0
        files = {f: os.path.getsize(os.path.join(path, f)) for f in sorted(os.listdir(path))}
        del tr
        pr = Trainer(Namespace(**args))
        if torch.cuda.is_available():
            torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = pr.save_predictions(f"{tmp}/pred", path)
        t_pred = time.perf_counter() - t0
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True).stdout.strip()
        print(json.dumps({"scale": a.scale, "n_inner": int(layout.n_inner), "nnz": int(layout.indices.size),
                          "mode": a.mode, "assign_scheme": a.assign_scheme,
                          "partition_digest_s": round(t_digest, 3), "checkpoint_save_s": round(t_save, 3),
                          "checkpoint_bytes": _du(path), "checkpoint_files": files,
                          "save_predictions_s": round(t_pred, 3), "predictions_bytes": os.path.getsize(out),
                          "card": torch.cuda.get_device_name(0), "nvidia_smi": smi}))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()

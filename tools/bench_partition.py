"""Partitioner benchmark: the products-shaped synthetic graph (config ogbn-products.yaml, full scale by default:
2.45 M nodes, ~126 M directed edges) with its node ids shuffled, partitioned at W = 2, 4, 8.

    python tools/bench_partition.py [--scale 1.0] [--parts 2 4 8] [--out result.json]

Per W it reports the time of each phase (host clock around device-synchronised work), the edge cut against the
generator's planted cut and against contiguous id blocks of the shuffled ids, the balance, and the halo rows and
wire bytes per training epoch of the resulting layout against the planted one.  Wire bytes per epoch: every halo
row crosses once per layer forward (widths F, H, H) and once per layer backward except the first (H, H); fp32
rows take 4 bytes per value, uniform 4-bit rows 0.5 byte per value plus 4 bytes of bf16 (scale, min).  The card
and its power limit are printed in the same run: a time means nothing without them.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def halo_rows(indptr, indices, part, W):
    """Rows each block receives: distinct (block, outside neighbour) pairs."""
    rows = np.repeat(np.arange(indptr.size - 1, dtype=np.int64), np.diff(indptr))
    pb, qb = part[rows], part[indices]
    cross = pb != qb
    key = np.unique(pb[cross].astype(np.int64) * (indptr.size - 1) + indices[cross])
    return np.bincount(key // (indptr.size - 1), minlength=W)


def wire_bytes(rows, F, H, layers):
    widths_fwd = [F] + [H] * (layers - 1)
    widths_bwd = [H] * (layers - 1)
    values = rows * (sum(widths_fwd) + sum(widths_bwd))
    exchanges = rows * (len(widths_fwd) + len(widths_bwd))
    return {"fp32": int(4 * values), "uniform4": int(values // 2 + 4 * exchanges)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--parts", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    import yaml
    from adaqp_b200 import partition as gp
    from adaqp_b200.manager.partition_synth import global_graph, spec_from_config
    if not torch.cuda.is_available():
        raise SystemExit("bench_partition.py measures the GPU partitioner and no CUDA device is visible")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(f"card: {card}", flush=True)
    with open(os.path.join(ROOT, "adaqp_b200", "config", "ogbn-products.yaml")) as f:
        cfg = yaml.safe_load(f)
    F, H, L = int(cfg["data"]["num_feats"]), int(cfg["model"]["hidden_dim"]), int(cfg["model"]["num_layers"])
    results = []
    for W in a.parts:
        t0 = time.perf_counter()
        spec = spec_from_config(cfg, W, a.scale)
        g, planted = global_graph(spec)
        n = g.num_nodes
        perm = np.random.default_rng(100 + W).permutation(n)
        planted_s = planted[perm]
        gs = g.permuted(perm)
        del g
        t_gen = time.perf_counter() - t0
        info = {}
        part = gp.partition(gs.indptr, gs.indices, W, seed=a.seed, info=info)
        m = (gs.indices.size - n) // 2
        cut = gp.edge_cut(gs.indptr, gs.indices, part)
        cut_planted = gp.edge_cut(gs.indptr, gs.indices, planted_s)
        cut_contig = gp.edge_cut(gs.indptr, gs.indices, (np.arange(n) * W // n).astype(np.int32))
        sizes = np.bincount(part, minlength=W)
        halo = halo_rows(gs.indptr, gs.indices, part, W)
        halo_p = halo_rows(gs.indptr, gs.indices, planted_s, W)
        r = {"W": W, "N": n, "undirected_edges": int(m), "card": card, "levels": info["levels"],
             "times_s": {k: round(v, 4) for k, v in info["times"].items()},
             "partition_total_s": round(sum(info["times"].values()), 4), "generate_s": round(t_gen, 1),
             "cut": cut, "cut_fraction": round(cut / m, 5), "planted_cut_fraction": round(cut_planted / m, 5),
             "cut_vs_planted": round(cut / cut_planted, 4), "contiguous_cut_fraction": round(cut_contig / m, 5),
             "max_block_over_mean": round(float(sizes.max()) * W / n, 5), "limit": gp.max_block_weight(n, W),
             "block_sizes": sizes.tolist(), "halo_rows": halo.tolist(), "halo_rows_planted": halo_p.tolist(),
             "wire_bytes_per_epoch": wire_bytes(int(halo.sum()), F, H, L),
             "wire_bytes_per_epoch_planted": wire_bytes(int(halo_p.sum()), F, H, L)}
        print(json.dumps(r), flush=True)
        results.append(r)
        del gs
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()

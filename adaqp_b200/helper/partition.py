"""Partition a dataset into the per-rank layout files Trainer reads (AdaQP/helper/partition.py).

`graph_patition_store` keeps the reference's name (typo included) and its skip-if-the-directory-exists
behaviour.  Instead of DGL + METIS it reads the raw files (helper.dataset), partitions on the GPU
(adaqp_b200.partition) and writes `<part_dir>/<dataset>/<W>part/part<rank>.npz` plus `partition_book.npz`.
"""
from __future__ import annotations

import os
import shutil
import time
from typing import Callable, Optional

import numpy as np


def graph_patition_store(dataset: str, partition_size: int, raw_dir: str = "dataset", part_dir: str = "part_data",
                         model_name: str = "gcn", seed: int = 0, log: Callable[[str], None] = print) -> Optional[dict]:
    """Returns a summary dict, or None when the partition directory already exists (nothing is done)."""
    partition_dir = f"{part_dir}/{dataset}/{partition_size}part"
    if os.path.exists(partition_dir):
        log(f"<{partition_dir} exists: nothing to do>")
        return None
    # absolute imports: the AdaQP alias loads this file as AdaQP.helper.partition too
    import torch
    from adaqp_b200 import partition as gp
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.helper.dataset import load_dataset
    from adaqp_b200.manager.graphEngine import save_rank_layout
    from adaqp_b200.manager.layout import layouts_from_raw, raw_partitions, save_partition_book

    MODELS = {"gcn": DistGNNType.DistGCN, "sage": DistGNNType.DistSAGE, "gat": DistGNNType.DistGAT,
              "gatv2": DistGNNType.DistGATv2}
    if model_name not in MODELS:
        raise ValueError(f"model_name must be one of {sorted(MODELS)}, got {model_name}")
    if not torch.cuda.is_available():
        raise RuntimeError("graph_partition.py partitions on the GPU and no CUDA device is visible")
    times = {}
    t0 = time.perf_counter()
    graph = load_dataset(dataset, raw_dir)
    times["read"] = time.perf_counter() - t0
    gp.check_k(graph.num_nodes, partition_size)
    info = {}
    part = gp.partition(graph.indptr, graph.indices, partition_size, seed=seed, info=info)
    t0 = time.perf_counter()
    model = MODELS[model_name]
    layouts = layouts_from_raw(raw_partitions(graph, part), model)
    times["layout"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    tmp_root = f"{part_dir}/.tmp-{dataset}-{partition_size}part-{os.getpid()}"
    for lay in layouts:
        save_rank_layout(lay, tmp_root, dataset)
    sizes = np.bincount(part, minlength=partition_size)
    header = {"dataset": dataset, "seed": int(seed), "k": int(partition_size), "model_name": model_name,
              "edge_cut": int(info["edge_cut"]), "block_sizes": [int(x) for x in sizes],
              "halo_rows": [int(L.n_halo) for L in layouts], "total_halo_rows": int(sum(L.n_halo for L in layouts)),
              "collapsed_multi_edges": int(graph.n_collapsed)}
    save_partition_book(part, tmp_root, dataset, header)
    os.makedirs(os.path.dirname(partition_dir), exist_ok=True)
    os.replace(f"{tmp_root}/{dataset}/{partition_size}part", partition_dir)
    shutil.rmtree(tmp_root)
    times["write"] = time.perf_counter() - t0
    n_und = (graph.indices.size - graph.num_nodes) // 2
    log(f"<{dataset}: N={graph.num_nodes} undirected edges={n_und} collapsed multi-edges={graph.n_collapsed}; "
        f"files written for model {model_name}>")
    log(f"edge cut: {info['edge_cut']} ({info['edge_cut'] / max(n_und, 1):.4f} of the edges), levels {info['levels']}")
    log(f"block sizes: {header['block_sizes']} (limit {gp.max_block_weight(graph.num_nodes, partition_size)})")
    log(f"halo rows per rank: {header['halo_rows']} (total {header['total_halo_rows']})")
    log("marginal share per rank: " + str([round(L.n_marginal / max(L.n_inner, 1), 4) for L in layouts]))
    times.update({f"partition.{k}": v for k, v in info["times"].items()})
    log("time [s]: " + ", ".join(f"{k} {v:.3f}" for k, v in times.items()))
    header["times"] = times
    return header

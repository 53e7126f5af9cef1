"""Convert dgl.distributed.partition_graph output (+ the reference's global degree files) into the
per-rank layout files this package reads (`<part_dir>/<dataset>/<W>part/part<rank>.npz`).

    python tools/convert_dgl_partition.py --part-dir data/part_data --dataset reddit --num-parts 4 --model gcn

Two layers, so that everything except the file reading is exercised by tests without DGL:

* `load_dgl_arrays` (needs DGL; runs where the partitions were made) reads one partition into a plain
  dict of numpy arrays with DGL's own shapes: local edge list (u -> v), `inner_node`, `NID` (global ids),
  `part_id`, `orig_id`, node features / labels / masks of the inner nodes, the partition book's global
  id ranges, and the global degree tensors the reference caches (helper/partition.py:67-68).
* `raw_from_arrays` + `convert` are DGL-free: they restate AdaQP/manager/conversion.py:17-54
  (convert_partition: keep the in-edges of the inner nodes, attach GLOBAL degrees through `orig_id`) and
  then run the same chain as the synthetic generator -- halo_requests -> send_side -> reorder ->
  convert_send_idx -> decompose (processing.py:40-79, conversion.py:56-172) -- and write the files.
  tests/test_converter.py feeds them a hand-built DGL-shaped fixture (shuffled edge list, edges into halo
  nodes, duplicate edges) and checks the result equals the generator's own layout field by field.
"""
from __future__ import annotations

import argparse
import os
import sys
from typing import Dict, List

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def load_dgl_arrays(part_config: str, rank: int, world: int, degree_dir: str) -> Dict[str, np.ndarray]:
    import dgl
    import torch
    g, nfeat, _, gpb, _, ntypes, _ = dgl.distributed.load_partition(part_config, rank)
    nt = ntypes[0]
    u, v = (t.numpy() for t in g.edges())
    starts = np.array([gpb.partid2nids(i)[0].item() for i in range(world)] + [gpb._num_nodes()], np.int64)
    return {"edges_u": u, "edges_v": v, "inner_node": g.ndata["inner_node"].bool().numpy(), "nid": g.ndata[dgl.NID].numpy(),
            "part_id": g.ndata["part_id"].numpy(), "orig_id": g.ndata["orig_id"].numpy(), "starts": starts,
            "feat": nfeat[nt + "/feat"].numpy(), "label": nfeat[nt + "/label"].numpy(),
            "train_mask": nfeat[nt + "/train_mask"].bool().numpy(), "val_mask": nfeat[nt + "/val_mask"].bool().numpy(),
            "test_mask": nfeat[nt + "/test_mask"].bool().numpy(),
            "in_degrees_global": torch.load(f"{degree_dir}/in_degrees.pt").numpy(),
            "out_degrees_global": torch.load(f"{degree_dir}/out_degrees.pt").numpy()}


def raw_from_arrays(a: Dict[str, np.ndarray], rank: int, world: int):
    """conversion.py:17-54 on plain arrays: inner nodes come first in a DGL partition; the hot path needs
    the dst-major CSR of the in-edges of the inner nodes (edges INTO halo nodes are dropped, multi-edges
    collapse), the halo nodes' global ids and owners, and the global degrees looked up by `orig_id`."""
    import scipy.sparse as sp
    from adaqp_b200.manager.partition_synth import RawPartition
    inner = np.asarray(a["inner_node"], bool)
    n_in = int(inner.sum())
    assert inner[:n_in].all() and not inner[n_in:].any(), "DGL stores the inner nodes first"
    n_all = inner.size
    u, v = np.asarray(a["edges_u"], np.int64), np.asarray(a["edges_v"], np.int64)
    keep = v < n_in
    A = sp.coo_matrix((np.ones(int(keep.sum()), np.int8), (v[keep], u[keep])), shape=(n_in, n_all)).tocsr()
    A.sum_duplicates()
    A.sort_indices()
    gid = np.asarray(a["nid"], np.int64)
    orig = np.asarray(a["orig_id"], np.int64)
    starts = np.asarray(a["starts"], np.int64)
    return RawPartition(
        rank=rank, num_parts=world, n_inner=n_in, inner_start=int(starts[rank]), starts=starts,
        indptr=A.indptr.astype(np.int64), indices=A.indices.astype(np.int32), halo_gid=gid[n_in:].astype(np.int64),
        halo_part=np.asarray(a["part_id"])[n_in:].astype(np.int32), feat=np.asarray(a["feat"], np.float32)[:n_in],
        label=np.asarray(a["label"])[:n_in], train_mask=np.asarray(a["train_mask"], bool)[:n_in],
        val_mask=np.asarray(a["val_mask"], bool)[:n_in], test_mask=np.asarray(a["test_mask"], bool)[:n_in],
        in_degrees=np.asarray(a["in_degrees_global"])[orig].astype(np.int64),
        out_degrees=np.asarray(a["out_degrees_global"])[orig].astype(np.int64),
        # predictions are keyed by DGL's reshuffled global id (dgl.NID), the numbering the partition book uses
        inner_gid=gid[:n_in].astype(np.int64))


def convert(raws: List, model_type) -> List:
    """The package's shared chain (manager.layout.layouts_from_raw), as graph_partition.py runs it."""
    from adaqp_b200.manager.layout import layouts_from_raw
    return layouts_from_raw(raws, model_type)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--part-dir", default="data/part_data")
    ap.add_argument("--dataset", required=True)
    ap.add_argument("--num-parts", type=int, required=True)
    ap.add_argument("--model", default="gcn", choices=["gcn", "sage"])
    ap.add_argument("--degree-dir", default=None)
    a = ap.parse_args()
    from adaqp_b200.helper import DistGNNType
    from adaqp_b200.manager.graphEngine import save_rank_layout
    model = DistGNNType.DistGCN if a.model == "gcn" else DistGNNType.DistSAGE
    cfg = f"{a.part_dir}/{a.dataset}/{a.num_parts}part/{a.dataset}.json"
    deg = a.degree_dir or f"graph_degrees/{a.dataset}"
    raws = [raw_from_arrays(load_dgl_arrays(cfg, r, a.num_parts, deg), r, a.num_parts) for r in range(a.num_parts)]
    for lay in convert(raws, model):
        print(save_rank_layout(lay, a.part_dir, a.dataset))


if __name__ == "__main__":
    main()

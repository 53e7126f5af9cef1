"""Step one of the workflow (the reference's graph_partition.py): cut a downloaded dataset into the per-rank
partition files that step two, main.py, trains on.  Partitioning runs on the GPU; no DGL, no network.

    python graph_partition.py --dataset ogbn-products --raw_dir data/dataset --partition_size 4
    torchrun --nproc_per_node=4 main.py --dataset ogbn-products --num_parts 4
"""
import argparse

from AdaQP.helper.partition import graph_patition_store

if __name__ == "__main__":
    parser = argparse.ArgumentParser(description="graph partition scripts")
    parser.add_argument("--dataset", type=str, default="reddit", help="training dataset")
    parser.add_argument("--raw_dir", type=str, default="data/dataset", help="dir to store raw dataset")
    parser.add_argument("--partition_dir", type=str, default="data/part_data", help="dir to store graph partition")
    parser.add_argument("--partition_size", type=int, default=2, help="graph partition size")
    parser.add_argument("--model_name", type=str, default="gcn", choices=["gcn", "sage", "gat", "gatv2"],
                        help="model the files are written for (the adaptive assigner's aggregation scores differ)")
    parser.add_argument("--seed", type=int, default=0, help="partitioner seed")
    args = parser.parse_args()
    graph_patition_store(args.dataset, args.partition_size, args.raw_dir, args.partition_dir,
                         model_name=args.model_name, seed=args.seed)

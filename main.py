"""Launcher with the reference's command line (main.py:7-14 of the reference); the
reference's own main.py also works unchanged with this repository on PYTHONPATH.

    torchrun --nproc_per_node=W --master_addr 127.0.0.1 main.py --dataset ogbn-products \
        --num_parts W --model_name gcn --mode AdaQP --assign_scheme adaptive
"""
import argparse

from AdaQP import Trainer

FLAGS = [
    ("--dataset", str, "reddit", "training dataset"),
    ("--num_parts", int, 4, "number of partitions"),
    ("--backend", str, "gloo", "control-plane backend for distributed training"),
    ("--init_method", str, "env://", "init method for distributed training"),
    ("--model_name", str, "gcn", "model for training"),
    ("--mode", str, "AdaQP", "training methods. optional modes: [Vanilla, AdaQP, AdaQP-q, AdaQP-p]"),
    ("--assign_scheme", str, "adaptive", "bit-width assignment scheme. optional schemes: [adaptive, random, uniform]"),
    ("--logger_level", str, "INFO", "logger level"),
]


def parse():
    p = argparse.ArgumentParser(description="distributed full graph training (H100-native hot path)")
    for flag, typ, default, text in FLAGS:
        p.add_argument(flag, type=typ, default=default, help=text)
    p.add_argument("--num_epoches", type=int, default=None, help="override the config's epoch count")
    p.add_argument("--aggregator_type", type=str, default=None,
                   help="GraphSAGE aggregator: mean, gcn or pool (default: the config's)")
    return p.parse_args()


if __name__ == "__main__":
    trainer = Trainer(parse())
    trainer.save(trainer.train())

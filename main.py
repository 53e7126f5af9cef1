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


def parse(argv=None):
    p = argparse.ArgumentParser(description="distributed full graph training (H100-native hot path)")
    for flag, typ, default, text in FLAGS:
        p.add_argument(flag, type=typ, default=default, help=text)
    p.add_argument("--num_epoches", type=int, default=None, help="override the config's epoch count")
    p.add_argument("--aggregator_type", type=str, default=None,
                   help="GraphSAGE aggregator: mean, gcn or pool (default: the config's)")
    p.add_argument("--appnp_k", type=int, default=None,
                   help="APPNP propagation steps K (default: the config's `appnp_k`, else 10)")
    p.add_argument("--appnp_alpha", type=float, default=None,
                   help="APPNP teleport probability alpha in [0, 1] (default: the config's `appnp_alpha`, else 0.1)")
    p.add_argument("--gcnii_layers", type=int, default=None,
                   help="GCNII propagation layers L (default: the config's `gcnii_layers`, else 8)")
    p.add_argument("--gcnii_alpha", type=float, default=None,
                   help="GCNII initial-residual weight alpha in [0, 1] (default: the config's `gcnii_alpha`, else 0.1)")
    p.add_argument("--gcnii_theta", type=float, default=None,
                   help="GCNII identity-mapping strength theta > 0, beta_l = log(theta / l + 1) "
                        "(default: the config's `gcnii_theta`, else 0.5)")
    p.add_argument("--checkpoint_dir", type=str, default=None,
                   help="directory for epoch checkpoints, `latest` and `best` (the best validation epoch's model)")
    p.add_argument("--checkpoint_every", type=int, default=None, help="write a checkpoint every N epochs (0: off)")
    p.add_argument("--resume", type=str, default=None,
                   help="continue training from a checkpoint directory, or `auto` for <checkpoint_dir>/latest; "
                        "with --predict_out: the checkpoint to predict from (default <checkpoint_dir>/best)")
    p.add_argument("--predict_out", type=str, default=None,
                   help="instead of training, write per-node predictions (logits by original node id) to this directory")
    p.add_argument("--correct_and_smooth", action="store_true",
                   help="with --predict_out: also write Correct & Smooth probabilities (cs_probs), which propagate the "
                        "train labels over the graph (single-label datasets only)")
    p.add_argument("--cs_correct_layers", type=int, default=None, help="C&S correct steps K1 (default 50)")
    p.add_argument("--cs_correct_alpha", type=float, default=None,
                   help="C&S correct propagation weight alpha1 in [0, 1] (default 0.8); 1 = pure propagation, the "
                        "reverse of --appnp_alpha, which is the teleport weight")
    p.add_argument("--cs_smooth_layers", type=int, default=None, help="C&S smooth steps K2 (default 50)")
    p.add_argument("--cs_smooth_alpha", type=float, default=None,
                   help="C&S smooth propagation weight alpha2 in [0, 1] (default 0.8); 1 = pure propagation, the "
                        "reverse of --appnp_alpha")
    p.add_argument("--cs_scale", type=str, default=None,
                   help="C&S error scale: `auto` (default; autoscale by the mean train error) or a number > 0 (fixed "
                        "scale, the train rows' errors held at each correct step)")
    args = p.parse_args(argv)
    if args.correct_and_smooth and not args.predict_out:
        p.error("--correct_and_smooth needs --predict_out")
    return args


if __name__ == "__main__":
    args = parse()
    if args.predict_out:
        checkpoint, args.resume = args.resume, None          # weights only: no training state is resumed
        Trainer(args).save_predictions(args.predict_out, checkpoint)
    else:
        trainer = Trainer(args)
        trainer.save(trainer.train())

"""Trainer: wires Communicator -> GraphEngine -> CommBuffer -> Assigner -> model and runs the
epoch loop.  Public surface of AdaQP/trainer/trainer.py:23-238 kept (`Trainer(args)`,
`.train() -> Tensor[8]`, `.save(records)`, the --mode table, the CSV columns), so the
reference's main.py drives it unchanged."""
from __future__ import annotations

import csv
import json
import os
from argparse import Namespace
from typing import Dict, Optional, Tuple

import numpy as np
import torch
import yaml
from torch import Tensor

from ..assigner import Assigner as assigner
from ..communicator import Communicator as comm
from ..communicator.p2p import layer_key_dims, with_cs_key
from ..cs import CSParams, cs_params
from ..helper import BitType
from ..manager import GraphEngine as engine
from ..model.distAPPNP import APPNP_ALPHA, APPNP_K
from ..model.distGCNII import GCNII_ALPHA, GCNII_LAYERS, GCNII_THETA
from ..model import ops
from ..model.registry import MODELS, buffer_shape
from ..manager.graphEngine import load_rank_layout
from . import checkpoint as ckpt
from .runtime_util import (_check_exchange_status, aggregate_accuracy, aggregate_F1, get_metrics, setup_logger,
                           sync_model, sync_seed, train_for_one_epoch, val_test)

RUNING_MODE = ["Vanilla", "AdaQP", "AdaQP-q", "AdaQP-p"]
# mode -> (message precision, overlap central aggregation with the exchange)
QUNAT_PARA_MAP: Dict[str, Tuple[str, bool]] = {"Vanilla": ("full", False), "AdaQP": ("quant", True),
                                               "AdaQP-q": ("quant", False), "AdaQP-p": ("full", True)}
GAT_HEADS = 4          # default of the yaml `model: gat_heads`
# run-time flags of Correct & Smooth -> cs_params arguments (None: the default)
CS_FLAGS = {"cs_correct_layers": "correct_layers", "cs_correct_alpha": "correct_alpha",
            "cs_smooth_layers": "smooth_layers", "cs_smooth_alpha": "smooth_alpha", "cs_scale": "scale"}


def exchange_key_dims(config: dict, key_dims: Optional[Dict[str, int]], cs: bool) -> Optional[Dict[str, int]]:
    """The exchange's key table: the model's own `key_dims` (None: the reference keys of buffer_shape) and, with
    Correct & Smooth, CS_KEY as wide as the output.  The Assigner and the checkpoints keep `key_dims`."""
    if not cs:
        return key_dims
    base = key_dims if key_dims is not None else layer_key_dims(buffer_shape(config, None))
    return with_cs_key(base, config["data"]["num_classes"])


def cs_config(config: dict) -> Optional[CSParams]:
    """The checked C&S parameters of the run (None: not requested).  C&S smooths softmax outputs, so a multilabel
    dataset is refused."""
    rt = config["runtime"]
    if not rt.get("correct_and_smooth"):
        return None
    if config["data"]["is_multilabel"]:
        raise ValueError(f"Correct & Smooth is defined on softmax outputs; dataset '{rt['dataset']}' is multilabel")
    return cs_params(**{arg: rt[flag] for flag, arg in CS_FLAGS.items() if rt.get(flag) is not None})


class Trainer(object):
    def __init__(self, runtime_args: Namespace):
        args = vars(runtime_args) if not isinstance(runtime_args, dict) else dict(runtime_args)
        dataset = args["dataset"]
        cfg_path = os.path.join(os.path.dirname(os.path.dirname(__file__)), "config", f"{dataset}.yaml")
        with open(cfg_path, "r") as f:
            self.config = yaml.load(f, Loader=yaml.FullLoader)
        self.config["runtime"].update({k: v for k, v in args.items() if v is not None})
        if os.environ.get("ADAQP_NUM_EPOCHES"):          # short runs of the unmodified reference main.py (no such flag there)
            self.config["runtime"]["num_epoches"] = int(os.environ["ADAQP_NUM_EPOCHES"])
        # extension: `assign_bits` / `assign_cycle` / `group_size` given at run time override the yaml's
        # `assignment:` section (the reference edits the yaml, e.g. assign_bits: 4 for uniform 4-bit)
        for k in ("assign_bits", "assign_cycle", "group_size", "coe_lambda"):
            if args.get(k) is not None:
                self.config["assignment"][k] = args[k]
        model = self.config["model"]
        model["gat_heads"] = int(args["gat_heads"]) if args.get("gat_heads") is not None else int(model.get("gat_heads", GAT_HEADS))
        # APPNP propagation steps K and teleport probability alpha: run-time value, else the yaml's, else the default
        for key, default in (("appnp_k", APPNP_K), ("appnp_alpha", APPNP_ALPHA)):
            model[key] = args[key] if args.get(key) is not None else model.get(key, default)
        # GCNII layers L, initial-residual weight alpha and identity-mapping strength theta, with the same precedence
        for key, default in (("gcnii_layers", GCNII_LAYERS), ("gcnii_alpha", GCNII_ALPHA), ("gcnii_theta", GCNII_THETA)):
            model[key] = args[key] if args.get(key) is not None else model.get(key, default)
        if args.get("aggregator_type") is not None:        # extension: run-time override of the yaml's aggregator
            model["aggregator_type"] = args["aggregator_type"]
        rt = self.config["runtime"]
        # extension: checkpoints (trainer/checkpoint.py); none of them set = no checkpoint files, as the reference
        rt.setdefault("checkpoint_dir", None)
        rt["checkpoint_every"] = int(rt.get("checkpoint_every") or 0)
        rt.setdefault("resume", None)
        if rt["checkpoint_every"] > 0 and not rt["checkpoint_dir"]:
            raise ValueError("checkpoint_every > 0 needs checkpoint_dir")
        self.resume_path, self.resume_epoch, self._partition_digest = None, 0, None
        self.cs = cs_config(self.config)
        self.exp_path = f"{rt['exp_path']}/{dataset}/{rt['num_parts']}part/{rt['model_name']}"
        self.logger = setup_logger("trainer.log", rt["logger_level"], with_file=True)
        self._set_communicator()
        if self.cs is not None and comm.ctx.transport != "p2p":
            raise NotImplementedError("Correct & Smooth runs on the p2p transport only (not the CPU gloo plumbing mode)")
        self._set_engine()
        if comm.get_rank() == 0:
            os.makedirs(self.exp_path, exist_ok=True)
        self._set_buffer()
        self._set_assigner()
        if engine.ctx.bit_type == BitType.QUANT:
            # adaptive starts from the uniform default until variances have been traced (:62-69)
            first = "uniform" if assigner.ctx.scheme == "adaptive" else None
            comm.ctx.update_buffer(assigner.ctx.get_assignment(engine.ctx.send_idx, runtime_scheme=first))
        self._set_model()

    # ---- setup --------------------------------------------------------------------------------
    def _set_communicator(self):
        rt = self.config["runtime"]
        self.communicator = comm(rt["backend"], rt["init_method"])
        self.logger.info(repr(self.communicator))

    def _set_engine(self):
        data, rt, model = self.config["data"], self.config["runtime"], self.config["model"]
        if rt["mode"] not in RUNING_MODE:
            raise ValueError(f"Invalid running mode: {rt['mode']}")
        self.spec = MODELS.get(rt["model_name"])
        if self.spec is None:
            raise ValueError(f"Invalid model type: {rt['model_name']}")
        self.spec.check(self.config)
        refusal = self.spec.p2p_only(self.config)
        if refusal is not None and comm.ctx.transport != "p2p":
            raise NotImplementedError(refusal)
        # the model's own exchange keys and widths (None: the reference's, built from buffer_shape)
        self.key_dims = self.spec.key_dims(self.config)
        precision, use_parallel = QUNAT_PARA_MAP[rt["mode"]]
        layout = None
        if rt["resume"]:
            # a checkpoint that does not belong to this run is refused before any device work or exchange
            layout = load_rank_layout(data["partition_path"], rt["dataset"], self.spec.kind)
            self._partition_digest = ckpt.partition_digest(layout)
            self.resume_path = ckpt.resolve(rt["resume"], rt["checkpoint_dir"])
            self.resume_epoch = ckpt.check_resume(self.resume_path, self.run_fields(), self._partition_digest,
                                                  rt["num_epoches"])
        self.engine = engine(rt["num_epoches"], data["partition_path"], rt["dataset"], precision,
                             self.spec.kind, use_parallel, layout=layout)
        engine.ctx.agg_type = model["aggregator_type"]
        engine.ctx.top_layer = model["num_layers"] - 1
        if engine.ctx.use_parallel:
            for g in (engine.ctx.graph, engine.ctx.bwd_graph):
                g.init_copy_buffers(data["num_feats"], model["hidden_dim"], model["num_layers"], engine.ctx.device)
        self.logger.info(repr(self.engine))

    def _set_buffer(self):
        comm.ctx.init_buffer(buffer_shape(self.config, self.key_dims), engine.ctx.send_idx, engine.ctx.recv_idx,
                             engine.ctx.bit_type, total_send_idx=engine.ctx.total_send_idx,
                             num_remote=engine.ctx.num_remove,
                             key_dims=exchange_key_dims(self.config, self.key_dims, self.cs is not None))
        self.spec.setup(engine.ctx, comm.ctx.comm_buffer.p2p)

    def run_fields(self) -> dict:
        """What a checkpoint's manifest records about the run (trainer/checkpoint.py)."""
        return ckpt.run_fields(self.config, self.key_dims)

    def _set_assigner(self):
        data, model, rt, asg = (self.config[k] for k in ("data", "model", "runtime", "assignment"))
        self.assigner = assigner(data["num_feats"], model["hidden_dim"], model["num_layers"],
                                 asg["profile_data_length"], rt["assign_scheme"], asg["assign_bits"],
                                 engine.ctx.scores, asg["group_size"], asg["coe_lambda"], asg["assign_cycle"],
                                 key_dims=self.key_dims)
        self.logger.info(self.assigner)

    def _set_model(self):
        self.model = self.spec.build(self.config).to(comm.ctx.device)

    # ---- runtime ----------------------------------------------------------------------------------
    def train(self):
        rt = self.config["runtime"]
        multilabel = self.config["data"]["is_multilabel"]
        if self.resume_path is None:
            sync_seed()
            self.model.reset_parameters()
            sync_model(self.model)
        optimizer = torch.optim.Adam(self.model.parameters(), lr=rt["learning_rate"], weight_decay=rt["weight_decay"])
        self.optimizer = optimizer
        criterion = torch.nn.BCEWithLogitsLoss(reduction="sum") if multilabel else torch.nn.CrossEntropyLoss(reduction="sum")
        eng = self.engine.ctx
        feats, labels = eng.feats, eng.labels
        n_train = torch.LongTensor([eng.train_mask.numel()])
        comm.all_reduce_sum(n_train)
        n_train = n_train.item()
        assign_time, train_time = [], []
        self.exposed_comm_ms, self.losses = [], []
        if self.resume_path is not None:
            # in place of seeding and initialising: model, optimizer, RNG states, Assigner and Recorder of epoch E
            rec = ckpt.load_run(self.resume_path, self.model, optimizer)
            assign_time, train_time, self.exposed_comm_ms, self.losses = (
                rec["assign_time"], rec["train_time"], rec["exposed_comm_ms"], rec["loss"])
            self.logger.info(f"<resumed from {self.resume_path} at epoch {self.resume_epoch}>")
        # per-epoch records of the whole run (resumed epochs included), as checkpoints carry them
        self.epoch_records = {"assign_time": assign_time, "train_time": train_time,
                              "exposed_comm_ms": self.exposed_comm_ms, "loss": self.losses}
        best_val = float(eng.recorder.epoches_metrics[:self.resume_epoch, 1].max()) if self.resume_epoch else -float("inf")
        for epoch in range(self.resume_epoch + 1, rt["num_epoches"] + 1):
            overhead, loss, traced, reduce_time = train_for_one_epoch(
                epoch, eng.graph, self.model, feats, labels, optimizer, criterion, n_train, eng.train_mask)
            assign_time.append(overhead)
            train_time.append(traced)
            self.exposed_comm_ms.append(getattr(eng, "last_exposed_comm_ms", 0.0))
            metrics = val_test(eng.graph, self.model, feats, labels, eng.train_mask, eng.val_mask, eng.test_mask, multilabel)
            info = (aggregate_F1 if multilabel else aggregate_accuracy)(loss, metrics, epoch)
            if epoch % rt["log_steps"] == 0:
                if comm.get_rank() == 0:
                    if not eng.use_parallel:
                        t = (f"Worker 0 | Total Time {traced[0]:.4f}s | Comm Time {traced[1]:.4f}s | Quant Time "
                             f"{traced[2]:.4f}s | Agg Time {traced[-1]:.4f}s | Reduce Time {reduce_time:.4f}s")
                    else:
                        t = (f"Worker 0 | Total Time {traced[0]:.4f}s | Comm Time {traced[1]:.4f}s | Quant Time "
                             f"{traced[2]:.4f}s | Central Agg Time {traced[3]:.4f}s | Marginal Agg Time "
                             f"{traced[4]:.4f}s | Reduce Time {reduce_time:.4f}s | Exposed Comm "
                             f"{self.exposed_comm_ms[-1]:.3f}ms")
                    self.logger.info(info + "\n" + t)
                comm.barrier()
            self.losses.append(float(loss.detach()))
            if rt["checkpoint_dir"]:
                # outside the timed region of the epoch
                row = eng.recorder.epoches_metrics[epoch - 1].tolist()
                if row[1] > best_val:
                    best_val = row[1]
                    if comm.get_rank() == 0:
                        ckpt.save_best(rt["checkpoint_dir"], epoch, self.model, self.run_fields(), row,
                                       "f1_micro" if multilabel else "accuracy")
                if rt["checkpoint_every"] > 0 and epoch % rt["checkpoint_every"] == 0:
                    if self._partition_digest is None:
                        self._partition_digest = ckpt.partition_digest(eng.layout)
                    ckpt.save(rt["checkpoint_dir"], epoch, self.model, optimizer, self.run_fields(),
                              self._partition_digest, self.epoch_records)
        tt = torch.tensor(train_time)
        records = torch.concat([torch.tensor(assign_time).sum().view(-1), tt.sum(dim=0)[0].view(-1), tt.mean(dim=0)])
        comm.ctx.delete_buffer()
        return records

    # ---- inference ----------------------------------------------------------------------------------
    def predict(self, checkpoint: str = None) -> Tensor:
        """Load model weights from an epoch or `best` checkpoint (default `<checkpoint_dir>/best`; `auto` = the
        latest epoch) and run one evaluation forward.  Returns this rank's [n_inner, C] logits in layout row order;
        `predict_metrics` holds the global train / val / test metric.  The run may use another `num_parts` or
        `mode` than the one that trained the weights."""
        rt, eng = self.config["runtime"], self.engine.ctx
        if checkpoint is None:
            if not rt["checkpoint_dir"]:
                raise ValueError("predict() needs a checkpoint directory or checkpoint_dir")
            checkpoint = os.path.join(rt["checkpoint_dir"], "best")
        path = ckpt.resolve(checkpoint, rt["checkpoint_dir"])
        self.predict_manifest = ckpt.load_weights(path, self.model, self.run_fields())
        self.predict_checkpoint = path
        self.model.eval()
        with torch.no_grad():
            logits = self.model(eng.graph, eng.feats)
        eng.timer.clear(is_train=False)
        _check_exchange_status()
        multilabel = self.config["data"]["is_multilabel"]
        m = []
        for mask in (eng.train_mask, eng.val_mask, eng.test_mask):
            m.extend(float(x) for x in get_metrics(eng.labels[mask], logits[mask], multilabel))
        m = torch.tensor(m, dtype=torch.float64)
        comm.all_reduce_sum(m)
        if multilabel:          # micro-F1 from the summed tp / predicted / actual counts, as aggregate_F1
            self.predict_metrics = [float(2 * m[3 * k] / max(float(m[3 * k + 1] + m[3 * k + 2]), 1.0)) for k in range(3)]
        else:
            self.predict_metrics = [float(m[2 * k] / max(float(m[2 * k + 1]), 1.0)) for k in range(3)]
        return logits

    def correct_and_smooth(self, logits: Tensor) -> Tensor:
        """Correct & Smooth (DESIGN §16) of predict()'s [n_inner, C] logits with this rank's train labels (val and
        test labels are never read); every rank calls it together.  Returns the smoothed probabilities and sets
        `cs_metrics`, their global train / val / test argmax accuracy.  Needs `correct_and_smooth` in the run's
        arguments, which adds the exchange key the steps use."""
        if self.cs is None:
            raise ValueError("correct_and_smooth() needs the run to be built with correct_and_smooth set")
        eng = self.engine.ctx
        y = torch.full((eng.num_inner,), -1, dtype=torch.int32, device=logits.device)
        y[eng.train_mask] = eng.labels[eng.train_mask].to(torch.int32)
        n_train = torch.LongTensor([eng.train_mask.numel()])
        comm.all_reduce_sum(n_train)
        with torch.no_grad():
            probs = ops.correct_and_smooth(eng.graph, logits, y, self.cs, int(n_train.item()))
        _check_exchange_status()
        m = []
        for mask in (eng.train_mask, eng.val_mask, eng.test_mask):
            m.extend(float(x) for x in get_metrics(eng.labels[mask], probs[mask], False))
        m = torch.tensor(m, dtype=torch.float64)
        comm.all_reduce_sum(m)
        self.cs_metrics = [float(m[2 * k] / max(float(m[2 * k + 1]), 1.0)) for k in range(3)]
        return probs

    def save_predictions(self, out_dir: str, checkpoint: str = None) -> str:
        """predict(), then each rank writes `out_dir/shard{r}.npz` (`node_id`, `logits`) and rank 0 merges the
        shards from disk into `out_dir/predictions.npz`: `node_id` int64 [N] ascending, `logits` float32 [N, C]
        and a JSON header with the checkpoint's epoch and the train / val / test metric.  With Correct & Smooth the
        file also holds `cs_probs` float32 [N, C] (correct_and_smooth of the logits, merged the same way) and the
        header its parameters (`correct_and_smooth`) and accuracies (`cs_train`, `cs_val`, `cs_test`)."""
        rank, W = comm.get_rank(), comm.get_world_size()
        gid = engine.ctx.layout.inner_gid
        if not all(comm.gather_all(gid is not None)):
            raise ValueError("the partition files carry no original node ids (inner_gid): re-partition with "
                             "graph_partition.py or tools/convert_dgl_partition.py to write predictions by node id")
        logits = self.predict(checkpoint)
        extra = {}
        if self.cs is not None:
            extra["cs_probs"] = self.correct_and_smooth(logits).cpu().numpy()
        os.makedirs(out_dir, exist_ok=True)
        np.savez(os.path.join(out_dir, f"shard{rank}.npz"), node_id=np.asarray(gid, np.int64),
                 logits=logits.float().cpu().numpy(), **extra)
        comm.barrier()
        final = os.path.join(out_dir, "predictions.npz")
        if rank == 0:
            shards = [np.load(os.path.join(out_dir, f"shard{r}.npz")) for r in range(W)]
            ids = np.concatenate([s["node_id"] for s in shards])
            order = np.argsort(ids, kind="stable")
            header = {"checkpoint": self.predict_checkpoint, "epoch": int(self.predict_manifest["epoch"]),
                      "num_parts": W, "metric": "f1_micro" if self.config["data"]["is_multilabel"] else "accuracy",
                      **dict(zip(("train", "val", "test"), self.predict_metrics))}
            merged = {}
            if self.cs is not None:
                header["correct_and_smooth"] = self.cs.as_dict()
                header.update(zip(("cs_train", "cs_val", "cs_test"), self.cs_metrics))
                merged["cs_probs"] = np.concatenate([s["cs_probs"] for s in shards])[order]
            tmp = os.path.join(out_dir, ".predictions.tmp.npz")
            with open(tmp, "wb") as f:
                np.savez(f, node_id=ids[order], logits=np.concatenate([s["logits"] for s in shards])[order],
                         header_json=np.frombuffer(json.dumps(header).encode("utf-8"), dtype=np.uint8), **merged)
            os.replace(tmp, final)
        comm.barrier()
        comm.ctx.delete_buffer()
        return final

    def save(self, time_records: Tensor):
        if comm.get_rank() != 0:
            comm.gather_any(time_records, None, dst=0)
            comm.barrier()
            return
        rows = [None] * comm.get_world_size()
        comm.gather_any(time_records, rows, dst=0)
        paths = {k: f"{self.exp_path}/{k}" for k in ("metrics", "time", "val_curve")}
        for p in paths.values():
            os.makedirs(p, exist_ok=True)
        name = self.config["runtime"]["mode"]
        if engine.ctx.bit_type == BitType.QUANT:
            name = f"{name}_{self.config['runtime']['assign_scheme']}"
        engine.ctx.recorder.display_final_statistics(f"{paths['metrics']}/{name}.txt", f"{paths['val_curve']}/{name}.pt",
                                                     self.config["runtime"]["model_name"])
        csv_path = f"{paths['time']}/{name}.csv"
        new_file = not os.path.exists(csv_path)
        with open(csv_path, "a") as f:
            w = csv.writer(f)
            if new_file:
                w.writerow(["Worker", "Overhead", "Total", "Per_epoch", "Comm", "Quant", "Central", "Marginal", "Full"])
            for worker, rec in enumerate(rows):
                line = [f"Worker {worker}"] + list(rec.numpy())
                assert len(line) == 9, f"Invalid write data length: {len(line)}"
                w.writerow(line)
        comm.barrier()

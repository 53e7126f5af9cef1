"""Epoch loop pieces: seeding, model sync, gradient reduction, train/eval steps, metrics.

Mirror of AdaQP/trainer/runtime_util.py:22-197 (function names and return values kept).
The gradient all-reduce is the first "next" row of SURVEY.md 8f: instead of one gloo
all_reduce per parameter on CUDA tensors (:71-77) the gradients are flattened into one
bucket and reduced once over NCCL (NVLink/NVSwitch) when the ranks own GPUs; on the CPU
plumbing configuration the reference's per-parameter gloo reduction is used.
"""
from __future__ import annotations

import logging
import time
from typing import Any, List, Tuple, Union

import numpy as np
import torch
import torch.distributed as dist
from torch import Tensor, nn
from torch.optim import Optimizer

from ..assigner import Assigner as assigner
from ..communicator import Communicator as comm
from ..helper import BitType
from ..manager import GraphEngine as engine
from ..model import ops

_nccl_group = None


def setup_logger(log_file, level=logging.INFO, with_file=True):
    lg = logging.getLogger("trainer")
    lg.setLevel(level)
    if with_file and not any(isinstance(h, logging.FileHandler) for h in lg.handlers):
        fh = logging.FileHandler(log_file)
        fh.setFormatter(logging.Formatter("%(asctime)s %(levelname)s %(message)s"))
        lg.addHandler(fh)
    return lg


def fix_seed(seed: int = 0):
    torch.manual_seed(seed)
    if torch.cuda.is_available():
        torch.cuda.manual_seed(seed)
        torch.cuda.manual_seed_all(seed)
    np.random.seed(seed)


def sync_seed(seed: int = None):
    """Rank 0 draws a wall-clock seed and broadcasts it (runtime_util.py:40-53); pass `seed`
    (or set ADAQP_SEED) for reproducible / parity runs."""
    import os
    box = [None]
    if comm.get_rank() == 0:
        env = os.environ.get("ADAQP_SEED")
        box[0] = seed if seed is not None else (int(env) if env else int(time.time() % (2 ** 32 - 1)))
    comm.broadcast_any(box, src=0)
    fix_seed(box[0])
    return box[0]


def _reduce_group():
    global _nccl_group
    if comm.ctx.device.type != "cuda" or comm.get_world_size() == 1 or not dist.is_nccl_available():
        return None
    if _nccl_group is None:
        import os
        want = os.environ.get("ADAQP_GRAD_REDUCE", "auto").lower()
        devs = comm.gather_all(str(torch.cuda.get_device_properties(comm.ctx.device).uuid))
        shared = len(set(devs)) < len(devs)          # NCCL refuses two ranks on one GPU (tests)
        _nccl_group = False if (want == "gloo" or shared) else dist.new_group(backend="nccl")
    return _nccl_group or None


def sync_model(model: nn.Module):
    """Every rank ends up with rank 0's parameters (sum of rank 0's values and zeros)."""
    grp = _reduce_group()
    for _, value in model.state_dict().items():
        if comm.get_rank() != 0:
            value.zero_()
        if grp is not None:
            dist.all_reduce(value.data, group=grp)
        else:
            comm.all_reduce_sum(value.data)


def average_gradients(model: nn.Module):
    """Sum the gradients over ranks (the loss is already divided by the global number of
    training samples, runtime_util.py:102)."""
    grads = [p.grad.data for p in model.parameters() if p.requires_grad and p.grad is not None]
    grp = _reduce_group()
    if grp is None:
        for g in grads:
            comm.all_reduce_sum(g)
        return
    flat = torch._utils._flatten_dense_tensors(grads)
    dist.all_reduce(flat, group=grp)
    for g, r in zip(grads, torch._utils._unflatten_dense_tensors(flat, grads)):
        g.copy_(r)


def _check_exchange_status():
    """A flag / ack spin that timed out inside the exchange kernels only sets the slab's status word (the
    kernels cannot raise): poll it once per epoch / evaluation, after the step's synchronisation point, and
    turn it into an exception instead of training on stale halo rows."""
    buf = comm.ctx.comm_buffer
    if buf is not None and getattr(buf, "p2p", None) is not None:
        buf.p2p.check_status()


def train_for_one_epoch(epoch: int, graph, model: nn.Module, input_data: Tensor, labels: Tensor,
                        optimizer: Optimizer, criterion: Union[nn.Module, Any], total_num_training_samples: int,
                        train_mask: Tensor) -> Tuple[Any, Tensor, List[float], float]:
    overhead = 0.0
    if epoch % assigner.ctx.assign_cycle == 1 and epoch != 1:
        if assigner.ctx.scheme in ["adaptive", "random"] and engine.ctx.bit_type == BitType.QUANT:
            logging.getLogger("trainer").info(f"<epoch {epoch}, updating bit-width...>")
            t0 = time.time()
            comm.ctx.update_buffer(assigner.ctx.get_assignment(engine.ctx.send_idx))
            overhead = time.time() - t0
    epoch_start = time.time()
    model.train()
    # the loss reads only the train rows: the output layer's aggregation computes just those (ops.loss_rows)
    with ops.loss_rows(train_mask):
        logits = model(graph, input_data)
    loss = criterion(logits[train_mask], labels[train_mask]) / total_num_training_samples
    optimizer.zero_grad()
    loss.backward()
    update_start = time.time()
    average_gradients(model)
    reduce_time = time.time() - update_start
    optimizer.step()
    if comm.ctx.device.type == "cuda":
        torch.cuda.synchronize()
    epoch_time = time.time() - epoch_start
    _check_exchange_status()
    engine.ctx.last_exposed_comm_ms = engine.ctx.timer.exposed_comm_ms()
    traced_time = engine.ctx.timer.epoch_traced_time()
    engine.ctx.timer.clear()
    traced_time.insert(0, epoch_time)
    return overhead, loss, traced_time, reduce_time


@torch.no_grad()
def val_test(graph, model: nn.Module, input_data: Tensor, labels: Tensor, train_mask: Tensor, val_mask: Tensor,
             test_mask: Tensor, is_multilabel: bool = False):
    model.eval()
    logits = model(graph, input_data)
    metrics = []
    for mask in (train_mask, val_mask, test_mask):
        metrics.extend(get_metrics(labels[mask], logits[mask], is_multilabel))
    engine.ctx.timer.clear(is_train=False)
    _check_exchange_status()
    return metrics


def get_metrics(labels: Tensor, logits: Tensor, is_F1):
    if is_F1:
        pred = logits > 0
        tp = torch.logical_and(pred == 1, labels == 1).float().sum()
        fp = torch.logical_and(pred == 1, labels == 0).float().sum()
        fn = torch.logical_and(pred == 0, labels == 1).float().sum()
        return [tp, tp + fp, tp + fn]
    correct = (torch.argmax(logits, dim=-1) == labels).float().sum()
    return [correct, labels.shape[0]]


def aggregate_accuracy(loss: Tensor, metrics: List[Union[float, int]], epoch: int) -> str:
    m = torch.FloatTensor([float(x) for x in metrics])
    comm.all_reduce_sum(m)
    train_acc, val_acc, test_acc = m[0] / m[1], m[2] / m[3], m[4] / m[5]
    loss = loss.detach().float().cpu()
    comm.all_reduce_sum(loss)
    engine.ctx.recorder.add_new_metrics(epoch, [train_acc, val_acc, test_acc])
    return (f"Epoch {epoch:05d} | Loss {loss.item():.4f} | Train Acc {train_acc * 100:.2f}% | "
            f"Val Acc {val_acc * 100:.2f}% | Test Acc {test_acc * 100:.2f}%")


def aggregate_F1(loss: Tensor, metrics: List[Union[float, int]], epoch: int) -> str:
    def safe(n, d):
        return n / (d if d != 0 else 1)
    m = torch.FloatTensor([float(x) for x in metrics])
    comm.all_reduce_sum(m)
    f1 = []
    for k in range(3):
        prec, rec = safe(m[3 * k], m[3 * k + 1]), safe(m[3 * k], m[3 * k + 2])
        f1.append(safe(2 * prec * rec, prec + rec))
    loss = loss.detach().float().cpu()
    comm.all_reduce_sum(loss)
    engine.ctx.recorder.add_new_metrics(epoch, f1)
    return (f"Epoch {epoch:05d} | Loss {loss.item():.4f} | Train F1 micro {f1[0] * 100:.2f}% | "
            f"Val F1 micro {f1[1] * 100:.2f}% | Test F1 micro {f1[2] * 100:.2f}%")

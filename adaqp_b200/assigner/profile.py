"""alpha-beta cost model of every (src, dst) channel: time_ms = alpha * MB + beta.

Reference: AdaQP/assigner/profile.py:18-106 times 200 `dist.send` payloads per peer pair
over gloo and fits a line with np.polyfit; that is kept for the 'gloo' transport.

On the 'p2p' transport the thing being modelled is the real exchange: ONE
`send_quant_kernel` launch per rank quantises, packs and stores to ALL peers, and one
`recv_quant_kernel` launch dequantises what arrived.  Both are issue-bound on the packed
bytes (one Philox block per byte), not link-bound, so a peer-copy timing says nothing
about them (round 1 timed `copy_` to the peer slab: at full scale the fitted slope was
~0 and `adaptive` chose 8 bits everywhere).  `_profile_p2p` therefore runs the real
kernel pair at uniform 2 / 4 / 8 bits for both layer widths, times each kernel ALONE with
CUDA events, and fits time = alpha * (MB this rank sends) + beta per RANK; every channel of
the rank carries the rank's (alpha, beta) and the solver's 'concurrent' schedule charges
the rank alpha * (MB of all its channels) + beta (assigner/solver.py).
"""
from __future__ import annotations

import time
from typing import Dict, Tuple

import numpy as np
import torch

from ..communicator import BITS_SET
from ..communicator import Communicator as comm
from ..helper import MessageType
from ..manager import GraphEngine as engine


def payload_sizes(num_nodes: int, feat_dim: int, hidden_dim: int, num_data: int) -> np.ndarray:
    """Byte sizes between the all-2-bit and all-8-bit payload of a channel (profile.py:25-28)."""
    low = round(num_nodes * min(feat_dim, hidden_dim) * BITS_SET[0] / 8)
    high = round(num_nodes * max(feat_dim, hidden_dim) * BITS_SET[-1] / 8)
    tol = round(low / 2)
    return np.linspace(max(low - tol, 1), high + tol, num_data).astype(np.int64)


def fit_cost_model(dataset: Tuple[Dict[str, np.ndarray], Dict[str, np.ndarray]]) -> Dict[str, np.ndarray]:
    sizes_mb, times_ms = dataset
    out = {}
    for k in sizes_mb:
        x, y = np.asarray(sizes_mb[k], np.float64), np.asarray(times_ms[k], np.float64)
        ab = np.polyfit(x, y, 1) if np.ptp(x) > 0 else np.array([0.0, float(y.mean())])
        out[k] = ab
    return out


def _profile_p2p(feat_dim, hidden_dim, num_data, warmup, reps: int = 5):
    """Per-rank (alpha, beta) of the real send + receive kernel pair.  Collective: every rank runs the
    same sequence of buffer updates and exchanges.  `num_data` (the reference's number of payload sizes)
    is not needed: the payloads are the three uniform bit-widths x two layer widths of the real plan."""
    buf = comm.ctx.comm_buffer
    ex = buf.p2p
    rank = comm.get_rank()
    dev = comm.ctx.device
    n_inner = engine.ctx.num_inner
    # the real exchanged widths of the first two forward keys (feat_dim / hidden_dim for GCN and SAGE; GAT exchanges
    # the projected rows, hidden_dim wide from layer 0 on)
    keys = [(k, ex.dims[k]) for k in ("forward0", "forward1") if k in ex.dims]
    xs = {k: torch.relu(torch.randn(n_inner, F, device=dev)) for k, F in keys}
    S = int(sum(hi - lo for lo, hi in ex.send_idx.values()))
    mbs, ts = [], []
    was = ex.profile
    for b in BITS_SET:
        assign = {k: {p: torch.full((hi - lo,), b, dtype=torch.int32) for p, (lo, hi) in ex.send_idx.items()} for k, _ in keys}
        buf._update(assign)
        for k, F in keys:
            for it in range(warmup + reps):
                if it == warmup:
                    torch.cuda.synchronize(dev)
                    comm.barrier()
                    ex.profile = True
                    ex.kernel_times_ms()
                ex.post_send_quant(k, xs[k], 1234, 0)
                ex.wait_flags_quant(k)
                ex.complete_recv_quant(k)
            t = ex.kernel_times_ms()
            ex.profile = False
            mbs.append(S * F * b / 8 / (1024 ** 2))
            ts.append((t["send"] + t["recv"]) / reps)
    ex.profile = was
    ex.check_status()
    buf._delete_train_buffer()
    comm.barrier()
    sizes_mb = {f"{rank}_{p}": np.asarray(mbs) for p in ex.send_idx}
    times_ms = {f"{rank}_{p}": np.asarray(ts) for p in ex.send_idx}
    return sizes_mb, times_ms


def _profile_gloo(feat_dim, hidden_dim, num_data, warmup):
    """profile.py:46-95: sender times dist.send of every payload, receivers drain."""
    rank, W = comm.get_rank(), comm.get_world_size()
    send_idx, recv_idx = engine.ctx.send_idx, engine.ctx.recv_idx
    sizes_mb, times_ms = {}, {}
    for sender in range(W):
        if sender == rank:
            for p, (lo, hi) in send_idx.items():
                sizes = payload_sizes(hi - lo, feat_dim, hidden_dim, num_data)
                ts = []
                for n in sizes:
                    buf = torch.zeros(int(n), dtype=torch.uint8)
                    reps = []
                    for it in range(1, 3 * warmup):
                        t0 = time.time()
                        comm.sync_send(buf, p, MessageType.DATA)
                        if it > warmup:
                            reps.append(time.time() - t0)
                    ts.append(1000 * sum(reps) / max(len(reps), 1))
                sizes_mb[f"{rank}_{p}"] = sizes / (1024 ** 2)
                times_ms[f"{rank}_{p}"] = np.asarray(ts)
        elif sender in recv_idx:
            for n in payload_sizes(len(recv_idx[sender]), feat_dim, hidden_dim, num_data):
                buf = torch.zeros(int(n), dtype=torch.uint8)
                for _ in range(1, 3 * warmup):
                    comm.sync_recv(buf, sender, MessageType.DATA)
        comm.barrier()
    return sizes_mb, times_ms


def generate_cost_model_dataset(feat_dim: int, hidden_dim: int, num_data: int, warmup: int):
    if comm.ctx.transport == "p2p":
        return _profile_p2p(feat_dim, hidden_dim, num_data, max(warmup, 1))
    return _profile_gloo(feat_dim, hidden_dim, num_data, max(warmup, 1))

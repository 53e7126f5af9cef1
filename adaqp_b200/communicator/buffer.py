"""CommBuffer: registry of the boundary-message buffers and the wire-format metadata.

Interface of AdaQP/communicator/buffer.py:22-264 (constructor, getters, _update, _delete,
BITS_SET, the typing aliases).  Two transports:

* 'p2p'  -- buffers are regions of the rank's device slab (communicator/p2p.py).
  Quantised "train" receive buffers are zero-copy views with exactly the reference's
  layout `(int8[sum_b qsize_b], bf16[2, S_p])`; there are no pinned host copies (entries
  are None) because nothing is staged through the host.
* 'gloo' -- the reference's buffers: pinned host send/recv tensors plus device receive
  tensors, sized by the same rule (buffer.py:154-248).

The auxiliary maps (per-bit original row ids and (q_size, rows) per peer,
buffer.py:188-231) are kept for both transports; receivers learn the senders' maps through
one all_gather_object per update, as in the reference.
"""
from __future__ import annotations

import logging
from typing import Dict, List, NewType, Tuple, Union

import torch
import torch.distributed as dist
from torch import Tensor

from ..helper import BitType
from . import p2p

logger = logging.getLogger("trainer")

Basic_Buffer_Type = NewType("Basic_Buffer_Type", Dict[int, Union[Tensor, Tuple[Tensor, Tensor]]])
Test_Buffer_Type = NewType("Test_Buffer_Type", List[Basic_Buffer_Type])
Train_Buffer_Type = NewType("Train_Buffer_Type", Dict[str, Basic_Buffer_Type])
Auxillary_Buffer_Type = NewType("Auxillary_Buffer_Type", Dict[str, Dict[int, Dict[int, Union[Tensor, Tuple[int, int]]]]])

BITS_SET = (2, 4, 8)


def _pin(t: Tensor) -> Tensor:
    return t.pin_memory() if torch.cuda.is_available() else t


class CommBuffer(object):
    def __init__(self, buffer_shape: List[int], send_idx: Dict[int, Tuple[int, int]],
                 recv_idx: Basic_Buffer_Type, bit_type: BitType, device: torch.device,
                 transport: str = None, total_send_idx: Tensor = None, num_remote: int = None,
                 exchange: "p2p.PeerExchange" = None, key_dims: Dict[str, int] = None):
        assert bit_type in [BitType.FULL, BitType.QUANT], f"bit_type should be either FULL or QUANT, but got {bit_type}"
        self.buffer_shape = [int(x) for x in buffer_shape]
        self.key_dims = key_dims          # per-key exchange widths (GAT); None = the layer keys of buffer_shape
        self.device = torch.device(device)
        self.bit_type = bit_type
        self.transport = transport or ("p2p" if self.device.type == "cuda" else "gloo")
        self.send_idx, self.recv_idx = send_idx, recv_idx
        self.test_recv_buffers_cpu: Test_Buffer_Type = []
        self.test_recv_buffers_gpu: Test_Buffer_Type = []
        self.test_send_buffers_cpu: Test_Buffer_Type = []
        self.train_recv_buffers_cpu: Train_Buffer_Type = {}
        self.train_recv_buffers_gpu: Train_Buffer_Type = {}
        self.train_send_buffers_cpu: Train_Buffer_Type = {}
        self.send_original_idx_buffers: Auxillary_Buffer_Type = {}
        self.recv_original_idx_buffers: Auxillary_Buffer_Type = {}
        self.recv_original_size_buffers: Auxillary_Buffer_Type = {}
        self.p2p: p2p.PeerExchange = exchange
        if self.transport == "p2p" and self.p2p is None:
            self._init_p2p(total_send_idx, num_remote)
        self._generate_test_buffer(send_idx, recv_idx)

    # ---- p2p rendezvous ------------------------------------------------------------------
    def _init_p2p(self, total_send_idx, num_remote):
        if total_send_idx is None or num_remote is None:
            from ..manager import GraphEngine as engine      # reference call sites pass neither
            total_send_idx, num_remote = engine.ctx.total_send_idx, engine.ctx.num_remove
        rank, W = dist.get_rank(), dist.get_world_size()
        ex = p2p.PeerExchange(rank, W, self.device, self.buffer_shape, self.send_idx, self.recv_idx,
                              total_send_idx, num_remote, key_dims=self.key_dims)
        metas = [None] * W
        dist.all_gather_object(metas, ex.local_meta())
        slab = ex.allocate(metas)
        handles = [None] * W
        dist.all_gather_object(handles, (self.device.index, slab.export_handle()))
        bases = {}
        for p, (dev_idx, h) in enumerate(handles):
            if p != rank and (p in ex.send_idx or p in ex.recv_idx):
                bases[p] = slab.open_peer(h)
        ex.connect(bases)
        dist.barrier()
        self.p2p = ex

    # ---- getters (buffer.py:52-72) -----------------------------------------------------
    def get_test_buffer(self, idx: int):
        return self.test_recv_buffers_cpu[idx], self.test_recv_buffers_gpu[idx], self.test_send_buffers_cpu[idx]

    def get_train_buffer(self, layer: str):
        if self.bit_type == BitType.FULL:
            return self.get_test_buffer(p2p.layer_index(layer))
        return self.train_recv_buffers_cpu[layer], self.train_recv_buffers_gpu[layer], self.train_send_buffers_cpu[layer]

    def get_auxillary_buffer(self, layer: str):
        return self.recv_original_idx_buffers[layer], self.recv_original_size_buffers[layer], self.send_original_idx_buffers[layer]

    # ---- fp32 "test" buffers (buffer.py:154-174) --------------------------------------------
    def _generate_test_buffer(self, send_idx, recv_idx):
        for li, dim in enumerate(self.buffer_shape):
            send_cpu, recv_cpu, recv_gpu = {}, {}, {}
            for pid, (lo, hi) in send_idx.items():
                send_cpu[pid] = _pin(torch.zeros((hi - lo, dim), dtype=torch.float32)) if self.transport == "gloo" else None
            for pid, idx in recv_idx.items():
                n = len(idx)
                if self.transport == "gloo":
                    recv_cpu[pid] = _pin(torch.zeros((n, dim), dtype=torch.float32))
                    recv_gpu[pid] = torch.zeros((n, dim), dtype=torch.float32, device=self.device)
                else:
                    recv_cpu[pid] = None
                    recv_gpu[pid] = self._halo_slice(f"test{li}", idx)
            self.test_send_buffers_cpu.append(send_cpu)
            self.test_recv_buffers_cpu.append(recv_cpu)
            self.test_recv_buffers_gpu.append(recv_gpu)

    def _halo_slice(self, key: str, idx):
        """Rows of the halo matrix a peer fills, as a view when they are one ascending run
        (true whenever halo nodes are grouped by owner); None otherwise."""
        idx = torch.as_tensor(idx).cpu()
        if len(idx) and int(idx[-1] - idx[0]) == len(idx) - 1 and bool((idx[1:] > idx[:-1]).all()):
            return self.p2p.halo(key)[int(idx[0]):int(idx[-1]) + 1]
        return None

    # ---- quantised "train" buffers (buffer.py:176-248) ---------------------------------------
    def _generate_train_buffer(self, bits_assignment_rst: Dict[str, Dict[int, Tensor]], bits: Tuple[int, ...] = BITS_SET):
        rank, W = dist.get_rank(), dist.get_world_size()
        send_sizes: Dict[str, Dict[int, Dict[int, Tuple[int, int]]]] = {}
        for layer, per_peer in bits_assignment_rst.items():
            # the key's real width (models with their own keys); the layer keys of buffer_shape otherwise
            dim = self.p2p.dims[layer] if self.p2p is not None else self.buffer_shape[p2p.layer_index(layer)]
            self.send_original_idx_buffers[layer] = {}
            send_sizes[layer] = {}
            for pid, cfg in per_peer.items():
                self.send_original_idx_buffers[layer][pid] = {}
                send_sizes[layer][pid] = {}
                for b in bits:
                    ids = torch.nonzero(torch.as_tensor(cfg) == b).view(-1)
                    if len(ids):
                        self.send_original_idx_buffers[layer][pid][b] = ids
                        send_sizes[layer][pid][b] = (p2p.qsize(len(ids), b, dim), len(ids))
        gathered = [None] * W
        payload = [self.send_original_idx_buffers, send_sizes]
        if self.transport == "p2p":
            payload.append(self.p2p.quant_meta(bits_assignment_rst))
        dist.all_gather_object(gathered, payload)
        for layer in self.send_original_idx_buffers:
            self.recv_original_idx_buffers[layer] = {}
            self.recv_original_size_buffers[layer] = {}
            for i in range(W):
                if i != rank and rank in gathered[i][0][layer]:
                    self.recv_original_idx_buffers[layer][i] = gathered[i][0][layer][rank]
                    self.recv_original_size_buffers[layer][i] = gathered[i][1][layer][rank]
        if self.transport == "p2p":
            self.p2p.update_quant([g[2] for g in gathered])
            for layer in self.send_original_idx_buffers:
                self.train_send_buffers_cpu[layer] = {pid: None for pid in send_sizes[layer]}
                self.train_recv_buffers_cpu[layer] = {pid: None for pid in self.recv_original_size_buffers[layer]}
                self.train_recv_buffers_gpu[layer] = {pid: self.p2p.recv_region(layer, pid)
                                                      for pid in self.recv_original_size_buffers[layer]}
            return
        for layer in self.send_original_idx_buffers:
            self.train_send_buffers_cpu[layer] = {}
            for pid, sizes in send_sizes[layer].items():
                qt = sum(s[0] for s in sizes.values())
                fp = sum(s[1] for s in sizes.values())
                self.train_send_buffers_cpu[layer][pid] = (_pin(torch.zeros(qt, dtype=torch.int8)),
                                                           _pin(torch.zeros((2, fp), dtype=torch.bfloat16)))
            self.train_recv_buffers_cpu[layer] = {}
            self.train_recv_buffers_gpu[layer] = {}
            for pid, sizes in self.recv_original_size_buffers[layer].items():
                qt = sum(s[0] for s in sizes.values())
                fp = sum(s[1] for s in sizes.values())
                self.train_recv_buffers_cpu[layer][pid] = (_pin(torch.zeros(qt, dtype=torch.int8)),
                                                           _pin(torch.zeros((2, fp), dtype=torch.bfloat16)))
                self.train_recv_buffers_gpu[layer][pid] = (torch.zeros(qt, dtype=torch.int8, device=self.device),
                                                           torch.zeros((2, fp), dtype=torch.bfloat16, device=self.device))

    # ---- delete / update (buffer.py:80-146,255-264) -------------------------------------------
    def _delete_train_buffer(self):
        for d in (self.send_original_idx_buffers, self.recv_original_idx_buffers, self.recv_original_size_buffers,
                  self.train_recv_buffers_cpu, self.train_recv_buffers_gpu, self.train_send_buffers_cpu):
            d.clear()

    def _delete_test_buffer(self):
        self.test_recv_buffers_cpu, self.test_recv_buffers_gpu, self.test_send_buffers_cpu = [], [], []

    def _delete(self):
        self._delete_test_buffer()
        self._delete_train_buffer()
        if self.p2p is not None:
            if self.device.type == "cuda":
                torch.cuda.synchronize(self.device)
            if dist.is_initialized():
                dist.barrier()          # nobody may still be storing into a slab that is freed
            self.p2p.close()
            self.p2p = None
        if torch.cuda.is_available():
            torch.cuda.empty_cache()
        logger.info(f"<worker{dist.get_rank() if dist.is_initialized() else 0} buffer delete done.>")

    def _update(self, *args, **kwargs):
        if self.bit_type == BitType.FULL:
            return
        self._delete_train_buffer()
        self._generate_train_buffer(*args, **kwargs)
        logger.info(f"<worker {dist.get_rank()} buffer update done>")

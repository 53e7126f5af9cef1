"""Assigner: per-row bit-width assignment for the quantised boundary exchange.

Scheme interface of AdaQP/assigner/assigner.py:22-80 kept: constructor arguments,
`get_assignment(send_idx, runtime_scheme=None) -> {layer_key: {peer: int32[rows]}}` with
values in BITS_SET, the `uniform` / `random` / `adaptive` schemes, `is_tracing`,
`traced_layer_data`, `assign_cycle`, class attribute `ctx`.  The adaptive scheme gathers
the per-channel variance / byte matrices on rank 0 as the reference does (:214-292) but
solves each layer with the exact structured solver of assigner/solver.py instead of
PuLP + Gurobi/CBC.
"""
from __future__ import annotations

import logging
import time
from itertools import chain
from typing import Dict, Tuple, Union

import numpy as np
import torch
from torch import Tensor

from ..communicator import BITS_SET
from ..communicator import Communicator as comm
from ..communicator.p2p import layer_key_dims, quantisable
from ..helper import BitType
from ..manager import GraphEngine as engine
from . import solver
from .profile import fit_cost_model, generate_cost_model_dataset

logger = logging.getLogger("trainer")

ASSIGNMENT_SCHEME = ("uniform", "random", "adaptive")


class Assigner(object):
    ctx: "Assigner" = None

    def __init__(self, feat_dim: int, hidden_dim: int, num_layers: int, num_data: int, scheme: str,
                 uniform_assign_bits: int, scores: Dict[int, Tuple[Tensor, Tensor]], group_size: int,
                 coe_lambda: float, assign_cycle: int = None, warmup: int = 1, key_dims: Dict[str, int] = None):
        assert scheme in ASSIGNMENT_SCHEME, f"assignment scheme {scheme} is not supported"
        # keys that travel quantised and their row widths: by default the reference's forward0..L-1 / backward1..L-1
        # with layer 0 feat_dim wide; a model with its own exchange (GAT) passes every key's real width
        if key_dims is None:
            key_dims = layer_key_dims([feat_dim] + [hidden_dim] * (num_layers - 1))
        self.key_dims = {k: int(v) for k, v in key_dims.items() if quantisable(k)}
        self.keys = list(self.key_dims)
        self.bits_set = torch.tensor(BITS_SET, dtype=torch.int32)
        self.bits_cost = torch.tensor([1 / (2 ** b - 1) ** 2 for b in BITS_SET], dtype=torch.float32)
        self.feat_dim, self.hidden_dim, self.num_layers = feat_dim, hidden_dim, num_layers
        self.num_data, self.warmup = num_data, warmup
        self._scheme = scheme
        self._scheme_map = {"uniform": self._get_uniform_assignment,
                            "random": self._get_random_sampling_assignment,
                            "adaptive": self._get_adaptive_assignment}
        self.uniform_assign_bits = uniform_assign_bits
        self.scores, self.group_size, self.coe_lambda = scores, group_size, coe_lambda
        self.assign_cycle = assign_cycle
        self.cost_model = None
        self.sample_rate = torch.full((len(BITS_SET),), 1.0 / len(BITS_SET))
        self.is_tracing = False
        self.traced_layer_data: Dict[str, Union[float, Tensor, Dict[int, Tensor]]] = {}
        self.group_idx: Dict[str, Dict[int, Tuple[Tensor, ...]]] = {}
        self.last_solve_seconds: Dict[str, float] = {}
        self.assignment: Dict[str, Dict[int, Tensor]] = None     # the last get_assignment() result (checkpoints)
        if scheme == "adaptive" and engine.ctx.bit_type == BitType.QUANT:
            self._init_adaptive()
        Assigner.ctx = self

    def _init_adaptive(self):
        logger.info(f"<worker {comm.get_rank()} preprocessing for adaptive bit-width assignment...>")
        self.cost_model = fit_cost_model(generate_cost_model_dataset(self.feat_dim, self.hidden_dim,
                                                                     self.num_data, self.warmup))
        self.is_tracing = True
        self.init_traced_data(self.num_layers)

    def __repr__(self):
        return f"<Assigner(rank: {comm.get_rank()}, default scheme={self._scheme})>"

    @property
    def scheme(self):
        return self._scheme

    def get_assignment(self, send_idx: Dict[int, Tuple[int, int]], runtime_scheme: str = None):
        scheme = self._scheme if runtime_scheme is None else runtime_scheme
        assert scheme in ASSIGNMENT_SCHEME, f"assignment scheme {scheme} is not supported"
        self.assignment = self._scheme_map[scheme](send_idx)
        return self.assignment

    # ---- checkpoint state (trainer/checkpoint.py) -------------------------------------------------
    def state_dict(self) -> dict:
        """Everything a resumed run needs to draw the same assignments as a run that never stopped: the current
        assignment, the traced variances accumulated since the last re-assignment (moved to the CPU), the fitted
        cost model (timed, so a fresh process would fit a different one), `is_tracing` and `sample_rate`.  Plain
        tensors, dicts and scalars only, so that `torch.load(..., weights_only=True)` reads it back."""
        def traced(v):
            return v.detach().cpu().clone() if isinstance(v, Tensor) else float(v)
        return {"scheme": self._scheme,
                "assignment": None if self.assignment is None else
                {k: {int(p): torch.as_tensor(b, dtype=torch.int32).cpu().clone() for p, b in per.items()}
                 for k, per in self.assignment.items()},
                "traced_layer_data": {k: traced(v) for k, v in self.traced_layer_data.items()},
                "cost_model": None if self.cost_model is None else
                {k: torch.from_numpy(np.array(v, np.float64)) for k, v in self.cost_model.items()},
                "is_tracing": bool(self.is_tracing),
                "sample_rate": self.sample_rate.clone()}

    def load_state_dict(self, state: dict, device: torch.device = None):
        """Inverse of state_dict(); traced accumulators go to `device` (default: the communicator's device)."""
        if state["scheme"] != self._scheme:
            raise ValueError(f"assigner state of scheme {state['scheme']!r} cannot be loaded into scheme {self._scheme!r}")
        if device is None:
            device = comm.ctx.device if comm.ctx is not None else torch.device("cpu")
        self.assignment = None if state["assignment"] is None else \
            {k: {int(p): b.clone() for p, b in per.items()} for k, per in state["assignment"].items()}
        self.traced_layer_data = {k: (v.to(device) if isinstance(v, Tensor) else float(v))
                                  for k, v in state["traced_layer_data"].items()}
        self.cost_model = None if state["cost_model"] is None else \
            {k: v.numpy().copy() for k, v in state["cost_model"].items()}
        self.is_tracing = bool(state["is_tracing"])
        self.sample_rate = state["sample_rate"].clone()

    # ---- simple schemes (:95-120) ------------------------------------------------------------
    def _get_uniform_assignment(self, send_idx):
        return {key: {pid: torch.full((hi - lo,), self.uniform_assign_bits, dtype=torch.int32)
                      for pid, (lo, hi) in send_idx.items()} for key in self.keys}

    def _get_random_sampling_assignment(self, send_idx):
        out = {}
        for key in self.keys:
            out[key] = {}
            for pid, (lo, hi) in send_idx.items():
                pick = torch.multinomial(self.sample_rate, hi - lo, replacement=True)
                out[key][pid] = self.bits_set[pick]
        return out

    # ---- adaptive scheme (:128-304) -------------------------------------------------------------
    def init_traced_data(self, num_layers: int):
        for key in self.keys:
            self.traced_layer_data[key] = 0.0

    def slice_traced_data(self, send_idx):
        sliced = {}
        for key, data in self.traced_layer_data.items():
            data = data.cpu() if isinstance(data, Tensor) else torch.zeros(max(hi for _, hi in send_idx.values()))
            sliced[key] = {pid: data[lo:hi] for pid, (lo, hi) in send_idx.items()}
        self.traced_layer_data = sliced

    def config_score_matrix(self, scores, group_size: int, feats_dim: int, hidden_dim: int):
        """Variance matrix [3 bits x G groups] and MB matrix per channel (:162-212): rows
        sorted by agg_score^2 * traced variance, chunked into groups of `group_size`."""
        rank = comm.get_rank()
        var_matrix, comm_matrix, idx_set = {}, {}, {}
        for key, per_peer in self.traced_layer_data.items():
            var_matrix[key], comm_matrix[key], idx_set[key] = {}, {}, {}
            dim = self.key_dims[key]
            for pid, traced in per_peer.items():
                agg = scores[pid][0] if "forward" in key else scores[pid][1]
                assert agg.shape == traced.shape
                combined = (agg ** 2) * traced
                srt, order = torch.sort(combined, descending=True)
                g_ids = torch.split(order, group_size)
                # reference expression, kept verbatim for parity (assigner.py:167-171 `group_data`): the SORTED
                # scores indexed by the group's ORIGINAL row ids, i.e. not the sum of the group's own scores
                g_var = torch.stack([srt[ids].sum() for ids in g_ids])
                var_matrix[key][f"{rank}_{pid}"] = (self.bits_cost.view(-1, 1) * g_var.view(1, -1)).numpy()
                idx_set[key][pid] = g_ids
                mb = (self.bits_set.view(-1, 1).float() * dim * group_size) / 8 / (1024 ** 2)
                comm_matrix[key][f"{rank}_{pid}"] = mb.repeat(1, len(g_ids)).numpy()
        self.group_idx = idx_set
        return var_matrix, comm_matrix

    def aggregate_params_get_solution(self, var_matrix, comm_matrix, coe_lambda: float):
        """Gather every rank's matrices on rank 0, solve per layer, scatter (:214-292)."""
        rank, W = comm.get_rank(), comm.get_world_size()
        params_list = [None] * W
        comm.gather_any([var_matrix, comm_matrix, self.cost_model], params_list if rank == 0 else None, dst=0)
        if rank != 0:
            per_rank = [None] * W
        else:
            model = dict(chain(*[p[2].items() for p in params_list]))
            layer_assign = {}
            for key in var_matrix:
                v = dict(chain(*[p[0][key].items() for p in params_list]))
                c = dict(chain(*[p[1][key].items() for p in params_list]))
                t0 = time.time()
                # 'p2p': one send launch per rank writes all peers (max over ranks); 'gloo': the reference's ring rounds
                schedule = "concurrent" if comm.ctx.transport == "p2p" else "ring"
                layer_assign[key], _ = solver.solve_layer(v, c, model, coe_lambda, W, schedule=schedule)
                self.last_solve_seconds[key] = time.time() - t0
                logger.info(f"layer {key} solving time: {self.last_solve_seconds[key]:.4f}s")
            per_rank = []
            for sender in range(W):
                mine = {}
                for key, chans in layer_assign.items():
                    mine[key] = {int(c.split("_")[1]): torch.from_numpy(b) for c, b in chans.items()
                                 if int(c.split("_")[0]) == sender}
                per_rank.append(mine)
        comm.barrier()
        out = [None]
        comm.scatter_any(out, per_rank, src=0)
        return out[0]

    def recover_assignment_from_group(self, group_assignments):
        result = {}
        for key, per_peer in self.traced_layer_data.items():
            result[key] = {}
            for pid, traced in per_peer.items():
                bits = torch.zeros(traced.shape[0], dtype=torch.int32)
                for ids, b in zip(self.group_idx[key][pid], group_assignments[key][pid]):
                    bits[ids] = b
                result[key][pid] = bits
        return result

    def _get_adaptive_assignment(self, send_idx):
        self.slice_traced_data(send_idx)
        var_matrix, comm_matrix = self.config_score_matrix(self.scores, self.group_size, self.feat_dim, self.hidden_dim)
        groups = self.aggregate_params_get_solution(var_matrix, comm_matrix, self.coe_lambda)
        result = self.recover_assignment_from_group(groups)
        self.traced_layer_data = {key: 0.0 for key in self.traced_layer_data}
        self.group_idx.clear()
        return result

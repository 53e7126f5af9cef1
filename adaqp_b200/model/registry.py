"""The model table: everything the Trainer, the checkpoints and the exchange set-up need to know about a model, keyed by
`--model_name`.  Each entry is a set of plain functions of the Trainer's resolved config (the yaml's `data`, `model` and
`runtime` sections with the run-time overrides applied).  Adding a model is one entry here plus its module, ops and
kernels."""
from __future__ import annotations

from dataclasses import dataclass
from typing import Callable, Dict, List, Optional

import torch
import torch.nn as nn

from .. import gatv2, sage_pool
from ..communicator.p2p import appnp_key_dims, gat_key_dims, gatv2_key_dims, sage_pool_key_dims
from ..helper import DistGNNType
from .distAPPNP import DistAPPNP, appnp_params
from .distGAT import DistGAT, gat_layer_shapes
from .distGATv2 import DistGATv2
from .distGCN import DistGCN
from .distGCNII import DistGCNII, gcnii_params
from .distSAGE import DistSAGE
from .ops import _full


def _none(*_) -> None:
    return None


@dataclass(frozen=True)
class ModelSpec:
    kind: DistGNNType
    build: Callable[[dict], nn.Module]                                 # the model, on the CPU
    check: Callable[[dict], object] = _none                           # raises ValueError on bad model parameters
    p2p_only: Callable[[dict], Optional[str]] = _none                 # why the gloo transport is refused (None: it is not)
    key_dims: Callable[[dict], Optional[Dict[str, int]]] = _none      # its own exchange keys and widths (None: the reference's)
    propagation: Callable[[dict], Optional[dict]] = _none             # the checkpoint manifest's `propagation` field
    setup: Callable[[object, object], None] = _none                   # (engine ctx, PeerExchange) once the buffers exist


def layer_widths(config: dict) -> List[int]:
    """The input width of every layer of the reference models: num_feats, then hidden_dim."""
    data, model = config["data"], config["model"]
    return [data["num_feats"]] + [model["hidden_dim"]] * (model["num_layers"] - 1)


def buffer_shape(config: dict, key_dims: Optional[Dict[str, int]]) -> List[int]:
    """The widths of the fp32 test{l} buffers: those of a model's own key table, else layer_widths."""
    if key_dims is None:
        return layer_widths(config)
    return [key_dims[f"test{i}"] for i in range(sum(k.startswith("test") for k in key_dims))]


def _common(config: dict) -> tuple:
    data, model = config["data"], config["model"]
    return (data["num_feats"], model["hidden_dim"], data["num_classes"], model["num_layers"], model["dropout_rate"],
            model["use_norm"])


def _gat_shapes(config: dict):
    data, model = config["data"], config["model"]
    return gat_layer_shapes(model["hidden_dim"], data["num_classes"], model["num_layers"], model["gat_heads"])


def _model_p2p_only(config: dict) -> str:
    return (f"model '{config['runtime']['model_name']}' runs on the p2p transport only; the CPU gloo plumbing mode "
            "(ADAQP_DEVICE=cpu / ADAQP_TRANSPORT=gloo) supports gcn and sage")


def _is_pool(config: dict) -> bool:
    return config["model"]["aggregator_type"] == "pool"


def _pool_p2p_only(config: dict) -> Optional[str]:
    if not _is_pool(config):
        return None
    return ("aggregator_type 'pool' runs on the p2p transport only; the CPU gloo plumbing mode "
            "(ADAQP_DEVICE=cpu / ADAQP_TRANSPORT=gloo) supports the mean and gcn aggregators")


def _sage_setup(eng, ex):
    """The backward match table of the max-pool aggregation, aligned with the CSR the kernels read; the peers'
    recv_idx come from the exchange's set-up all-gather."""
    if eng.agg_type != "pool":
        return
    g = _full(eng.graph)
    want = sage_pool.pool_want(g.indptr.cpu().numpy(), g.indices.cpu().numpy(), g.n_inner, ex.recv_idx,
                               ex.send_idx, ex.total_send_idx, ex.peer_recv_idx)
    eng.pool_want = torch.from_numpy(want).to(g.device)


def _gatv2_setup(eng, ex):
    """GATv2's backward tables, aligned with the CSR the kernels read: the halo-transposed CSR (the inner
    destinations of every halo row) and the fold table (the push-region rows of every inner row)."""
    g = _full(eng.graph)
    hp, hd = gatv2.halo_table(g.indptr.cpu().numpy(), g.indices.cpu().numpy(), g.n_inner, ex.num_remote)
    fp, fpos = gatv2.fold_table(g.n_inner, ex.send_peers, ex.send_idx, ex.total_send_idx)
    eng.gatv2_halo = tuple(torch.from_numpy(a).to(g.device) for a in (hp, hd))
    eng.gatv2_fold = tuple(torch.from_numpy(a).to(g.device) for a in (fp, fpos))


# 'gat', 'gatv2', 'appnp', 'gcnii' and SAGE's 'pool' aggregator are extensions beyond the reference's two models
MODELS: Dict[str, ModelSpec] = {
    "gcn": ModelSpec(DistGNNType.DistGCN, build=lambda c: DistGCN(*_common(c))),
    "sage": ModelSpec(
        DistGNNType.DistSAGE,
        build=lambda c: DistSAGE(*_common(c), c["model"]["aggregator_type"]),
        p2p_only=_pool_p2p_only,
        # max-pool exchanges the pooled rows p of every layer (plus backward0 and the arg rows)
        key_dims=lambda c: sage_pool_key_dims(layer_widths(c)) if _is_pool(c) else None,
        setup=_sage_setup),
    "gat": ModelSpec(
        DistGNNType.DistGAT,
        build=lambda c: DistGAT(*_common(c), heads=c["model"]["gat_heads"]),
        check=_gat_shapes, p2p_only=_model_p2p_only,
        # the projected rows z of every layer (plus backward0 and the attention scalars)
        key_dims=lambda c: gat_key_dims(*_gat_shapes(c))),
    "gatv2": ModelSpec(
        DistGNNType.DistGATv2,
        build=lambda c: DistGATv2(*_common(c), heads=c["model"]["gat_heads"]),
        check=_gat_shapes, p2p_only=_model_p2p_only,
        # the source projection zs of every layer, and its halo gradients pushed back
        key_dims=lambda c: gatv2_key_dims(_gat_shapes(c)[0]),
        setup=_gatv2_setup),
    "appnp": ModelSpec(
        DistGNNType.DistAPPNP,
        build=lambda c: DistAPPNP(*_common(c), k=c["model"]["appnp_k"], alpha=c["model"]["appnp_alpha"]),
        check=lambda c: appnp_params(c["model"]["appnp_k"], c["model"]["appnp_alpha"]),
        p2p_only=_model_p2p_only,
        # num_classes-wide rows at each of its K steps
        key_dims=lambda c: appnp_key_dims(c["data"]["num_classes"], int(c["model"]["appnp_k"])),
        propagation=lambda c: {"k": int(c["model"]["appnp_k"]), "alpha": float(c["model"]["appnp_alpha"])}),
    "gcnii": ModelSpec(
        DistGNNType.DistGCNII,
        build=lambda c: DistGCNII(c["data"]["num_feats"], c["model"]["hidden_dim"], c["data"]["num_classes"],
                                  c["model"]["dropout_rate"], layers=c["model"]["gcnii_layers"],
                                  alpha=c["model"]["gcnii_alpha"], theta=c["model"]["gcnii_theta"]),
        check=lambda c: gcnii_params(c["model"]["gcnii_layers"], c["model"]["gcnii_alpha"], c["model"]["gcnii_theta"]),
        p2p_only=_model_p2p_only,
        # APPNP's key table, hidden_dim wide, one step per layer
        key_dims=lambda c: appnp_key_dims(c["model"]["hidden_dim"], int(c["model"]["gcnii_layers"])),
        propagation=lambda c: {"layers": int(c["model"]["gcnii_layers"]), "alpha": float(c["model"]["gcnii_alpha"]),
                               "theta": float(c["model"]["gcnii_theta"])}),
}

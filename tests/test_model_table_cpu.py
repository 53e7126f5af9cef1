"""The model table (adaqp_b200/model/registry.py), entry by entry, against literal expectations: the exchange key table
CommBuffer / PeerExchange are given, the test-buffer shape, the Assigner's keys with their order and widths, the
checkpoint manifest's run fields and the model's parameter names and shapes.  The values were recorded from the
Trainer before the table existed, when each of them was its own per-model branch; checkpoints written then must still
resume and load, so none of them may change."""
import pytest
import torch

from adaqp_b200.assigner import Assigner
from adaqp_b200.communicator.p2p import PeerExchange, quantisable
from adaqp_b200.helper import DistGNNType
from adaqp_b200.model.registry import MODELS, buffer_shape
from adaqp_b200.trainer import checkpoint as ckpt


def _cfg(model_name, agg="mean", num_layers=3, hidden_dim=64, gat_heads=4, appnp_k=10, gcnii_theta=0.5):
    return {"data": {"num_feats": 100, "num_classes": 47},
            "model": {"num_layers": num_layers, "hidden_dim": hidden_dim, "aggregator_type": agg, "gat_heads": gat_heads,
                      "dropout_rate": 0.5, "use_norm": True, "appnp_k": appnp_k, "appnp_alpha": 0.1, "gcnii_layers": 8,
                      "gcnii_alpha": 0.1, "gcnii_theta": gcnii_theta},
            "runtime": {"dataset": "ogbn-products", "model_name": model_name, "num_parts": 2, "mode": "AdaQP",
                        "assign_scheme": "uniform"}}


def _assigner(num_layers, hidden_dim, key_dims=None):
    return Assigner(100, hidden_dim, num_layers, 10, "uniform", 8, {}, 100, 0.5, 50, key_dims=key_dims)


# (model_name, aggregator_type) -> what the Trainer builds for _cfg(model_name, aggregator_type)
EXPECTED = {
    ("gcn", "mean"): {
        "key_dims": None,
        "shape": [100, 64, 64],
        "assigner": [("forward0", 100), ("forward1", 64), ("forward2", 64), ("backward1", 64), ("backward2", 64)],
        "propagation": None,
        "params": ("convs.0.weight:100x64 convs.0.bias:64 convs.1.weight:64x64 convs.1.bias:64 convs.2.weight:64x47 "
                   "convs.2.bias:47 norms.0.weight:64 norms.0.bias:64 norms.1.weight:64 norms.1.bias:64"),
    },
    ("sage", "mean"): {
        "key_dims": None,
        "shape": [100, 64, 64],
        "assigner": [("forward0", 100), ("forward1", 64), ("forward2", 64), ("backward1", 64), ("backward2", 64)],
        "propagation": None,
        "params": ("sages.0.bias:64 sages.0.fc_self.weight:64x100 sages.0.fc_neigh.weight:64x100 sages.1.bias:64 "
                   "sages.1.fc_self.weight:64x64 sages.1.fc_neigh.weight:64x64 sages.2.bias:47 "
                   "sages.2.fc_self.weight:47x64 sages.2.fc_neigh.weight:47x64 norms.0.weight:64 norms.0.bias:64 "
                   "norms.1.weight:64 norms.1.bias:64"),
    },
    ("sage", "gcn"): {
        "key_dims": None,
        "shape": [100, 64, 64],
        "assigner": [("forward0", 100), ("forward1", 64), ("forward2", 64), ("backward1", 64), ("backward2", 64)],
        "propagation": None,
        "params": ("sages.0.bias:64 sages.0.fc_neigh.weight:64x100 sages.1.bias:64 sages.1.fc_neigh.weight:64x64 "
                   "sages.2.bias:47 sages.2.fc_neigh.weight:47x64 norms.0.weight:64 norms.0.bias:64 "
                   "norms.1.weight:64 norms.1.bias:64"),
    },
    ("sage", "pool"): {
        "key_dims": {"test0": 100, "test1": 64, "test2": 64, "forward0": 100, "forward1": 64, "forward2": 64,
                     "backward0": 100, "backward1": 64, "backward2": 64, "pool_arg0": 100,
                     "pool_arg1": 64, "pool_arg2": 64},
        "shape": [100, 64, 64],
        "assigner": [("forward0", 100), ("forward1", 64), ("forward2", 64), ("backward0", 100), ("backward1", 64),
                     ("backward2", 64)],
        "propagation": None,
        "params": ("sages.0.bias:64 sages.0.fc_pool.weight:100x100 sages.0.fc_pool.bias:100 "
                   "sages.0.fc_self.weight:64x100 sages.0.fc_neigh.weight:64x100 sages.1.bias:64 "
                   "sages.1.fc_pool.weight:64x64 sages.1.fc_pool.bias:64 sages.1.fc_self.weight:64x64 "
                   "sages.1.fc_neigh.weight:64x64 sages.2.bias:47 sages.2.fc_pool.weight:64x64 "
                   "sages.2.fc_pool.bias:64 sages.2.fc_self.weight:47x64 sages.2.fc_neigh.weight:47x64 "
                   "norms.0.weight:64 norms.0.bias:64 norms.1.weight:64 norms.1.bias:64"),
    },
    ("gat", "mean"): {
        "key_dims": {"test0": 64, "test1": 64, "test2": 47, "forward0": 64, "forward1": 64, "forward2": 47,
                     "backward0": 64, "backward1": 64, "backward2": 47, "attn_fwd0": 4,
                     "attn_bwd0": 12, "attn_fwd1": 4, "attn_bwd1": 12, "attn_fwd2": 1,
                     "attn_bwd2": 3},
        "shape": [64, 64, 47],
        "assigner": [("forward0", 64), ("forward1", 64), ("forward2", 47), ("backward0", 64), ("backward1", 64),
                     ("backward2", 47)],
        "propagation": None,
        "params": ("convs.0.weight:100x64 convs.0.attn_l:4x16 convs.0.attn_r:4x16 convs.0.bias:64 "
                   "convs.1.weight:64x64 convs.1.attn_l:4x16 convs.1.attn_r:4x16 convs.1.bias:64 "
                   "convs.2.weight:64x47 convs.2.attn_l:1x47 convs.2.attn_r:1x47 convs.2.bias:47 norms.0.weight:64 "
                   "norms.0.bias:64 norms.1.weight:64 norms.1.bias:64"),
    },
    ("gatv2", "mean"): {
        "key_dims": {"test0": 64, "test1": 64, "test2": 47, "forward0": 64, "forward1": 64, "forward2": 47,
                     "push0": 64, "push1": 64, "push2": 47},
        "shape": [64, 64, 47],
        "assigner": [("forward0", 64), ("forward1", 64), ("forward2", 47)],
        "propagation": None,
        "params": ("convs.0.W_s:100x64 convs.0.b_s:64 convs.0.W_d:100x64 convs.0.b_d:64 convs.0.attn:4x16 "
                   "convs.1.W_s:64x64 convs.1.b_s:64 convs.1.W_d:64x64 convs.1.b_d:64 convs.1.attn:4x16 "
                   "convs.2.W_s:64x47 convs.2.b_s:47 convs.2.W_d:64x47 convs.2.b_d:47 convs.2.attn:1x47 "
                   "norms.0.weight:64 norms.0.bias:64 norms.1.weight:64 norms.1.bias:64"),
    },
    ("appnp", "mean"): {
        "key_dims": {"test0": 47, "test1": 47, "test2": 47, "test3": 47, "test4": 47, "test5": 47, "test6": 47,
                     "test7": 47, "test8": 47, "test9": 47, "forward0": 47, "forward1": 47,
                     "forward2": 47, "forward3": 47, "forward4": 47, "forward5": 47,
                     "forward6": 47, "forward7": 47, "forward8": 47, "forward9": 47,
                     "backward0": 47, "backward1": 47, "backward2": 47, "backward3": 47,
                     "backward4": 47, "backward5": 47, "backward6": 47, "backward7": 47,
                     "backward8": 47, "backward9": 47},
        "shape": [47, 47, 47, 47, 47, 47, 47, 47, 47, 47],
        "assigner": [("forward0", 47), ("forward1", 47), ("forward2", 47), ("forward3", 47), ("forward4", 47),
                     ("forward5", 47), ("forward6", 47), ("forward7", 47), ("forward8", 47),
                     ("forward9", 47), ("backward0", 47), ("backward1", 47), ("backward2", 47),
                     ("backward3", 47), ("backward4", 47), ("backward5", 47), ("backward6", 47),
                     ("backward7", 47), ("backward8", 47), ("backward9", 47)],
        "propagation": {"k": 10, "alpha": 0.1},
        "params": ("lins.0.weight:100x64 lins.0.bias:64 lins.1.weight:64x64 lins.1.bias:64 lins.2.weight:64x47 "
                   "lins.2.bias:47 norms.0.weight:64 norms.0.bias:64 norms.1.weight:64 norms.1.bias:64"),
    },
    ("gcnii", "mean"): {
        "key_dims": {"test0": 64, "test1": 64, "test2": 64, "test3": 64, "test4": 64, "test5": 64, "test6": 64,
                     "test7": 64, "forward0": 64, "forward1": 64, "forward2": 64, "forward3": 64,
                     "forward4": 64, "forward5": 64, "forward6": 64, "forward7": 64,
                     "backward0": 64, "backward1": 64, "backward2": 64, "backward3": 64,
                     "backward4": 64, "backward5": 64, "backward6": 64, "backward7": 64},
        "shape": [64, 64, 64, 64, 64, 64, 64, 64],
        "assigner": [("forward0", 64), ("forward1", 64), ("forward2", 64), ("forward3", 64), ("forward4", 64),
                     ("forward5", 64), ("forward6", 64), ("forward7", 64), ("backward0", 64),
                     ("backward1", 64), ("backward2", 64), ("backward3", 64), ("backward4", 64),
                     ("backward5", 64), ("backward6", 64), ("backward7", 64)],
        "propagation": {"layers": 8, "alpha": 0.1, "theta": 0.5},
        "params": ("lins.0.weight:100x64 lins.0.bias:64 lins.1.weight:64x47 lins.1.bias:47 convs.0.weight:64x64 "
                   "convs.1.weight:64x64 convs.2.weight:64x64 convs.3.weight:64x64 convs.4.weight:64x64 "
                   "convs.5.weight:64x64 convs.6.weight:64x64 convs.7.weight:64x64"),
    },
}


@pytest.mark.parametrize("name,agg", list(EXPECTED))
def test_model_table(name, agg):
    cfg, want = _cfg(name, agg), EXPECTED[(name, agg)]
    key_dims = MODELS[name].key_dims(cfg)
    assert key_dims == want["key_dims"]
    if key_dims is not None:
        assert list(key_dims) == list(want["key_dims"])             # the exchange's key order is its slab layout
    assert buffer_shape(cfg, key_dims) == want["shape"]
    assert list(_assigner(3, 64, key_dims).key_dims.items()) == want["assigner"]
    # the manifest records a model's own table whole, and the reference's as the Assigner's keys
    manifest_keys = want["key_dims"] if want["key_dims"] is not None else dict(want["assigner"])
    assert ckpt.run_fields(cfg, key_dims) == {
        "dataset": "ogbn-products", "model_name": name, "aggregator_type": agg, "gat_heads": 4,
        "layer_dims": [100, 64, 64, 47], "num_parts": 2, "mode": "AdaQP", "assign_scheme": "uniform",
        "key_dims": manifest_keys, "propagation": want["propagation"]}
    model = MODELS[name].build(cfg)
    got = " ".join(f"{k}:{'x'.join(map(str, v.shape))}" for k, v in model.state_dict().items())
    assert got == want["params"]


def test_kinds():
    assert {name: spec.kind for name, spec in MODELS.items()} == {
        "gcn": DistGNNType.DistGCN, "sage": DistGNNType.DistSAGE, "gat": DistGNNType.DistGAT,
        "gatv2": DistGNNType.DistGATv2, "appnp": DistGNNType.DistAPPNP, "gcnii": DistGNNType.DistGCNII}


def test_checks_and_transport_refusals():
    for name, agg in EXPECTED:
        MODELS[name].check(_cfg(name, agg))
    for name, bad in (("gat", {"gat_heads": 3}), ("gatv2", {"gat_heads": 3}), ("appnp", {"appnp_k": 0}),
                      ("gcnii", {"gcnii_theta": 0})):
        with pytest.raises(ValueError):
            MODELS[name].check(_cfg(name, **bad))
    refusals = {(name, agg): MODELS[name].p2p_only(_cfg(name, agg)) for name, agg in EXPECTED}
    gloo = "the CPU gloo plumbing mode (ADAQP_DEVICE=cpu / ADAQP_TRANSPORT=gloo) supports"
    assert refusals == {
        ("gcn", "mean"): None, ("sage", "mean"): None, ("sage", "gcn"): None,
        ("sage", "pool"): f"aggregator_type 'pool' runs on the p2p transport only; {gloo} the mean and gcn aggregators",
        ("gat", "mean"): f"model 'gat' runs on the p2p transport only; {gloo} gcn and sage",
        ("gatv2", "mean"): f"model 'gatv2' runs on the p2p transport only; {gloo} gcn and sage",
        ("appnp", "mean"): f"model 'appnp' runs on the p2p transport only; {gloo} gcn and sage",
        ("gcnii", "mean"): f"model 'gcnii' runs on the p2p transport only; {gloo} gcn and sage"}


def test_reference_keys_from_layer_ten_on():
    """From 11 layers on the keys have two-digit layer numbers: forward10 / backward10 are hidden_dim wide in the
    Assigner, the manifest and the exchange alike."""
    cfg = _cfg("gcn", num_layers=11, hidden_dim=256)
    shape = [100] + [256] * 10
    ex = PeerExchange(0, 1, "cpu", shape, {}, {}, torch.zeros(0, dtype=torch.int64), 0)
    exchange = {k: d for k, d in ex.dims.items() if quantisable(k)}
    assigner = _assigner(11, 256).key_dims
    assert list(assigner.items()) == list(exchange.items())
    assert ckpt.run_fields(cfg, None)["key_dims"] == exchange
    assert exchange["forward0"] == 100 and exchange["forward10"] == exchange["backward10"] == 256

"""The GCN / GraphSAGE training-step check of tests/test_gpu_gnn_step.py on CPU/gloo (ADAQP_DEVICE=cpu), without a
GPU: two ranks, one step, logits, loss and every parameter gradient against the float64 model of the unpartitioned
graph, at the GPU test's bounds.  This checks the harness and the float64 model themselves, and the host
aggregation (manager/graph_cpu.spmm_cpu) with its self term and mean; where the GPU and CPU runs disagree, this one
tells whether the fault is in the reference or in the kernels.  The per-layer check reads the p2p receive slab, so
it runs on the GPU only."""
import pytest

from test_gpu_gnn_step import check_step, spawn


@pytest.mark.parametrize("model,agg", [("gcn", "mean"), ("sage", "gcn")])
@pytest.mark.parametrize("mode", ["Vanilla", "AdaQP-p"])
def test_two_rank_cpu_training_step(model, agg, mode):
    res = spawn(2, dict(model=model, agg=agg, mode=mode, device="cpu"), timeout=600)
    r = res[0]
    print(f"\n{model}-{agg} {mode} on CPU: logits {r['logit_err']:.3g} loss {r['loss_err']:.3g} "
          f"grad {max(r['grad_err'].values()):.3g} ({max(r['grad_err'], key=r['grad_err'].get)})")
    check_step(res, 2, fp32=True, layer_checked=False)

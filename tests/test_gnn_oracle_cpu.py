"""The GCN / GraphSAGE aggregation oracles (oracle/oracle.py) and the float64 torch layers (oracle/gnn_oracle.py)
against each other, without a GPU.

* sage_gcn_aggregation forward / backward equal a scipy-sparse float64 restatement of the reference formulas on a
  small symmetric graph with self-loops, an isolated node and halo columns;
* on a symmetric graph the backward oracles of GCN, SAGE mean and SAGE gcn equal the autograd gradient of the torch
  layers.  The distributed backward uses the reference's out-degree formulas, so this is what makes the float64
  model a valid arbiter of the distributed training step (tests/test_gpu_gnn_step.py).
"""
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import gnn_oracle as G  # noqa: E402
from oracle import oracle as O  # noqa: E402


def _symmetric(n, deg, seed, isolated=()):
    """CSR of a random symmetric graph on n nodes with every self-loop, except the `isolated` nodes, which have no
    edge at all."""
    rng = np.random.RandomState(seed)
    m = n * deg // 2
    a, b = rng.randint(0, n, m), rng.randint(0, n, m)
    keep = ~np.isin(a, isolated) & ~np.isin(b, isolated)
    a, b = a[keep], b[keep]
    loops = np.setdiff1d(np.arange(n), isolated)
    A = sp.coo_matrix((np.ones(2 * a.size + loops.size), (np.r_[a, b, loops], np.r_[b, a, loops])), shape=(n, n)).tocsr()
    A.data[:] = 1.0
    A.sort_indices()
    return A


def test_sage_gcn_aggregation_matches_scipy():
    """Rows 0..n_in-1 are a rank's inner nodes, columns >= n_in its halo; degrees are the global ones."""
    n, n_in, F = 400, 260, 23
    A = _symmetric(n, 6, seed=3, isolated=(7, 300))
    deg = np.asarray(A.sum(1)).ravel().astype(np.int64)          # symmetric: in-degree == out-degree
    assert deg[7] == 0 and deg[300] == 0
    local = A[:n_in]
    assert local[:, n_in:].nnz > 0                                # some rows read halo columns
    ip, ix = local.indptr.astype(np.int64), local.indices.astype(np.int64)
    rng = np.random.RandomState(0)
    x = rng.standard_normal((n, F)).astype(np.float32)
    x64 = x.astype(np.float64)
    norm = 1.0 / (np.maximum(deg, 1) + 1.0)
    want_f = (local @ x64 + x64[:n_in]) * norm[:n_in, None]
    want_b = local @ (x64 * norm[:, None]) + x64[:n_in] * norm[:n_in, None]
    got_f = O.sage_gcn_aggregation(ip, ix, x, deg, deg, n_in)
    got_b = O.sage_gcn_aggregation(ip, ix, x, deg, deg, n_in, backward=True)
    mass = np.abs(local) @ np.abs(x64) + np.abs(x64[:n_in])
    # the oracle rounds the norms (and in the backward each scaled row) to fp32, as the reference does
    assert np.all(np.abs(got_f - want_f) <= 2e-7 * mass * norm[:n_in, None])
    assert np.all(np.abs(got_b - want_b) <= 2e-7 * mass)
    # the isolated node: its own row over (0 + 1) -- the clamp, not a division by zero
    np.testing.assert_allclose(got_f[7], x64[7] / 2, rtol=1e-7)
    np.testing.assert_allclose(got_b[7], x64[7] / 2, rtol=1e-7)
    # the self term is really there, in both directions
    assert np.abs(got_f - (local @ x64) * norm[:n_in, None]).max() > 0.1
    assert np.abs(got_b - local @ (x64 * norm[:, None])).max() > 0.1


@pytest.mark.parametrize("kind", ["gcn", "sage_mean", "sage_gcn"])
def test_backward_oracle_is_the_autograd_gradient(kind):
    """d<g, layer(x)>/dx from float64 autograd == the backward aggregation oracle fed g W^T (plus g Ws for the
    self path of SAGE mean), on a symmetric graph with an isolated node."""
    n, F = 300, 12
    A = _symmetric(n, 5, seed=11, isolated=(5,))
    ip, ix = A.indptr.astype(np.int64), A.indices.astype(np.int64)
    deg = np.diff(ip)
    src = torch.from_numpy(ix)
    dst = torch.from_numpy(np.repeat(np.arange(n), deg))
    rng = np.random.RandomState(1)
    # fp32-representable inputs, identity W for the aggregation path so the oracle sees g exactly
    x = torch.tensor(rng.standard_normal((n, F)).astype(np.float32), dtype=torch.float64, requires_grad=True)
    g = rng.standard_normal((n, F)).astype(np.float32)
    eye = torch.eye(F, dtype=torch.float64)
    b = torch.zeros(F, dtype=torch.float64)
    Ws = torch.tensor(rng.standard_normal((F, F)), dtype=torch.float64)
    if kind == "gcn":
        y = G.torch_gcn_layer(src, dst, x, eye, b)
        fwd = O.gcn_aggregation(ip, ix, x.detach().numpy(), deg, deg, n)
        bwd = O.gcn_aggregation(ip, ix, g, deg, deg, n, backward=True)
    elif kind == "sage_mean":
        y = G.torch_sage_layer(src, dst, x, eye, b, Ws, "mean")
        fwd = O.sage_aggregation(ip, ix, x.detach().numpy(), deg, deg, n) + x.detach().numpy() @ Ws.numpy().T
        bwd = O.sage_aggregation(ip, ix, g, deg, deg, n, backward=True) + g.astype(np.float64) @ Ws.numpy()
    else:
        y = G.torch_sage_layer(src, dst, x, eye, b, None, "gcn")
        fwd = O.sage_gcn_aggregation(ip, ix, x.detach().numpy(), deg, deg, n)
        bwd = O.sage_gcn_aggregation(ip, ix, g, deg, deg, n, backward=True)
    (y * torch.from_numpy(g.astype(np.float64))).sum().backward()
    scale_f = np.abs(fwd).max()
    scale_b = np.abs(bwd).max()
    np.testing.assert_allclose(y.detach().numpy(), fwd, rtol=0, atol=1e-6 * scale_f)
    np.testing.assert_allclose(x.grad.numpy(), bwd, rtol=0, atol=1e-6 * scale_b)
    # the torch layers count the degrees on the edge list
    in_deg, out_deg = G.degrees(src, dst, n)
    assert np.array_equal(in_deg.numpy(), deg) and np.array_equal(out_deg.numpy(), deg)


def test_torch_layers_use_weights_as_stored():
    """GCN's W is [in, out] (x W); SAGE's fc weights are nn.Linear [out, in] (x W^T); gcn has no self path."""
    n, Fi, Fo = 50, 6, 4
    A = _symmetric(n, 3, seed=2)
    src = torch.from_numpy(A.indices.astype(np.int64))
    dst = torch.from_numpy(np.repeat(np.arange(n), np.diff(A.indptr)))
    rng = np.random.RandomState(4)
    x = torch.tensor(rng.standard_normal((n, Fi)))
    W = torch.tensor(rng.standard_normal((Fi, Fo)))
    Wn, Ws = torch.tensor(rng.standard_normal((Fo, Fi))), torch.tensor(rng.standard_normal((Fo, Fi)))
    b = torch.tensor(rng.standard_normal(Fo))
    deg = np.diff(A.indptr)
    xn = x.numpy()
    gcn = O.gcn_aggregation(A.indptr, A.indices, xn, deg, deg, n) @ W.numpy() + b.numpy()
    np.testing.assert_allclose(G.torch_gcn_layer(src, dst, x, W, b).numpy(), gcn, rtol=1e-6, atol=1e-6)
    mean = O.sage_aggregation(A.indptr, A.indices, xn, deg, deg, n) @ Wn.numpy().T + xn @ Ws.numpy().T + b.numpy()
    np.testing.assert_allclose(G.torch_sage_layer(src, dst, x, Wn, b, Ws, "mean").numpy(), mean, rtol=1e-6, atol=1e-6)
    sgcn = O.sage_gcn_aggregation(A.indptr, A.indices, xn, deg, deg, n) @ Wn.numpy().T + b.numpy()
    np.testing.assert_allclose(G.torch_sage_layer(src, dst, x, Wn, b, None, "gcn").numpy(), sgcn, rtol=1e-6, atol=1e-6)

"""Column-sliced aggregation (option spmm_slice_cols) is bitwise equal to the unsliced kernel.

Each forced slice width (64, 128, 52 -- which slices F = 100 as 52 + 48 -- and the automatic choice) is
compared with `spmm_slice_cols` = F (one slice: the unsliced spmm_csr_kernel) using torch.equal, for the
GCN forward / backward norms, SAGE mean and gcn (self term), central and marginal row ranges, the two-pass
local + halo (accumulate) form of the marginal rows, and a hub row of in-degree above 100 000.
Widths that do not divide into 16-byte slices (F = 47, 13) run the unsliced kernel."""
import contextlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

WIDTHS = [64, 128, 52, 0]   # 0 = automatic


def lib():
    from adaqp_b200 import build as b
    b.build()
    from adaqp_b200 import _lib
    return _lib


@contextlib.contextmanager
def slice_cols(w):
    _lib = lib()
    old = _lib.get_option("spmm_slice_cols")
    _lib.set_option("spmm_slice_cols", w)
    try:
        yield
    finally:
        _lib.set_option("spmm_slice_cols", old)


def layouts(W, n, deg, F, seed):
    lib()
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    spec = SynthSpec(name="t", num_nodes=n, num_edges=n * deg, num_parts=W, num_feats=F, num_classes=5,
                     cross_fraction=0.3 if W > 1 else 0.0, community_size=64, seed=seed)
    return prepare_all_in_process(spec)


def kinds(g):
    return {"gcn_fwd": dict(pre=g.norm["out_-0.5"], post=g.norm["in_-0.5"]),
            "gcn_bwd": dict(pre=g.norm["in_-0.5"], post=g.norm["out_-0.5"]),
            "sage_mean": dict(pre=None, post=None, mean=True),
            "sage_mean_bwd": dict(pre=g.norm["out_-1"], post=None),
            "sage_gcn": dict(pre=None, post=g.norm["in_+1_-1"], add_self=True)}


def all_outputs(g, L, xl, xh):
    """Every aggregation form the trainer uses, as one list of tensors."""
    from adaqp_b200.manager.graph import spmm
    outs = []
    for kw in kinds(g).values():
        outs.append(spmm(g, xl, xh, **kw))
        outs.append(spmm(g, xl, None, row_begin=0, row_end=L.n_central, **kw))
        outs.append(spmm(g, xl, xh, row_begin=L.n_central, row_end=L.n_inner, **kw))
        if L.n_halo:
            two = torch.empty(L.n_inner - L.n_central, xl.shape[1], device=xl.device)
            spmm(g, xl, None, row_begin=L.n_central, row_end=L.n_inner, out=two, part="local", **kw)
            spmm(g, xl, xh, row_begin=L.n_central, row_end=L.n_inner, out=two, part="halo", **kw)
            outs.append(two)
    torch.cuda.synchronize()
    return outs


@pytest.mark.parametrize("F", [256, 100, 200, 300, 47, 13])
@pytest.mark.parametrize("W", [1, 3])
def test_forced_and_automatic_slices_are_bitwise_unsliced(F, W):
    from adaqp_b200.manager.graph import LocalGraph
    dev = torch.device("cuda:0")
    L = layouts(W, 1500, 14, F, seed=F + W)[-1]
    g = LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, dev)
    gen = torch.Generator(device="cpu").manual_seed(F)
    xl = torch.randn(L.n_inner, F, generator=gen).to(dev)
    xh = torch.randn(L.n_halo, F, generator=gen).to(dev) if L.n_halo else None
    if W > 1:
        assert L.n_halo > 0 and 0 < L.n_central < L.n_inner
    with slice_cols(F):
        ref = all_outputs(g, L, xl, xh)
    for w in WIDTHS:
        with slice_cols(w):
            got = all_outputs(g, L, xl, xh)
        for i, (a, b) in enumerate(zip(got, ref)):
            assert torch.equal(a, b), (w, i)


def test_hub_row_and_strided_slices():
    """A destination row with 120 000 in-neighbours, on column views with row pitch > F."""
    from adaqp_b200.manager.graph import LocalGraph, spmm
    dev = torch.device("cuda:0")
    rng = np.random.RandomState(7)
    n_inner, n_halo, hub = 3000, 400, 17
    deg = rng.randint(0, 20, size=n_inner)
    deg[hub] = 120_000
    cols = [np.sort(rng.randint(0, n_inner + n_halo, size=d)).astype(np.int32) for d in deg]
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    indices = np.concatenate(cols).astype(np.int32)
    in_deg = deg.astype(np.int64)
    out_deg = np.bincount(indices, minlength=n_inner + n_halo)[:n_inner].astype(np.int64)
    g = LocalGraph(indptr, indices, in_deg, out_deg, n_inner, n_halo, dev)
    big = torch.randn(n_inner + n_halo, 300, device=dev)
    for lo, F in [(0, 256), (4, 256), (8, 100)]:
        xl, xh = big[:n_inner, lo:lo + F], big[n_inner:, lo:lo + F]
        for kw in kinds(g).values():
            with slice_cols(F):
                ref = spmm(g, xl, xh, **kw)
            for w in WIDTHS:
                with slice_cols(w):
                    got = spmm(g, xl, xh, **kw)
                assert torch.equal(got, ref), (lo, F, w)
    assert int(indptr[hub + 1] - indptr[hub]) > 100_000


def test_invalid_slice_width_is_an_error():
    from adaqp_b200.manager.graph import LocalGraph, spmm
    dev = torch.device("cuda:0")
    L = layouts(1, 600, 8, 300, seed=1)[0]
    g = LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, dev)
    xl = torch.randn(L.n_inner, 300, device=dev)
    for w in [50, 200]:      # not a multiple of 4; wider than a warp's 128 columns but narrower than F
        with slice_cols(w), pytest.raises(RuntimeError, match="slice width"):
            spmm(g, xl, None, None, None)

"""Every instantiation of the CSR aggregation kernels against the float64 oracle, in every form the trainer uses.

spmm_csr_kernel<VEC, CHUNKS> is picked by the widest vector that divides F and the row pitches (VEC) and by
ceil(F / (32 VEC)) (CHUNKS); 16-byte rows of a multiple of 128 columns above 128 take spmm_csr_sliced_kernel in
128-column slices.  The F values below reach each of them:

    vec4: 388 -> CHUNKS 4, 700 -> 6, 1000 -> 8      vec2: 50 -> 2, 250 -> 4, 382 -> 6, 1022 -> 16
    vec1: 201 -> 8, 511 -> 16, 1023 -> 32           sliced: 384 (3 slices), 640 (5), 1024 (8, the ABI maximum)

(vec4 CHUNKS 1-3, vec2 CHUNKS 10 and vec1 CHUNKS 4 are in test_gpu_spmm.py.)  Forms: GCN forward / backward, SAGE
mean forward / backward, SAGE gcn forward / backward (self term), each over all rows and as the central rows plus
the marginal rows in two passes (local sources, then the halo sources accumulated), written into row views of a
larger sentinel-filled buffer as decomposed_graph_propagation does with out[num_central:].  Bound: |got - oracle|
<= 4e-6 * (L1 mass of the element's terms; worst observed on an H100 4.0e-7, fp32 rounding of rows of a few dozen
terms), and every row outside the view keeps its sentinel bit for bit."""
import contextlib

import numpy as np
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu

TOL = 4e-6
SENTINEL = -7.25e30


def lib():
    from adaqp_b200 import build as b
    b.build()
    from adaqp_b200 import _lib
    return _lib


@contextlib.contextmanager
def option(name, value):
    _lib = lib()
    old = _lib.get_option(name)
    _lib.set_option(name, value)
    try:
        yield
    finally:
        _lib.set_option(name, old)


def layouts(W, n, deg, F, seed):
    lib()
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    spec = SynthSpec(name="t", num_nodes=n, num_edges=n * deg, num_parts=W, num_feats=F, num_classes=5,
                     cross_fraction=0.3 if W > 1 else 0.0, community_size=64, seed=seed)
    return prepare_all_in_process(spec)


def forms(g):
    """name -> (spmm keyword arguments, oracle function, backward)."""
    return {"gcn_fwd": (dict(pre=g.norm["out_-0.5"], post=g.norm["in_-0.5"]), O.gcn_aggregation, False),
            "gcn_bwd": (dict(pre=g.norm["in_-0.5"], post=g.norm["out_-0.5"]), O.gcn_aggregation, True),
            "sage_mean_fwd": (dict(pre=None, post=None, mean=True), O.sage_aggregation, False),
            "sage_mean_bwd": (dict(pre=g.norm["out_-1"], post=None), O.sage_aggregation, True),
            "sage_gcn_fwd": (dict(pre=None, post=g.norm["in_+1_-1"], add_self=True), O.sage_gcn_aggregation, False),
            "sage_gcn_bwd": (dict(pre=g.norm["out_+1_-1"], post=None, add_self=True), O.sage_gcn_aggregation, True)}


class Case:
    def __init__(self, W, F, seed, n=1500, deg=14):
        from adaqp_b200.manager.graph import LocalGraph
        self.dev = torch.device("cuda:0")
        self.L = L = layouts(W, n, deg, F, seed)[-1]
        if W > 1:
            assert L.n_halo > 0 and 0 < L.n_central < L.n_inner
        self.g = LocalGraph(L.indptr, L.indices, L.in_degrees, L.out_degrees, L.n_inner, L.n_halo, self.dev)
        rng = np.random.RandomState(seed)
        self.x = rng.standard_normal((L.n_inner + L.n_halo, F)).astype(np.float32)
        self.xl = torch.from_numpy(self.x[:L.n_inner]).to(self.dev)
        self.xh = torch.from_numpy(self.x[L.n_inner:]).to(self.dev) if L.n_halo else None
        self.ip, self.ix = L.indptr, L.indices.astype(np.int64)

    def oracle(self, fn, bwd):
        L = self.L
        want = fn(self.ip, self.ix, self.x, L.in_degrees, L.out_degrees, L.n_inner, backward=bwd)
        mass = fn(self.ip, self.ix, np.abs(self.x), L.in_degrees, L.out_degrees, L.n_inner, backward=bwd)
        return want, mass

    def check(self, got, fn, bwd, lo=0, hi=None):
        """Worst error / mass of rows [lo, hi) of the aggregation; asserts the bound."""
        hi = self.L.n_inner if hi is None else hi
        want, mass = self.oracle(fn, bwd)
        err = np.abs(got.cpu().numpy().astype(np.float64) - want[lo:hi])
        ratio = err / np.maximum(mass[lo:hi], 1e-300)
        assert np.all((err == 0) | (mass[lo:hi] > 0))
        worst = float(ratio.max())
        assert worst <= TOL, (worst, np.unravel_index(ratio.argmax(), ratio.shape))
        return worst

    def into_view(self, kw, lo, hi, two_pass):
        """Rows [lo, hi) written into rows [1 + lo, 1 + hi) of a sentinel buffer of n_inner + 2 rows; checks the
        rows outside the view and returns the view."""
        from adaqp_b200.manager.graph import spmm
        n, F = self.L.n_inner, self.x.shape[1]
        buf = torch.full((n + 2, F), SENTINEL, device=self.dev)
        view = buf[1 + lo:1 + hi]
        if two_pass:
            spmm(self.g, self.xl, None, row_begin=lo, row_end=hi, out=view, part="local", **kw)
            spmm(self.g, self.xl, self.xh, row_begin=lo, row_end=hi, out=view, part="halo", **kw)
        else:
            spmm(self.g, self.xl, self.xh, row_begin=lo, row_end=hi, out=view, **kw)
        torch.cuda.synchronize()
        outside = torch.cat([buf[:1 + lo], buf[1 + hi:]])
        assert bool((outside == SENTINEL).all()), "rows outside [row_begin, row_end) were written"
        return view

    def run_all(self, names=None):
        """Every form: all rows in one launch, then central rows + marginal rows in two passes, each into a view."""
        from adaqp_b200.manager.graph import spmm
        L, worst = self.L, {}
        for name, (kw, fn, bwd) in forms(self.g).items():
            if names and name not in names:
                continue
            w = self.check(spmm(self.g, self.xl, self.xh, **kw), fn, bwd)
            w = max(w, self.check(self.into_view(kw, 0, L.n_inner, False), fn, bwd))
            if L.n_halo:
                cen = self.into_view(kw, 0, L.n_central, False)
                mar = self.into_view(kw, L.n_central, L.n_inner, True)
                w = max(w, self.check(cen, fn, bwd, 0, L.n_central), self.check(mar, fn, bwd, L.n_central, L.n_inner))
            worst[name] = w
        return worst


@pytest.mark.parametrize("F", [388, 700, 1000, 50, 250, 382, 1022, 201, 511, 1023, 384, 640, 1024])
@pytest.mark.parametrize("W", [1, 3])
def test_every_kernel_instantiation_matches_oracle(F, W):
    worst = Case(W, F, seed=F + W).run_all()
    print(f"\nspmm F={F} W={W}: worst error / mass {max(worst.values()):.3g}")


@pytest.mark.parametrize("impl", [1, 3, 4])
@pytest.mark.parametrize("F", [256, 100, 602, 13])
def test_sage_gcn_matches_oracle_under_every_impl(impl, F):
    """spmm_impl 3 / 4 (TMA row copies) run where F <= 256 has 16-byte rows and fall back to the default kernel
    elsewhere (F = 602, 13)."""
    case = Case(3, F, seed=F + impl)
    with option("spmm_impl", impl):
        worst = case.run_all(("sage_gcn_fwd", "sage_gcn_bwd"))
    print(f"\nsage_gcn impl={impl} F={F}: worst error / mass {max(worst.values()):.3g}")


@pytest.mark.parametrize("slice_cols", [32, 64, 128])
@pytest.mark.parametrize("F", [256, 384, 1024])
def test_sage_gcn_matches_oracle_under_forced_slices(slice_cols, F):
    case = Case(3, F, seed=F + slice_cols)
    with option("spmm_slice_cols", slice_cols):
        worst = case.run_all(("sage_gcn_fwd", "sage_gcn_bwd"))
    print(f"\nsage_gcn slice_cols={slice_cols} F={F}: worst error / mass {max(worst.values()):.3g}")

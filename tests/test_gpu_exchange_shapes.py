"""Every instantiation of the quantised exchange kernels against the C oracle, at the shapes, grids, worlds and rows
where they can go wrong.

W ranks are simulated on one device (their slabs address each other directly, the same stores a peer GPU receives
over NVLink).  Before each exchange the key's qdata, params and halo regions of every slab are filled with a
sentinel byte; afterwards the whole span is compared with an image built from the oracle: the wire bytes the
oracle marks valid, the bf16 params, the received halo rows, and the sentinel everywhere else (each segment's
unwritten trailing byte, the padding up to every region's end, halo rows nobody sends).  Everything is bit-exact;
the rows of test_edge_rows compare NaN equal to NaN whatever its payload, and a row minimum of zero modulo its
sign (the warp reduction may return either zero of a row that holds both; the halo stays bit-exact because
q / scale + (+-0) is the same value)."""
import contextlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from exchange_cases import BYTE_ROW_KINDS, RECV_VIEWS, SHAPES, Shape
from oracle import oracle as O

pytestmark = pytest.mark.gpu

SENT = 0xA5
SENT32 = np.frombuffer(bytes([SENT] * 4), np.int32)[0]
EINVAL, ELIMIT = -1, -3          # include/adaqp_b200.h
KEY = "forward0"


@pytest.fixture(scope="module")
def env():
    from adaqp_b200 import build
    build.build()
    from adaqp_b200 import _lib
    return _lib


@contextlib.contextmanager
def options(_lib, **kv):
    old = {k: _lib.get_option(k) for k in kv}
    try:
        for k, v in kv.items():
            _lib.set_option(k, v)
        yield
    finally:
        for k, v in old.items():
            _lib.set_option(k, v)


_LAYS = {}


def synth_ranks(W, n, seed):
    from adaqp_b200.manager.layout import prepare_all_in_process
    from adaqp_b200.manager.partition_synth import SynthSpec
    if (W, n, seed) not in _LAYS:
        spec = SynthSpec(name="t", num_nodes=n, num_edges=n * 10, num_parts=W, num_feats=16, num_classes=5,
                         cross_fraction=0.3, community_size=64, seed=seed)
        _LAYS[W, n, seed] = prepare_all_in_process(spec)
    return _LAYS[W, n, seed]


def hand_ranks(rng):
    """A world the synthetic partitioner never builds: 0 -> 1 and 2 -> 0 are one-directional channels (send_side
    omits peers that request nothing), 2 -> 0 carries a single row, rank 1 has 3 halo rows nobody sends, rank 2
    receives nothing (num_remote 0) and rank 3 has no channel at all."""
    e = np.zeros(0, np.int64)
    return [SimpleNamespace(n_inner=60, n_halo=1, send_idx={1: (0, 37)},
                            total_send_idx=rng.choice(60, 37, replace=False).astype(np.int64), recv_idx={2: np.array([0])}),
            SimpleNamespace(n_inner=30, n_halo=40, send_idx={}, total_send_idx=e,
                            recv_idx={0: rng.permutation(40)[:37].astype(np.int64)}),
            SimpleNamespace(n_inner=20, n_halo=0, send_idx={0: (0, 1)}, total_send_idx=np.array([7]), recv_idx={}),
            SimpleNamespace(n_inner=10, n_halo=0, send_idx={}, total_send_idx=e, recv_idx={})]


def device_rows(x, shape, dev):
    """x as columns [col, col + F) of a [n, F + pad] device tensor whose other columns hold NaN, so that a read
    past F poisons the row's range."""
    buf = torch.full((x.shape[0], shape.ld), float("nan"), device=dev)
    v = buf[:, shape.col:shape.col + shape.F]
    v.copy_(torch.from_numpy(np.ascontiguousarray(x)))
    if x.shape[0]:
        assert v.stride(0) == shape.ld and v.data_ptr() % 16 == shape.base_mod16
    return v


def byte_row_kinds(assign):
    kinds = set()
    for per_peer in assign:
        for bits in per_peer.values():
            for b in (2, 4, 8):
                n, wpt = int((bits == b).sum()), 8 // b
                if n >= wpt:
                    kinds.add((b, "full"))
                if n % wpt:
                    kinds.add((b, "tail"))
    return kinds


def received_rows(e):
    """Halo rows some peer sends rank e."""
    return np.unique(np.concatenate([np.asarray(v, np.int64) for v in e.recv_idx.values()] + [np.zeros(0, np.int64)]))


class World:
    def __init__(self, ranks, dims, timeout_ns=5_000_000_000):
        from adaqp_b200.communicator.p2p import PeerExchange, wire_in_process
        self.dev = torch.device("cuda:0")
        self.ranks, self.dims, W = ranks, dict(dims), len(ranks)
        self.exs = [PeerExchange(r, W, self.dev, [1], R.send_idx, {p: torch.from_numpy(np.asarray(v)) for p, v in R.recv_idx.items()},
                                 torch.from_numpy(np.asarray(R.total_send_idx)), R.n_halo, timeout_ns=timeout_ns, key_dims=self.dims)
                    for r, R in enumerate(ranks)]
        wire_in_process(self.exs)
        self.keep = []

    def close(self):
        for e in self.exs:
            e.close()

    # ---- inputs and assignments
    def inputs(self, F, rng):
        return [rng.standard_normal((R.n_inner, F)).astype(np.float32) for R in self.ranks]

    def assignment(self, rng, bits=None):
        """[rank][peer] -> int32 bits of every row the rank sends the peer; random over {2, 4, 8} unless `bits`."""
        out = []
        for R in self.ranks:
            out.append({p: (np.full(hi - lo, bits, np.int32) if bits else
                            np.array([2, 4, 8], np.int32)[rng.randint(0, 3, hi - lo)]) for p, (lo, hi) in R.send_idx.items()})
        return out

    def apply(self, assign_by_key):
        from adaqp_b200.communicator.p2p import update_quant_in_process
        per_rank = [{k: {p: torch.from_numpy(a[r][p]) for p in a[r]} for k, a in assign_by_key.items()}
                    for r in range(len(self.ranks))]
        update_quant_in_process(self.exs, per_rank)

    # ---- slab regions
    def span(self, r, key):
        from adaqp_b200.communicator.p2p import _up
        lay, F = self.exs[r].layout, self.dims[key]
        q = [lay.qdata_off[(key, p)] for p in sorted(lay.recv_rows) if (key, p) in lay.qdata_off]
        lo = min(q) if q else lay.halo_off[key]
        return lo, lay.halo_off[key] + _up(4 * F * max(lay.num_remote, 1))

    def fill(self, key):
        for r, e in enumerate(self.exs):
            lo, hi = self.span(r, key)
            e.slab.view(lo, (hi - lo,), torch.uint8).fill_(SENT)

    def sync(self):
        torch.cuda.synchronize()
        for e in self.exs:
            e.check_status()

    # ---- quantised exchange
    def post_quant(self, key, xs, seeds, offs, shape=None, gathered=False, traces=None):
        shape = shape or Shape(self.dims[key])
        self.fill(key)
        for r, (e, R) in enumerate(zip(self.exs, self.ranks)):
            x = device_rows(xs[r][R.total_send_idx] if gathered else xs[r], shape, self.dev)
            self.keep.append(x)
            e.post_send_quant(key, x, seeds[r], offs[r], trace=None if traces is None else traces[r], gathered=gathered)

    def recv_quant(self, key):
        for e in self.exs:
            e.complete_recv_quant(key)

    def oracle(self, key, xs, assign, seeds, offs):
        sends = [x[R.total_send_idx] for x, R in zip(xs, self.ranks)]
        return O.exchange_quant(sends, [R.send_idx for R in self.ranks], [R.recv_idx for R in self.ranks],
                                [R.n_halo for R in self.ranks], assign, seeds, offs, return_wire=True)

    def check_quant(self, key, want, wire, new_offs, offs, edge=False):
        self.sync()
        for r, e in enumerate(self.exs):
            assert e.quant_plans[key].philox_increment == new_offs[r] - offs[r]
            self.check_slab(r, key, want[r], wire, edge)

    def exchange(self, key, xs, assign, seeds, offs, edge=False, **kw):
        """One quantised exchange of `key`, checked against the oracle; returns the oracle's halos."""
        self.post_quant(key, xs, seeds, offs, **kw)
        self.recv_quant(key)
        want, wire, new_offs = self.oracle(key, xs, assign, seeds, offs)
        self.check_quant(key, want, wire, new_offs, offs, edge)
        return want

    def check_slab(self, r, key, want_r, wire, edge):
        """Rank r's span of `key` against the oracle image: wire[p][r] = (qdata, params, valid) of every peer p
        (None for an fp32 key), want_r = the oracle's halo."""
        e, F = self.exs[r], self.dims[key]
        lay = e.layout
        lo, hi = self.span(r, key)
        got = e.slab.view(lo, (hi - lo,), torch.uint8).cpu().numpy()
        img = np.full(hi - lo, SENT, np.uint8)
        ok = np.zeros(hi - lo, bool)            # positions where a documented equivalence is allowed
        regions = []
        for p in (e.recv_peers if wire is not None else ()):
            wq, wprm, valid = wire[p][r]
            q0, p0 = lay.qdata_off[(key, p)] - lo, lay.params_off[(key, p)] - lo
            img[q0:q0 + wq.size][valid] = wq[valid]
            img[p0:p0 + wprm.nbytes] = np.ascontiguousarray(wprm, np.uint16).view(np.uint8).reshape(-1)
            regions += [(q0, f"qdata from {p}"), (q0 + wq.size, f"qdata padding from {p}"),
                        (p0, f"params from {p}"), (p0 + wprm.nbytes, f"params padding from {p}")]
            if edge:                             # the wire minimum modulo the sign of zero
                S = wprm.shape[1]
                mins = slice(p0 + 2 * S, p0 + 4 * S)
                gz = (got[mins].view(np.uint16) & 0x7FFF) == 0
                wz = (img[mins].view(np.uint16) & 0x7FFF) == 0
                ok[mins] |= np.repeat(gz & wz, 2)
        h0 = lay.halo_off[key] - lo
        n = e.num_remote
        rows = received_rows(e)
        img[h0:h0 + 4 * F * n].view(np.float32).reshape(n, F)[rows] = want_r[rows]
        regions += [(h0, "halo"), (h0 + 4 * F * n, "halo padding")]
        if edge:
            both = np.isnan(got[h0:h0 + 4 * F * n].view(np.float32)) & np.isnan(img[h0:h0 + 4 * F * n].view(np.float32))
            ok[h0:h0 + 4 * F * n] |= np.repeat(both, 4)
        bad = np.nonzero((got != img) & ~ok)[0]
        if bad.size:
            first = bad[0]
            name = [nm for s, nm in sorted(regions) if s <= first][-1]
            raise AssertionError(f"rank {r} key {key}: {bad.size} bytes differ from the oracle image; first at "
                                 f"span byte {first} ({name}): got {got[first]:#04x}, want {img[first]:#04x}")

    def recv_again(self, _lib, key, want, pad, col, edge=False):
        """Run the receive a second time on the same seq and landed payload into columns [col, col + F) of a
        sentinel-filled [num_remote + 2, F + pad] buffer (rows 1 .. num_remote); checks the rows received and that
        nothing else in the buffer was touched.  Re-posting the acks with the same seq is harmless."""
        F = self.dims[key]
        for r, e in enumerate(self.exs):
            n = e.num_remote
            buf = torch.full((n + 2, F + pad), int(SENT32), dtype=torch.int32, device=self.dev)
            out = buf.view(torch.float32)[1:n + 1, col:col + F]
            plan = e.quant_plans[key]
            rc = e._lib.adaqp_recv_quant(out.data_ptr(), F + pad, F, plan.recv_items.data_ptr(), plan.n_recv,
                                         plan.recv_chans.data_ptr(), plan.n_recv_chans, e.seq[key], e._work_ptr(key, 1),
                                         e.status.data_ptr(), e.timeout_ns, _lib.stream_ptr(None))
            _lib.check(rc, "adaqp_recv_quant")
            self.sync()
            img = np.full((n + 2, F + pad), SENT32, np.int32)
            rows = received_rows(e)
            img[1:n + 1, col:col + F][rows] = want[r][rows].view(np.int32)
            got = buf.cpu().numpy()
            bad = got != img
            if edge:
                bad[1:n + 1, col:col + F] &= ~(np.isnan(got[1:n + 1, col:col + F].view(np.float32))
                                              & np.isnan(img[1:n + 1, col:col + F].view(np.float32)))
            assert not bad.any(), (r, pad, col, np.argwhere(bad)[:5].tolist())


def seeds_offs(W, big=False):
    if big:   # the high words of the Philox key and of the block counter
        return [2 ** 32 + 977 * r + 5 for r in range(W)], [2 ** 34 + 2 ** 33 + 8 * r for r in range(W)]
    return [1000 + r for r in range(W)], [8 * r for r in range(W)]


# ------------------------------------------------------------------ a, b: every rung, no stray writes
@pytest.mark.parametrize("shape", SHAPES, ids=[s.name for s in SHAPES])
def test_every_instantiation_matches_oracle(env, shape):
    F = shape.F
    w = World(synth_ranks(3, 1500, 3), {KEY: F})
    try:
        rng = np.random.RandomState(F + shape.pad)
        assign = w.assignment(rng)
        assert BYTE_ROW_KINDS <= byte_row_kinds(assign)
        w.apply({KEY: assign})
        xs = w.inputs(F, rng)
        for x in xs:
            x[::13] = 0.0                     # constant rows: scale = inf
        seeds, offs = seeds_offs(3)
        want = w.exchange(KEY, xs, assign, seeds, offs, shape=shape)
        for pad, col in RECV_VIEWS:
            w.recv_again(env, KEY, want, pad, col)
        w.exchange(KEY, xs, assign, seeds, offs, shape=shape, gathered=True)
    finally:
        w.close()


# ------------------------------------------------------------------ c: persistent grids
def warp_spans(items, nwarps):
    """Fewest items and fewest channels any warp of a persistent grid handles."""
    return (min(items[w::nwarps].size for w in range(nwarps)),
            min(np.unique(items["chan"][w::nwarps]).size for w in range(nwarps)))


@pytest.mark.parametrize("F", [256, 602, 201])
def test_persistent_grids_match_default_grid(env, F):
    from adaqp_b200.communicator.p2p import build_recv_items, build_send_items
    w = World(synth_ranks(3, 1500, 3), {KEY: F})
    try:
        rng = np.random.RandomState(F)
        assign = w.assignment(rng)
        w.apply({KEY: assign})
        xs = w.inputs(F, rng)
        seeds, offs = seeds_offs(3)
        for r, e in enumerate(w.exs):
            si, _ = build_send_items(e.send_peers, e.send_idx, e.total_send_idx, assign[r], F)
            ri, _ = build_recv_items(e.recv_peers, e.recv_idx, {p: assign[p][r] for p in e.recv_peers}, F)
            for items in (si, ri):
                n_items, n_chans = warp_spans(items, 3 * 8)
                assert n_items >= 2 and n_chans >= 2, (r, n_items, n_chans)
        def halos():
            return [e.halo(KEY).cpu().numpy().view(np.uint32) for e in w.exs]

        w.exchange(KEY, xs, assign, seeds, offs)
        ref = halos()
        for ctas in (1, 3):
            with options(env, exch_send_ctas=ctas, exch_recv_ctas=ctas):
                w.exchange(KEY, xs, assign, seeds, offs)
            for got, want in zip(halos(), ref):
                np.testing.assert_array_equal(got, want)
    finally:
        w.close()


def fp_exchange(w, key, xs, shape=None):
    """One fp32 exchange of `key`; checks every slab's halo region against the oracle image."""
    F = w.dims[key]
    shape = shape or Shape(F)
    w.fill(key)
    for e, x in zip(w.exs, xs):
        xt = device_rows(x, shape, w.dev)
        w.keep.append(xt)
        e.post_send_fp(key, xt)
    for e in w.exs:
        e.complete_recv_fp(key)
    w.sync()
    want = O.exchange_fp([x[R.total_send_idx] for x, R in zip(xs, w.ranks)], [R.send_idx for R in w.ranks],
                         [R.recv_idx for R in w.ranks], [R.n_halo for R in w.ranks])
    for r in range(len(w.exs)):
        w.check_slab(r, key, want[r], None, False)
    for e in w.exs:
        e.release_fp(key)
    return want


def test_fp32_persistent_grid(env):
    F = 100
    w = World(synth_ranks(3, 1500, 3), {"test0": F})
    try:
        rng = np.random.RandomState(5)
        for R in w.ranks:                        # one item per row, channel by channel
            items = np.zeros(R.total_send_idx.size, [("chan", np.int64)])
            items["chan"] = np.concatenate([np.full(hi - lo, ci) for ci, (lo, hi) in enumerate(R.send_idx.values())])
            n_items, n_chans = warp_spans(items, 8)
            assert n_items >= 2 and n_chans >= 2
        xs = w.inputs(F, rng)
        with options(env, exch_send_ctas=1):
            fp_exchange(w, "test0", xs)
            fp_exchange(w, "test0", w.inputs(F, rng))
    finally:
        w.close()


# ------------------------------------------------------------------ d: eight ranks, sparse peer graphs
@pytest.mark.parametrize("F", [256, 602])
def test_eight_ranks(env, F):
    w = World(synth_ranks(8, 4000, 8), {KEY: F})
    try:
        rng = np.random.RandomState(F)
        assign = w.assignment(rng)
        w.apply({KEY: assign})
        seeds, offs = seeds_offs(8)
        xs = w.inputs(F, rng)
        w.exchange(KEY, xs, assign, seeds, offs)
        w.exchange(KEY, xs, assign, seeds, [o + 4096 for o in offs], gathered=True)
    finally:
        w.close()


@pytest.mark.parametrize("F", [256, 47])
def test_one_directional_and_empty_channels(env, F):
    rng = np.random.RandomState(F)
    w = World(hand_ranks(rng), {KEY: F, "test0": F})
    try:
        assert [e.num_remote for e in w.exs] == [1, 40, 0, 0]
        assign = w.assignment(rng)
        assign[2][0][:] = 2                      # one row at 2 bits: one byte-row with 3 rows missing
        w.apply({KEY: assign})
        e3 = w.exs[3].quant_plans[KEY]
        assert e3.n_send_chans == 0 and e3.n_recv_chans == 0
        seeds, offs = seeds_offs(4)
        for rep in range(2):
            xs = w.inputs(F, rng)
            w.exchange(KEY, xs, assign, seeds, [o + 4096 * rep for o in offs])
            fp_exchange(w, "test0", xs)
    finally:
        w.close()


# ------------------------------------------------------------------ e: re-assignment, keys in flight
def test_reassignment_keeps_the_ack_protocol(env):
    F = 256
    w = World(synth_ranks(3, 1500, 4), {KEY: F})
    try:
        rng = np.random.RandomState(11)
        seeds, offs = seeds_offs(3)
        for i, bits in enumerate((2, None, 8, None)):
            assign = w.assignment(rng, bits)
            w.apply({KEY: assign})
            w.exchange(KEY, w.inputs(F, rng), assign, seeds, [o + 65536 * i for o in offs])
        assert all(e.seq[KEY] == 4 for e in w.exs)
    finally:
        w.close()


def test_two_keys_in_flight_received_in_reverse(env):
    dims = {"forward0": 602, "forward1": 256}
    w = World(synth_ranks(3, 1500, 4), dims)
    try:
        rng = np.random.RandomState(12)
        assign = {k: w.assignment(rng) for k in dims}
        w.apply(assign)
        seeds, offs = seeds_offs(3)
        offs1 = [o + (1 << 20) for o in offs]
        xs = {k: w.inputs(F, rng) for k, F in dims.items()}
        w.post_quant("forward0", xs["forward0"], seeds, offs)
        w.post_quant("forward1", xs["forward1"], seeds, offs1)
        w.recv_quant("forward1")
        w.recv_quant("forward0")
        for k, o in (("forward0", offs), ("forward1", offs1)):
            want, wire, new_offs = w.oracle(k, xs[k], assign[k], seeds, o)
            w.check_quant(k, want, wire, new_offs, o)
    finally:
        w.close()


# ------------------------------------------------------------------ f: rows at the edges
def edge_inputs(w, F, rng):
    """Every sent row gets one of: NaN, +inf, -inf, a range that overflows to inf, a subnormal range (scale inf: q
    saturates into the neighbouring rows' bits, as in the reference), a constant row, a zero row, a minimum that
    mixes -0.0 and +0.0 under a positive maximum, or plain data."""
    xs = w.inputs(F, rng)
    for x, R in zip(xs, w.ranks):
        for i, row in enumerate(np.unique(R.total_send_idx)):
            c = rng.randint(0, F)
            v = x[row]
            kind = i % 9
            if kind == 0:
                v[c] = np.nan
            elif kind == 1:
                v[c] = np.inf
            elif kind == 2:
                v[c] = -np.inf
            elif kind == 3:
                v[:] = rng.uniform(-3e38, 3e38, F)
                v[0], v[-1] = 3e38, -3e38
            elif kind == 4:
                v[:] = np.where(rng.rand(F) < 0.5, 0.0, 1e-40)
                v[0], v[-1] = 0.0, 1e-40
            elif kind == 5:
                v[:] = 1.5
            elif kind == 6:
                v[:] = 0.0
            elif kind == 7:
                v[:] = np.abs(v)
                v[rng.rand(F) < 0.3] = 0.0
                v[rng.rand(F) < 0.3] = -0.0
                v[0], v[-1] = -0.0, 0.0
    return xs


@pytest.mark.parametrize("F", [256, 602, 47])
def test_edge_rows(env, F):
    w = World(synth_ranks(3, 1500, 5), {KEY: F})
    try:
        rng = np.random.RandomState(F + 1)
        assign = w.assignment(rng)
        w.apply({KEY: assign})
        xs = edge_inputs(w, F, rng)
        assert np.isnan(xs[0]).any() and np.isinf(xs[0]).any() and (np.signbit(xs[0]) & (xs[0] == 0)).any()
        assert ((xs[0] > 0) & (xs[0] < np.finfo(np.float32).tiny)).any()
        seeds, offs = seeds_offs(3, big=True)
        want = w.exchange(KEY, xs, assign, seeds, offs, edge=True)
        for pad, col in RECV_VIEWS:
            w.recv_again(env, KEY, want, pad, col, edge=True)
        w.exchange(KEY, xs, assign, seeds, offs, edge=True, gathered=True)
    finally:
        w.close()


# ------------------------------------------------------------------ g: fp32 exchange, trace
FP_WIDTHS = (1, 3, 12, 1030, 2048)


@pytest.mark.parametrize("view", [(0, 0), (4, 0), (1, 1)], ids=["contiguous", "ld+4", "ld+1_col1"])
def test_fp32_widths_and_strides(env, view):
    dims = {f"test{i}": F for i, F in enumerate(FP_WIDTHS)}
    w = World(synth_ranks(3, 1500, 6), dims)
    try:
        rng = np.random.RandomState(view[0])
        for key, F in dims.items():
            fp_exchange(w, key, w.inputs(F, rng), Shape(F, *view))
    finally:
        w.close()


@pytest.mark.parametrize("F", [100, 1024])
def test_trace_is_exact_fp32(env, F):
    w = World(synth_ranks(3, 1500, 7), {KEY: F})
    try:
        rng = np.random.RandomState(F)
        assign = w.assignment(rng)
        w.apply({KEY: assign})
        seeds, offs = seeds_offs(3)
        traces = [torch.zeros(R.total_send_idx.size, device=w.dev) for R in w.ranks]
        mirror = [np.zeros(R.total_send_idx.size, np.float32) for R in w.ranks]
        coef = np.float32(F / 6.0)
        for rep in range(2):
            xs = w.inputs(F, rng)
            w.exchange(KEY, xs, assign, seeds, [o + 4096 * rep for o in offs], traces=traces)
            for m, x, R in zip(mirror, xs, w.ranks):
                s = x[R.total_send_idx]
                rg = s.max(1) - s.min(1)
                m[:] = m + coef * (rg * rg)
        for t, m in zip(traces, mirror):
            np.testing.assert_array_equal(t.cpu().numpy().view(np.uint32), m.view(np.uint32))
    finally:
        w.close()


# ------------------------------------------------------------------ h: argument errors
def test_refused_calls_launch_nothing(env):
    """F above 1024, an offset that is not a multiple of 4 and more than 64 channels are refused with their error
    codes before anything is launched: no flag or ack word moves and the generator offset stays where it was."""
    gen = torch.cuda.default_generators[0]
    off0 = gen.get_offset()
    w = World(synth_ranks(3, 1500, 3), {KEY: 256, "forward1": 1025})
    try:
        rng = np.random.RandomState(1)
        w.apply({k: w.assignment(rng) for k in w.dims})
        e, L, stream = w.exs[0], w.exs[0]._lib, env.stream_ptr(None)
        x = torch.zeros(w.ranks[0].n_inner, 1025, device=w.dev)
        scratch = torch.zeros(8, dtype=torch.int32, device=w.dev)   # work counter, and every word of the 65 channels
        work, word = scratch.data_ptr(), scratch.data_ptr() + 16

        def send(F, base_offset, items, n_items, chans, n_chans):
            return L.adaqp_send_quant(x.data_ptr(), x.stride(0), F, items, n_items, chans, n_chans, None, 7, base_offset,
                                      1, work, e.status.data_ptr(), 1000, stream)

        def recv(F, items, n_items, chans, n_chans):
            return L.adaqp_recv_quant(x.data_ptr(), F, F, items, n_items, chans, n_chans, 1, work, e.status.data_ptr(),
                                      1000, stream)

        wide, plan = e.quant_plans["forward1"], e.quant_plans[KEY]
        assert send(1025, 0, wide.send_items.data_ptr(), wide.n_send, wide.send_chans.data_ptr(), wide.n_send_chans) == ELIMIT
        assert recv(1025, wide.recv_items.data_ptr(), wide.n_recv, wide.recv_chans.data_ptr(), wide.n_recv_chans) == ELIMIT
        assert send(256, 6, plan.send_items.data_ptr(), plan.n_send, plan.send_chans.data_ptr(), plan.n_send_chans) == EINVAL
        sc, rc = np.zeros(65, env.SEND_CHAN_DTYPE), np.zeros(65, env.RECV_CHAN_DTYPE)
        for t in (sc, rc):
            for f in ("qdata", "params", "flag", "ack"):
                t[f] = word
        sc["fp_rows"] = word
        schans, rchans = (torch.from_numpy(t.view(np.uint8)).to(w.dev) for t in (sc, rc))
        assert send(256, 0, work, 0, schans.data_ptr(), 65) == ELIMIT
        assert recv(256, work, 0, rchans.data_ptr(), 65) == ELIMIT
        w.sync()
        assert not bool(scratch.any())
        for f in w.exs:
            for k in w.dims:    # the flag words of every key, then its ack words
                assert not bool(f.slab.view(f.layout.flag_off[k], (64,), torch.int32).any()), (f.rank, k)
        assert gen.get_offset() == off0
    finally:
        w.close()

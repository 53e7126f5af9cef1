"""NVLink/NVSwitch peer-to-peer data plane for the boundary-message exchange.

Replaces the pinned-host staging + gloo isend/irecv data path of
AdaQP/communicator/comm.py:166-222 and the buffer registry of
AdaQP/communicator/buffer.py:154-248: every rank owns ONE device slab holding, per layer
key, (a) a region per source peer that receives that peer's packed bytes and bf16
parameters in the reference wire format, (b) the fp32 halo matrix [num_remote, F] that
both exchange flavours fill, and (c) flag / ack words.  Peers map each other's slab
(CUDA IPC across processes; plain pointers inside one process) and the kernels of
csrc/exchange.cu store into it directly.  The control plane (metadata, IPC handles,
bit assignments) stays on the host process group, as in the reference
(buffer.py:219-231 all_gather_object).

Layer keys: 'forward{l}', 'backward{l}' (training) and 'test{l}' (evaluation, always fp32,
buffer.py:32-34 "test" buffers).  GATv2's 'push{l}' keys run the other way: the holder of a halo row sends it back
to the row's owner, whose push region has one fp32 row per position of its total_send_idx.
"""
from __future__ import annotations

import ctypes as C
import re
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import _lib

BITS_SET = (2, 4, 8)   # buffer.py:20
ALIGN = 256
DEFAULT_TIMEOUT_NS = 30_000_000_000


def _up(x: int, a: int = ALIGN) -> int:
    return (x + a - 1) // a * a


def layer_keys(num_layers: int) -> List[str]:
    """Exchange keys in a fixed order shared by all ranks (assigner.py:98-101 + eval)."""
    keys = [f"test{i}" for i in range(num_layers)]
    keys += [f"forward{i}" for i in range(num_layers)]
    keys += [f"backward{i}" for i in range(1, num_layers)]
    return keys


def layer_index(key: str) -> int:
    """Layer (or propagation step) index of a key: its whole trailing number ('forward10' -> 10).  The reference reads
    the last character (buffer.py:63,201), which is the same for every key below 10."""
    m = re.search(r"(\d+)$", key)
    if m is None:
        raise ValueError(f"exchange key {key!r} has no layer index")
    return int(m.group(1))


def key_dim(key: str, buffer_shape: Sequence[int]) -> int:
    return int(buffer_shape[layer_index(key)])


def layer_key_dims(buffer_shape: Sequence[int]) -> Dict[str, int]:
    """The reference models' key table: layer_keys, each as wide as its layer's entry of buffer_shape."""
    return {k: key_dim(k, buffer_shape) for k in layer_keys(len(buffer_shape))}


def attn_keys(layer: int) -> Tuple[str, str]:
    """fp32 keys of GAT's per-row attention scalars: el rows with the forward exchange, [er | lse | s] rows with the
    backward exchange.  Training and evaluation never have the same key in flight, so both use them."""
    return f"attn_fwd{layer}", f"attn_bwd{layer}"


def gat_key_dims(widths: Sequence[int], heads: Sequence[int]) -> Dict[str, int]:
    """Exchange keys and widths of a GAT model whose layer l exchanges rows of z_l (width widths[l], heads[l] heads):
    test / forward / backward keys of every layer (backward0 included: dW_0 needs the gradient of remote
    destinations), then the attention keys."""
    L = len(widths)
    dims = {f"test{i}": int(widths[i]) for i in range(L)}
    dims.update({f"forward{i}": int(widths[i]) for i in range(L)})
    dims.update({f"backward{i}": int(widths[i]) for i in range(L)})
    for i in range(L):
        fwd, bwd = attn_keys(i)
        dims[fwd], dims[bwd] = int(heads[i]), 3 * int(heads[i])
    return dims


def pool_arg_key(layer: int) -> str:
    """fp32 key of the SAGE max-pool arg rows (int32 bit patterns), sent with the backward exchange of the layer."""
    return f"pool_arg{layer}"


def sage_pool_key_dims(widths: Sequence[int]) -> Dict[str, int]:
    """Exchange keys and widths of a SAGE max-pool model whose layer l exchanges rows of p_l = relu(fc_pool(x_l))
    (width widths[l], the layer's input width): test / forward / backward keys of every layer (backward0 included:
    dW_pool of layer 0 needs the gradient of remote destinations), then the arg keys."""
    L = len(widths)
    dims = {f"test{i}": int(widths[i]) for i in range(L)}
    dims.update({f"forward{i}": int(widths[i]) for i in range(L)})
    dims.update({f"backward{i}": int(widths[i]) for i in range(L)})
    dims.update({pool_arg_key(i): int(widths[i]) for i in range(L)})
    return dims


def appnp_key_dims(num_classes: int, k: int) -> Dict[str, int]:
    """Exchange keys of APPNP with K propagation steps: step k exchanges h_k on forward{k} (test{k} in evaluation)
    and g_{k+1} on backward{k}; backward0 is needed because the MLP's weight gradients need g_0 at remote
    destinations.  Every key is num_classes wide.  GCNII with L layers uses the same table, hidden_dim wide: layer l
    exchanges its input on forward{l-1} and its output gradient on backward{l-1}."""
    C = int(num_classes)
    dims = {f"test{i}": C for i in range(k)}
    dims.update({f"forward{i}": C for i in range(k)})
    dims.update({f"backward{i}": C for i in range(k)})
    return dims


def push_key(layer: int) -> str:
    """fp32 key of GATv2's pushed halo-row gradients: the holder of a halo row sends the row's source-side gradient
    back to its owner."""
    return f"push{layer}"


def is_push(key: str) -> bool:
    return key.startswith("push")


def gatv2_key_dims(widths: Sequence[int]) -> Dict[str, int]:
    """Exchange keys and widths of a GATv2 model whose layer l exchanges rows of zs_l (width widths[l]): test /
    forward keys of every layer, then the push keys.  zd and the attention logits never leave their rank, so there
    are no backward keys."""
    L = len(widths)
    dims = {f"test{i}": int(widths[i]) for i in range(L)}
    dims.update({f"forward{i}": int(widths[i]) for i in range(L)})
    dims.update({push_key(i): int(widths[i]) for i in range(L)})
    return dims


# fp32 key of Correct & Smooth's propagation steps (model/ops.py correct_and_smooth): every step of a pass reuses it
CS_KEY = "cs0"


def with_cs_key(key_dims: Dict[str, int], num_classes: int) -> Dict[str, int]:
    """A key table with CS_KEY appended, num_classes wide."""
    return {**key_dims, CS_KEY: int(num_classes)}


def quantisable(key: str) -> bool:
    """Keys that may travel quantised (training exchanges of layer rows); test, attention and arg keys are fp32."""
    return key.startswith(("forward", "backward"))


def qsize(n: int, bits: int, F: int) -> int:
    """buffer.py:181-186."""
    wpt = 8 // bits
    n_round = n + (wpt - n % wpt) % wpt
    return (bits * n_round * F + 8) // 8


# ------------------------------------------------------------------------------ layout
@dataclass
class SlabLayout:
    """Byte offsets inside one rank's slab.  A pure function of (world size, layer dims,
    rows received from every peer, num_remote, rows sent), so every rank can compute every peer's
    layout from the all-gathered row counts.  The region of a push key holds `push_rows` rows (the
    length of total_send_idx), every other key's `num_remote`."""
    world_size: int
    keys: List[str]
    dims: Dict[str, int]
    recv_rows: Dict[int, int]            # src peer -> rows it sends me
    num_remote: int
    flag_off: Dict[str, int] = field(default_factory=dict)   # + 4 * src
    ack_off: Dict[str, int] = field(default_factory=dict)    # + 4 * dst
    qdata_off: Dict[Tuple[str, int], int] = field(default_factory=dict)
    params_off: Dict[Tuple[str, int], int] = field(default_factory=dict)
    halo_off: Dict[str, int] = field(default_factory=dict)
    work_off: int = 0
    status_off: int = 0
    total: int = 0
    push_rows: int = 0

    @staticmethod
    def build(world_size: int, keys: List[str], dims: Dict[str, int], recv_rows: Dict[int, int],
              num_remote: int, push_rows: int = 0) -> "SlabLayout":
        L = SlabLayout(world_size, list(keys), dict(dims), dict(recv_rows), int(num_remote), push_rows=int(push_rows))
        off = 0
        for k in keys:
            L.flag_off[k] = off
            off += _up(4 * world_size, 128)
            L.ack_off[k] = off
            off += _up(4 * world_size, 128)
        L.status_off = off
        off += 128
        L.work_off = off                      # 2 words per key (send / recv side counters)
        off += _up(8 * len(keys), 128)
        off = _up(off)
        for k in keys:
            F = dims[k]
            if quantisable(k):
                for p in sorted(recv_rows):
                    n = recv_rows[p]
                    L.qdata_off[(k, p)] = off
                    off += _up(n * F + 3 + 16)     # worst case: all rows 8-bit, 3 segments' trailing bytes
                    L.params_off[(k, p)] = off
                    off += _up(4 * n)
            L.halo_off[k] = off
            off += _up(4 * F * max(push_rows if is_push(k) else num_remote, 1))
        L.total = _up(off, 4096)
        return L


class Slab:
    """Device memory owned through the C ABI (cudaMalloc), exportable over CUDA IPC."""

    def __init__(self, nbytes: int, device: torch.device):
        self.device = device
        self.nbytes = int(nbytes)
        L = _lib.load()
        ptr = C.c_void_p()
        with torch.cuda.device(device):
            _lib.check(L.adaqp_slab_alloc(C.byref(ptr), self.nbytes), "adaqp_slab_alloc")
        self.ptr = int(ptr.value)
        self._opened: Dict[int, int] = {}

    def export_handle(self) -> bytes:
        buf = C.create_string_buffer(_lib.IPC_HANDLE_BYTES)
        _lib.check(_lib.load().adaqp_ipc_export(self.ptr, buf), "adaqp_ipc_export")
        return bytes(buf.raw)

    def open_peer(self, handle: bytes) -> int:
        out = C.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().adaqp_ipc_open(handle, C.byref(out)), "adaqp_ipc_open")
        self._opened[int(out.value)] = 1
        return int(out.value)

    def view(self, offset: int, shape, dtype: torch.dtype) -> torch.Tensor:
        """Zero-copy torch view of a slab region (the slab outlives all views)."""
        n = int(np.prod(shape)) if len(shape) else 1
        itemsize = torch.empty((), dtype=dtype).element_size()
        assert offset + n * itemsize <= self.nbytes
        typestr = {torch.float32: "<f4", torch.int8: "|i1", torch.uint8: "|u1",
                   torch.int16: "<i2", torch.int32: "<i4", torch.bfloat16: "<i2"}[dtype]

        class _Holder:
            pass

        h = _Holder()
        h.__cuda_array_interface__ = {"shape": tuple(int(s) for s in shape), "typestr": typestr,
                                      "data": (self.ptr + offset, False), "version": 2}
        t = torch.as_tensor(h, device=self.device)
        if dtype == torch.bfloat16:
            t = t.view(torch.bfloat16)
        return t

    def close(self):
        L = _lib.load()
        for p in list(self._opened):
            L.adaqp_ipc_close(p)
        self._opened.clear()
        if self.ptr:
            L.adaqp_slab_free(self.ptr)
            self.ptr = 0


def _to_device_bytes(arr: np.ndarray, device) -> torch.Tensor:
    if arr.size == 0:
        return torch.zeros(8, dtype=torch.uint8, device=device)
    return torch.from_numpy(arr.view(np.uint8).reshape(-1).copy()).to(device)


# ------------------------------------------------------------------------------ plans
@dataclass
class FpPlan:
    items: torch.Tensor          # adaqp_fp_item[], gathering from the local message matrix
    items_compat: torch.Tensor   # same with src_row = position in send_messages
    n_items: int
    chans: torch.Tensor
    n_chans: int
    flags_ptrs: torch.Tensor     # const uint32_t*[n_recv] local flags to wait on
    acks_ptrs: torch.Tensor      # uint32_t*[n_recv] peer-mapped ack words
    n_recv: int


@dataclass
class QuantPlan:
    send_items: torch.Tensor
    send_items_compat: torch.Tensor
    n_send: int
    send_chans: torch.Tensor
    n_send_chans: int
    recv_items: torch.Tensor
    n_recv: int
    recv_chans: torch.Tensor
    n_recv_chans: int
    philox_increment: int        # total generator advance of one exchange
    wire: Dict[int, Tuple[int, int]]   # src peer -> (qdata bytes, rows) of the reference wire format


def build_send_items(send_peers: Sequence[int], send_idx: Dict[int, Tuple[int, int]], total_send_idx: np.ndarray,
                     bits_by_peer: Dict[int, np.ndarray], F: int) -> Tuple[np.ndarray, int]:
    """Sender work items of one layer key (pure host code, unit-tested against the oracle's wire
    layout): for each peer in dict order, for each bit-width in (2, 4, 8) with rows, one item per
    byte-row.  Mirrors the loop nest of op_util.py:194-209 / buffer.py:195-204: segment k of a
    peer starts at the sum of the previous segments' qsize (payload + 1 unwritten byte), its rows
    are the ascending local ids with that bit-width, and every segment consumes one
    philox_engine_inputs(F * 8/bits) of the generator.  Returns (items, total generator advance)."""
    items: List[np.ndarray] = []
    rel = 0
    for ci, p in enumerate(send_peers):
        lo, hi = send_idx[p]
        bits_p = np.asarray(bits_by_peer[p])
        assert bits_p.size == hi - lo
        seg_off = prm_off = 0
        for b in BITS_SET:
            ids = np.nonzero(bits_p == b)[0]          # ascending local ids (torch.nonzero)
            if ids.size == 0:
                continue
            wpt = 8 // b
            g = (ids.size + wpt - 1) // wpt
            it = np.zeros(g, _lib.SEND_ITEM_DTYPE)
            pos = np.full(g * wpt, -1, np.int64)
            pos[:ids.size] = lo + ids
            pos = pos.reshape(g, wpt)
            it["send_pos"][:, :wpt] = pos
            it["send_pos"][:, wpt:] = -1
            it["src_row"][:, :wpt] = np.where(pos >= 0, total_send_idx[np.maximum(pos, 0)], -1)
            it["src_row"][:, wpt:] = -1
            it["dst_off"] = seg_off + np.arange(g, dtype=np.int64) * F
            it["param_pos"] = prm_off + np.arange(g, dtype=np.int64) * wpt
            it["group"] = np.arange(g)
            it["rel_offset"] = rel
            it["chan"] = ci
            it["bits"] = b
            it["nrows"] = np.minimum(wpt, ids.size - np.arange(g) * wpt)
            items.append(it)
            seg_off += qsize(ids.size, b, F)
            prm_off += ids.size
            rel += ((F * wpt + 3) // 4) * 4          # philox_engine_inputs rounding
    out = np.concatenate(items) if items else np.zeros(0, _lib.SEND_ITEM_DTYPE)
    return out, rel


def build_push_items(recv_peers: Sequence[int], recv_idx: Dict[int, np.ndarray],
                     owner_send_idx: Dict[int, Tuple[int, int]]) -> np.ndarray:
    """Holder-side work items of a push key (pure host code): for each peer p in recv order, halo row recv_idx[p][j]
    goes to row lo + j of p's push region, where (lo, hi) = p's send_idx[me], the same rows in the same order as p
    sent them."""
    items = np.zeros(int(sum(np.asarray(recv_idx[p]).size for p in recv_peers)), _lib.FP_ITEM_DTYPE)
    n = 0
    for ci, p in enumerate(recv_peers):
        ridx = np.asarray(recv_idx[p], np.int64)
        lo, hi = owner_send_idx[p]
        if hi - lo != ridx.size:
            raise RuntimeError(f"peer {p} sends {hi - lo} rows, {ridx.size} expected")
        sl = items[n:n + ridx.size]
        sl["src_row"] = ridx
        sl["chan"] = ci
        sl["dst_row"] = lo + np.arange(ridx.size, dtype=np.int64)
        n += ridx.size
    return items


def build_recv_items(recv_peers: Sequence[int], recv_idx: Dict[int, np.ndarray], bits_from_peer: Dict[int, np.ndarray],
                     F: int) -> Tuple[np.ndarray, Dict[int, Tuple[int, int]]]:
    """Receiver work items (op_util.py:216-235): segment layout as on the sender; row j of a segment
    lands at halo row recv_idx[p][orig_ids[j]].  Returns (items, {peer: (wire bytes, rows)})."""
    items: List[np.ndarray] = []
    wire: Dict[int, Tuple[int, int]] = {}
    for ci, p in enumerate(recv_peers):
        bits_p = np.asarray(bits_from_peer[p])
        ridx = np.asarray(recv_idx[p])
        assert bits_p.size == ridx.size
        seg_off = prm_off = 0
        for b in BITS_SET:
            ids = np.nonzero(bits_p == b)[0]
            if ids.size == 0:
                continue
            wpt = 8 // b
            g = (ids.size + wpt - 1) // wpt
            it = np.zeros(g, _lib.RECV_ITEM_DTYPE)
            dst = np.full(g * wpt, -1, np.int64)
            dst[:ids.size] = ridx[ids]                # remote[recv_idx[p]][orig_ids]
            it["dst_row"][:, :wpt] = dst.reshape(g, wpt)
            it["dst_row"][:, wpt:] = -1
            it["src_off"] = seg_off + np.arange(g, dtype=np.int64) * F
            it["param_pos"] = prm_off + np.arange(g, dtype=np.int64) * wpt
            it["chan"] = ci
            it["bits"] = b
            it["nrows"] = np.minimum(wpt, ids.size - np.arange(g) * wpt)
            items.append(it)
            seg_off += qsize(ids.size, b, F)
            prm_off += ids.size
        wire[p] = (seg_off, int(ridx.size))
    out = np.concatenate(items) if items else np.zeros(0, _lib.RECV_ITEM_DTYPE)
    return out, wire


class PeerExchange:
    """Data plane of one rank.

    send_idx / recv_idx / total_send_idx follow the reference's contract
    (conversion.py:92-106, processing.py:53-60).  `gather(obj) -> list` is the control
    plane all_gather (comm.all_gather_any in multi-process runs; tests wire ranks
    in-process through `connect`).  `key_dims` (ordered key -> row width, e.g. gat_key_dims) replaces the
    default table, layer_key_dims(buffer_shape)."""

    def __init__(self, rank: int, world_size: int, device: torch.device, buffer_shape: Sequence[int],
                 send_idx: Dict[int, Tuple[int, int]], recv_idx: Dict[int, torch.Tensor],
                 total_send_idx: torch.Tensor, num_remote: int, timeout_ns: int = DEFAULT_TIMEOUT_NS,
                 key_dims: Optional[Dict[str, int]] = None):
        self.rank, self.world_size, self.device = rank, world_size, torch.device(device)
        self.buffer_shape = [int(x) for x in buffer_shape]
        self.num_layers = len(self.buffer_shape)
        if key_dims is None:
            key_dims = layer_key_dims(self.buffer_shape)
        self.keys = list(key_dims)
        self.dims = {k: int(v) for k, v in key_dims.items()}
        self.send_idx = {int(p): (int(lo), int(hi)) for p, (lo, hi) in send_idx.items()}
        self.recv_idx = {int(p): torch.as_tensor(v).cpu().numpy().astype(np.int64) for p, v in recv_idx.items()}
        self.total_send_idx = torch.as_tensor(total_send_idx).cpu().numpy().astype(np.int64)
        self.num_remote = int(num_remote)
        self.timeout_ns = int(timeout_ns)
        self.send_peers = list(self.send_idx.keys())       # dict order, as the reference iterates
        self.recv_peers = list(self.recv_idx.keys())
        self.seq = {k: 0 for k in self.keys}
        self.layouts: Dict[int, SlabLayout] = {}
        self.peer_base: Dict[int, int] = {}
        self.peer_recv_idx: Dict[int, np.ndarray] = {}      # peer -> peer's recv_idx[me]
        self.peer_send_idx: Dict[int, Tuple[int, int]] = {}  # peer -> peer's send_idx[me]
        self.fp_plans: Dict[str, FpPlan] = {}
        self.quant_plans: Dict[str, QuantPlan] = {}
        self.slab: Optional[Slab] = None
        self._lib = _lib.load()
        # kernel-alone timings (bench / profiling only): when `profile` is set every send / receive launch is
        # bracketed by CUDA events on its own stream; resolved by kernel_times_ms()
        self.profile = False
        self._prof: Dict[str, List[Tuple[torch.cuda.Event, torch.cuda.Event]]] = {"send": [], "recv": []}

    # ---- rendezvous ---------------------------------------------------------------
    def local_meta(self) -> dict:
        """What the other ranks need to know about me (all-gathered by the caller)."""
        return {"rank": self.rank,
                "recv_rows": {p: int(v.size) for p, v in self.recv_idx.items()},
                "num_remote": self.num_remote,
                "recv_idx": self.recv_idx,
                "send_idx": self.send_idx,
                "total_send": int(self.total_send_idx.size)}

    def allocate(self, metas: List[dict]):
        for m in metas:
            self.layouts[m["rank"]] = SlabLayout.build(self.world_size, self.keys, self.dims,
                                                       m["recv_rows"], m["num_remote"], m["total_send"])
            if m["rank"] != self.rank and self.rank in m["recv_idx"]:
                self.peer_recv_idx[m["rank"]] = np.asarray(m["recv_idx"][self.rank], np.int64)
            if m["rank"] != self.rank and self.rank in m["send_idx"]:
                self.peer_send_idx[m["rank"]] = tuple(int(x) for x in m["send_idx"][self.rank])
        for p, (lo, hi) in self.send_idx.items():
            want = self.layouts[p].recv_rows.get(self.rank, 0)
            if want != hi - lo:
                raise RuntimeError(f"rank {self.rank}: send count to {p} is {hi - lo}, peer expects {want}")
        self.layout = self.layouts[self.rank]
        self.slab = Slab(self.layout.total, self.device)
        self.peer_base[self.rank] = self.slab.ptr
        lay = self.layout
        self.status = self.slab.view(lay.status_off, (4,), torch.int32)
        return self.slab

    def connect(self, peer_bases: Dict[int, int]):
        """peer rank -> device pointer of its slab as seen from this process."""
        self.peer_base.update({int(p): int(b) for p, b in peer_bases.items()})
        self._build_fp_plans()

    # ---- helpers ------------------------------------------------------------------
    def _work_ptr(self, key: str, side: int) -> int:
        return self.slab.ptr + self.layout.work_off + 8 * self.keys.index(key) + 4 * side

    def halo(self, key: str) -> torch.Tensor:
        """The received rows of a key: [num_remote, F], or for a push key the push region [len(total_send_idx), F]
        (row i holds the gradient pushed for send position i)."""
        F = self.dims[key]
        rows = self.layout.push_rows if is_push(key) else self.num_remote
        return self.slab.view(self.layout.halo_off[key], (rows, F), torch.float32)

    def recv_region(self, key: str, p: int) -> Tuple[torch.Tensor, torch.Tensor]:
        """(int8[sum q], bf16[2, S]) views of what peer p wrote: the tensors the reference
        holds in train_recv_buffers_gpu[key][p] (buffer.py:240-248)."""
        nbytes, rows = self.quant_plans[key].wire[p]
        q = self.slab.view(self.layout.qdata_off[(key, p)], (nbytes,), torch.int8)
        prm = self.slab.view(self.layout.params_off[(key, p)], (2, rows), torch.bfloat16)
        return q, prm

    def check_status(self):
        st = self.status.cpu().tolist()
        if st[0] != 0:
            kind = {1: "flag", 2: "ack"}.get(st[0], str(st[0]))
            raise RuntimeError(f"rank {self.rank}: {kind} wait timed out on channel {st[1]}")

    # ---- fp32 plans ---------------------------------------------------------------
    def _build_fp_plans(self):
        me = self.rank
        for key in self.keys:
            if is_push(key):
                self._build_push_plan(key)
                continue
            F = self.dims[key]
            items = np.zeros(int(sum(hi - lo for lo, hi in self.send_idx.values())), _lib.FP_ITEM_DTYPE)
            chans = np.zeros(len(self.send_peers), _lib.SEND_CHAN_DTYPE)
            n = 0
            for ci, p in enumerate(self.send_peers):
                lo, hi = self.send_idx[p]
                lay_p = self.layouts[p]
                chans[ci]["fp_rows"] = self.peer_base[p] + lay_p.halo_off[key]
                chans[ci]["flag"] = self.peer_base[p] + lay_p.flag_off[key] + 4 * me
                chans[ci]["ack"] = self.slab.ptr + self.layout.ack_off[key] + 4 * p
                chans[ci]["S"] = hi - lo
                sl = items[n:n + hi - lo]
                sl["src_row"] = self.total_send_idx[lo:hi]
                sl["chan"] = ci
                sl["dst_row"] = self.peer_recv_idx[p]
                n += hi - lo
            compat = items.copy()
            compat["src_row"] = np.arange(items.size, dtype=np.int32)
            flags = np.array([self.slab.ptr + self.layout.flag_off[key] + 4 * p for p in self.recv_peers], np.uint64)
            acks = np.array([self.peer_base[p] + self.layouts[p].ack_off[key] + 4 * me for p in self.recv_peers], np.uint64)
            self.fp_plans[key] = FpPlan(
                items=_to_device_bytes(items, self.device), items_compat=_to_device_bytes(compat, self.device),
                n_items=int(items.size), chans=_to_device_bytes(chans, self.device), n_chans=len(self.send_peers),
                flags_ptrs=_to_device_bytes(flags, self.device), acks_ptrs=_to_device_bytes(acks, self.device),
                n_recv=len(self.recv_peers))

    def _build_push_plan(self, key: str):
        """The roles of _build_fp_plans swapped: I send my halo rows to their owners (my recv peers) and wait on the
        flags of, and ack, the peers I send to in the forward direction."""
        me = self.rank
        items = build_push_items(self.recv_peers, self.recv_idx, self.peer_send_idx)
        chans = np.zeros(len(self.recv_peers), _lib.SEND_CHAN_DTYPE)
        for ci, p in enumerate(self.recv_peers):
            lay_p = self.layouts[p]
            chans[ci]["fp_rows"] = self.peer_base[p] + lay_p.halo_off[key]
            chans[ci]["flag"] = self.peer_base[p] + lay_p.flag_off[key] + 4 * me
            chans[ci]["ack"] = self.slab.ptr + self.layout.ack_off[key] + 4 * p
            chans[ci]["S"] = self.recv_idx[p].size
        flags = np.array([self.slab.ptr + self.layout.flag_off[key] + 4 * p for p in self.send_peers], np.uint64)
        acks = np.array([self.peer_base[p] + self.layouts[p].ack_off[key] + 4 * me for p in self.send_peers], np.uint64)
        dev_items = _to_device_bytes(items, self.device)
        self.fp_plans[key] = FpPlan(
            items=dev_items, items_compat=dev_items, n_items=int(items.size), chans=_to_device_bytes(chans, self.device),
            n_chans=len(self.recv_peers), flags_ptrs=_to_device_bytes(flags, self.device),
            acks_ptrs=_to_device_bytes(acks, self.device), n_recv=len(self.send_peers))

    # ---- quantised plans ----------------------------------------------------------
    def quant_meta(self, assignment: Dict[str, Dict[int, torch.Tensor]]) -> dict:
        """Per-key per-destination bit-width of every row I send (all-gathered so that
        receivers learn the segment layout, as buffer.py:219-231 does)."""
        return {key: {int(p): np.asarray(torch.as_tensor(b).cpu().numpy(), np.int8) for p, b in per.items()}
                for key, per in assignment.items()}

    def update_quant(self, metas: List[dict]):
        """(Re)build send/recv tables from every rank's assignment (CommBuffer._update)."""
        me = self.rank
        self.quant_plans.clear()
        mine = metas[me]
        for key in mine:
            F = self.dims[key]
            chans = np.zeros(len(self.send_peers), _lib.SEND_CHAN_DTYPE)
            for ci, p in enumerate(self.send_peers):
                lo, hi = self.send_idx[p]
                lay_p = self.layouts[p]
                chans[ci]["qdata"] = self.peer_base[p] + lay_p.qdata_off[(key, me)]
                chans[ci]["params"] = self.peer_base[p] + lay_p.params_off[(key, me)]
                chans[ci]["flag"] = self.peer_base[p] + lay_p.flag_off[key] + 4 * me
                chans[ci]["ack"] = self.slab.ptr + self.layout.ack_off[key] + 4 * p
                chans[ci]["S"] = hi - lo
            send_items, rel = build_send_items(self.send_peers, self.send_idx, self.total_send_idx,
                                               {p: np.asarray(mine[key][p]) for p in self.send_peers}, F)
            compat = send_items.copy()
            compat["src_row"] = compat["send_pos"]
            rchans = np.zeros(len(self.recv_peers), _lib.RECV_CHAN_DTYPE)
            for ci, p in enumerate(self.recv_peers):
                rchans[ci]["qdata"] = self.slab.ptr + self.layout.qdata_off[(key, p)]
                rchans[ci]["params"] = self.slab.ptr + self.layout.params_off[(key, p)]
                rchans[ci]["flag"] = self.slab.ptr + self.layout.flag_off[key] + 4 * p
                rchans[ci]["ack"] = self.peer_base[p] + self.layouts[p].ack_off[key] + 4 * me
                rchans[ci]["S"] = self.recv_idx[p].size
            recv_items, wire = build_recv_items(self.recv_peers, self.recv_idx,
                                                {p: np.asarray(metas[p][key][me]) for p in self.recv_peers}, F)
            self.quant_plans[key] = QuantPlan(
                send_items=_to_device_bytes(send_items, self.device),
                send_items_compat=_to_device_bytes(compat, self.device), n_send=int(send_items.size),
                send_chans=_to_device_bytes(chans, self.device), n_send_chans=len(self.send_peers),
                recv_items=_to_device_bytes(recv_items, self.device), n_recv=int(recv_items.size),
                recv_chans=_to_device_bytes(rchans, self.device), n_recv_chans=len(self.recv_peers),
                philox_increment=rel, wire=wire)

    # ---- profiling ----------------------------------------------------------------
    def _bracket(self, kind: str, stream):
        if not self.profile:
            return None
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        a = torch.cuda.Event(enable_timing=True)
        a.record(st)
        return (kind, st, a)

    def _close(self, tok):
        if tok is None:
            return
        kind, st, a = tok
        b = torch.cuda.Event(enable_timing=True)
        b.record(st)
        self._prof[kind].append((a, b))

    def kernel_times_ms(self, clear: bool = True) -> Dict[str, float]:
        """Sum of the event-timed durations of the send / receive kernels since the last call."""
        torch.cuda.synchronize(self.device)
        out = {k: float(sum(a.elapsed_time(b) for a, b in v)) for k, v in self._prof.items()}
        out["launches"] = {k: len(v) for k, v in self._prof.items()}
        if clear:
            self._prof = {"send": [], "recv": []}
        return out

    # ---- launches -----------------------------------------------------------------
    def _next_seq(self, key: str) -> int:
        self.seq[key] += 1
        return self.seq[key]

    def post_send_fp(self, key: str, x: torch.Tensor, gathered: bool = False, stream=None) -> int:
        """Launch the fp32 gather + peer store kernel.  x = local message matrix, or the
        already gathered send_messages when gathered=True (msg_all2all_GLOO signature)."""
        plan = self.fp_plans[key]
        F = self.dims[key]
        assert x.dtype == torch.float32 and x.shape[1] == F and x.stride(1) == 1
        assert not (gathered and is_push(key)), "a push key sends the halo rows in place"
        seq = self._next_seq(key)
        items = plan.items_compat if gathered else plan.items
        tok = self._bracket("send", stream)
        rc = self._lib.adaqp_send_fp32(x.data_ptr(), x.stride(0), F, items.data_ptr(), plan.n_items,
                                       plan.chans.data_ptr(), plan.n_chans, F, seq,
                                       self._work_ptr(key, 0), self.status.data_ptr(), self.timeout_ns,
                                       _lib.stream_ptr(stream))
        _lib.check(rc, "adaqp_send_fp32")
        self._close(tok)
        return seq

    def complete_recv_fp(self, key: str, stream=None) -> torch.Tensor:
        plan = self.fp_plans[key]
        rc = self._lib.adaqp_wait_flags(plan.flags_ptrs.data_ptr(), plan.n_recv, self.seq[key],
                                        self.status.data_ptr(), self.timeout_ns, _lib.stream_ptr(stream))
        _lib.check(rc, "adaqp_wait_flags")
        return self.halo(key)

    def wait_flags_quant(self, key: str, stream=None):
        """One-CTA flag wait ahead of the receive kernel, so that a full grid never spins on
        SMs the overlapped aggregation could use."""
        plan = self.fp_plans[key]
        rc = self._lib.adaqp_wait_flags(plan.flags_ptrs.data_ptr(), plan.n_recv, self.seq[key],
                                        self.status.data_ptr(), self.timeout_ns, _lib.stream_ptr(stream))
        _lib.check(rc, "adaqp_wait_flags")

    def release_fp(self, key: str, stream=None):
        """After the consumer of halo(key) has been enqueued: let the senders overwrite it."""
        plan = self.fp_plans[key]
        rc = self._lib.adaqp_post_acks(plan.acks_ptrs.data_ptr(), plan.n_recv, self.seq[key],
                                       _lib.stream_ptr(stream))
        _lib.check(rc, "adaqp_post_acks")

    def post_send_quant(self, key: str, x: torch.Tensor, seed: int, base_offset: int,
                        trace: Optional[torch.Tensor] = None, gathered: bool = False, stream=None) -> int:
        plan = self.quant_plans[key]
        F = self.dims[key]
        assert x.dtype == torch.float32 and x.shape[1] == F and x.stride(1) == 1
        seq = self._next_seq(key)
        items = plan.send_items_compat if gathered else plan.send_items
        tok = self._bracket("send", stream)
        rc = self._lib.adaqp_send_quant(x.data_ptr(), x.stride(0), F, items.data_ptr(), plan.n_send,
                                        plan.send_chans.data_ptr(), plan.n_send_chans,
                                        trace.data_ptr() if trace is not None else None,
                                        seed, base_offset, seq, self._work_ptr(key, 0),
                                        self.status.data_ptr(), self.timeout_ns, _lib.stream_ptr(stream))
        _lib.check(rc, "adaqp_send_quant")
        self._close(tok)
        return seq

    def complete_recv_quant(self, key: str, stream=None) -> torch.Tensor:
        plan = self.quant_plans[key]
        F = self.dims[key]
        halo = self.halo(key)
        tok = self._bracket("recv", stream)
        rc = self._lib.adaqp_recv_quant(halo.data_ptr(), F, F, plan.recv_items.data_ptr(), plan.n_recv,
                                        plan.recv_chans.data_ptr(), plan.n_recv_chans, self.seq[key],
                                        self._work_ptr(key, 1), self.status.data_ptr(), self.timeout_ns,
                                        _lib.stream_ptr(stream))
        _lib.check(rc, "adaqp_recv_quant")
        self._close(tok)
        return halo

    def close(self):
        if self.slab is not None:
            self.slab.close()
            self.slab = None


def wire_in_process(exchanges: List[PeerExchange]):
    """Single-process simulation of W ranks on one device (tests, smoke): every rank's
    slab is directly addressable, so peer pointers are the slabs' own addresses."""
    metas = [e.local_meta() for e in exchanges]
    for e in exchanges:
        e.allocate(metas)
    bases = {e.rank: e.slab.ptr for e in exchanges}
    for e in exchanges:
        e.connect(bases)
    return exchanges


def update_quant_in_process(exchanges: List[PeerExchange], assignments: List[Dict[str, Dict[int, torch.Tensor]]]):
    metas = [e.quant_meta(a) for e, a in zip(exchanges, assignments)]
    for e in exchanges:
        e.update_quant(metas)

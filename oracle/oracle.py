"""CPU oracle for the AdaQP boundary-exchange + aggregation path.

TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, __graft_entry__.smoke()
and bench.py's cpu_baseline / --impl reference legs may import this module.
adaqp_b200/ never imports it.

numpy + ctypes front end of oracle/quant_oracle.c plus numpy restatements of
the reference's host-side orchestration (paths relative to the reference tree, raywan-110/AdaQP):

  mixed_quantize     AdaQP/model/op_util.py:189-209 + AdaQP/communicator/buffer.py:176-204
  mixed_dequantize   AdaQP/model/op_util.py:211-236
  exchange_*         AdaQP/model/op_util.py:137-187, AdaQP/communicator/comm.py:166-222
  gcn_aggregation    AdaQP/model/ops.py:17-32
  sage_aggregation   AdaQP/model/ops.py:34-67 (mean)
  sage_gcn_aggregation  AdaQP/model/ops.py:34-67 (gcn)
  full/decomposed propagation   AdaQP/model/ops.py:132-193

Parity pinning: see the header of quant_oracle.c (reference quant_cuda outputs
recorded under tests/golden/ + Philox known-answer vectors).
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Sequence, Tuple

import numpy as np

from . import build as _build

BITS_SET = (2, 4, 8)  # buffer.py:20

_lib = None


def lib():
    global _lib
    if _lib is None:
        path = _build.build_oracle()
        L = C.CDLL(path)
        u32p = C.POINTER(C.c_uint32)
        f32p = C.POINTER(C.c_float)
        u8p = C.POINTER(C.c_uint8)
        u16p = C.POINTER(C.c_uint16)
        i64p = C.POINTER(C.c_int64)
        f64p = C.POINTER(C.c_double)
        L.oracle_philox4x32_10.argtypes = [u32p, u32p, u32p]
        L.oracle_curand_uniform.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.c_int]
        L.oracle_curand_uniform.restype = C.c_float
        L.oracle_pack.argtypes = [f32p, f32p, f32p, C.c_int64, C.c_int64, C.c_int,
                                  C.c_uint64, C.c_uint64, u8p]
        L.oracle_pack_at.argtypes = [f32p, f32p, f32p, C.c_int64, C.c_int64, C.c_int,
                                     C.c_uint64, C.c_uint64, C.c_int64, u8p]
        L.oracle_unpack.argtypes = [u8p, f32p, f32p, C.c_int64, C.c_int64, C.c_int, f32p]
        L.oracle_pack_f16.argtypes = [u16p, u16p, u16p, C.c_int64, C.c_int64, C.c_int, C.c_uint64, C.c_uint64, u8p]
        L.oracle_unpack_f16.argtypes = [u8p, u16p, u16p, C.c_int64, C.c_int64, C.c_int, u16p]
        L.oracle_half_to_float_n.argtypes = [u16p, C.c_int64, f32p]
        L.oracle_float_to_half_n.argtypes = [f32p, C.c_int64, u16p]
        L.oracle_minmax_scale.argtypes = [f32p, C.c_int64, C.c_int64, C.c_int, f32p, f32p, f32p]
        L.oracle_f32_to_bf16_n.argtypes = [f32p, C.c_int64, u16p]
        L.oracle_bf16_to_f32_n.argtypes = [u16p, C.c_int64, f32p]
        L.oracle_aggregate.argtypes = [i64p, i64p, f32p, f32p, f32p, C.c_int64, C.c_int64,
                                       C.c_int, f64p]
        _lib = L
    return _lib


def _p(a: np.ndarray, ct):
    return a.ctypes.data_as(C.POINTER(ct))


def _f32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32)


# --------------------------------------------------------------------------
# RNG
# --------------------------------------------------------------------------
def philox4x32_10(ctr: Sequence[int], key: Sequence[int]) -> Tuple[int, int, int, int]:
    c = np.array(ctr, dtype=np.uint32)
    k = np.array(key, dtype=np.uint32)
    o = np.zeros(4, dtype=np.uint32)
    lib().oracle_philox4x32_10(_p(c, C.c_uint32), _p(k, C.c_uint32), _p(o, C.c_uint32))
    return tuple(int(x) for x in o)


def curand_uniform(seed: int, subsequence: int, offset: int, i: int = 0) -> float:
    return float(lib().oracle_curand_uniform(seed, subsequence, offset, i))


def philox_offset_increment(F: int, bits: int) -> int:
    """What one pack call adds to the CUDA generator's Philox offset:
    philox_engine_inputs(F * 8/bits) rounds the increment up to a multiple of 4
    (quantization_cuda_kernel.cu:71; ATen CUDAGeneratorImpl)."""
    inc = F * (8 // bits)
    return ((inc + 3) // 4) * 4


# --------------------------------------------------------------------------
# single-precision codec (quant_cuda.pack/unpack_single_precision)
# --------------------------------------------------------------------------
def packed_nbytes(N: int, F: int, bits: int) -> int:
    """Bytes the pack kernel writes."""
    wpt = 8 // bits
    return ((N + wpt - 1) // wpt) * F


def qsize(N: int, F: int, bits: int) -> int:
    """Length of the tensor pack returns (buffer.py:181-186): payload + 1."""
    wpt = 8 // bits
    n_round = N + (wpt - N % wpt) % wpt
    return (bits * n_round * F + 8) // 8


def pack(data, mn, scale, bits: int, seed: int, offset: int) -> np.ndarray:
    data = _f32(data)
    N, F = data.shape
    mn = _f32(mn)
    scale = _f32(scale)
    out = np.zeros(packed_nbytes(N, F, bits), dtype=np.uint8)
    lib().oracle_pack(_p(data, C.c_float), _p(mn, C.c_float), _p(scale, C.c_float),
                      N, F, bits, seed, offset, _p(out, C.c_uint8))
    return out


def pack_at(data, mn, scale, bits: int, seed: int, offset: int, group0: int) -> np.ndarray:
    """Bytes [group0*F, group0*F + ceil(N/wpt)*F) of a pack call whose rows
    [group0*wpt, group0*wpt + N) are `data` (same Philox subsequences as the full call)."""
    data = _f32(data)
    N, F = data.shape
    mn = _f32(mn)
    scale = _f32(scale)
    out = np.zeros(packed_nbytes(N, F, bits), dtype=np.uint8)
    if N:
        lib().oracle_pack_at(_p(data, C.c_float), _p(mn, C.c_float), _p(scale, C.c_float),
                             N, F, bits, seed, offset, group0, _p(out, C.c_uint8))
    return out


def unpack(packed, bits: int, scale, mn, N: int, F: int) -> np.ndarray:
    packed = np.ascontiguousarray(packed, dtype=np.uint8)
    assert packed.size >= packed_nbytes(N, F, bits)
    scale = _f32(scale)
    mn = _f32(mn)
    out = np.zeros((N, F), dtype=np.float32)
    lib().oracle_unpack(_p(packed, C.c_uint8), _p(scale, C.c_float), _p(mn, C.c_float),
                        N, F, bits, _p(out, C.c_float))
    return out


def _u16(a) -> np.ndarray:
    a = np.asarray(a)
    if a.dtype == np.float16:
        a = a.view(np.uint16)
    return np.ascontiguousarray(a, dtype=np.uint16)


def pack_f16(data, mn, scale, bits: int, seed: int, offset: int) -> np.ndarray:
    """fp16 instantiation of pack_single_precision; inputs are float16 arrays (or their uint16 bits)."""
    data, mn, scale = _u16(data), _u16(mn), _u16(scale)
    N, F = data.shape
    out = np.zeros(packed_nbytes(N, F, bits), dtype=np.uint8)
    if N:
        lib().oracle_pack_f16(_p(data, C.c_uint16), _p(mn, C.c_uint16), _p(scale, C.c_uint16), N, F, bits, seed, offset,
                              _p(out, C.c_uint8))
    return out


def unpack_f16(packed, bits: int, scale, mn, N: int, F: int) -> np.ndarray:
    packed = np.ascontiguousarray(packed, dtype=np.uint8)
    scale, mn = _u16(scale), _u16(mn)
    out = np.zeros((N, F), dtype=np.uint16)
    if N:
        lib().oracle_unpack_f16(_p(packed, C.c_uint8), _p(scale, C.c_uint16), _p(mn, C.c_uint16), N, F, bits, _p(out, C.c_uint16))
    return out.view(np.float16)


def half_roundtrip_check(f32: np.ndarray) -> np.ndarray:
    """float -> half bits with the oracle's own converter (tests compare it with numpy's)."""
    f32 = _f32(f32).reshape(-1)
    out = np.zeros(f32.size, np.uint16)
    lib().oracle_float_to_half_n(_p(f32, C.c_float), f32.size, _p(out, C.c_uint16))
    return out


def minmax_scale(data, bits: int):
    data = _f32(data)
    N, F = data.shape
    rmin = np.zeros(N, np.float32)
    rmax = np.zeros(N, np.float32)
    scale = np.zeros(N, np.float32)
    if N:
        lib().oracle_minmax_scale(_p(data, C.c_float), N, F, bits, _p(rmin, C.c_float),
                                  _p(rmax, C.c_float), _p(scale, C.c_float))
    return rmin, rmax, scale


def to_bf16(x) -> np.ndarray:
    x = _f32(x).reshape(-1)
    out = np.zeros(x.size, np.uint16)
    if x.size:
        lib().oracle_f32_to_bf16_n(_p(x, C.c_float), x.size, _p(out, C.c_uint16))
    return out


def from_bf16(h) -> np.ndarray:
    h = np.ascontiguousarray(h, dtype=np.uint16).reshape(-1)
    out = np.zeros(h.size, np.float32)
    if h.size:
        lib().oracle_bf16_to_f32_n(_p(h, C.c_uint16), h.size, _p(out, C.c_float))
    return out


# --------------------------------------------------------------------------
# mixed-bit wire format (one src -> dst channel of one layer key)
# --------------------------------------------------------------------------
def bit_groups(bits_assign) -> Dict[int, np.ndarray]:
    """buffer.py:195-204: per bit-width, ascending local row ids; empty bits skipped."""
    bits_assign = np.asarray(bits_assign)
    out = {}
    for b in BITS_SET:
        ids = np.nonzero(bits_assign == b)[0]
        if ids.size:
            out[b] = ids
    return out


def mixed_quantize(rows, bits_assign, seed: int, offset: int):
    """Quantize the rows sent to one peer (op_util.py:194-209).

    Returns (qdata uint8[sum qsize], params uint16[2, S] (bf16 bits), valid
    mask over qdata (False on each segment's unwritten trailing byte), offset
    after the calls).  Segments in bit order (2,4,8); one pack call -- i.e. one
    generator advance -- per non-empty segment."""
    rows = _f32(rows)
    S, F = rows.shape
    groups = bit_groups(bits_assign)
    qparts: List[np.ndarray] = []
    vparts: List[np.ndarray] = []
    sc: List[np.ndarray] = []
    mnl: List[np.ndarray] = []
    for b, ids in groups.items():
        sub = rows[ids]
        rmin, _rmax, scale = minmax_scale(sub, b)
        payload = pack(sub, rmin, scale, b, seed, offset)
        offset += philox_offset_increment(F, b)
        seg = np.zeros(qsize(len(ids), F, b), np.uint8)
        seg[:payload.size] = payload
        valid = np.zeros(seg.size, bool)
        valid[:payload.size] = True
        qparts.append(seg)
        vparts.append(valid)
        sc.append(to_bf16(scale))
        mnl.append(to_bf16(rmin))
    if qparts:
        qdata = np.concatenate(qparts)
        valid = np.concatenate(vparts)
        params = np.stack([np.concatenate(sc), np.concatenate(mnl)], 0)
    else:
        qdata = np.zeros(0, np.uint8)
        valid = np.zeros(0, bool)
        params = np.zeros((2, 0), np.uint16)
    return qdata, params, valid, offset


def mixed_dequantize(qdata, params, bits_assign, F: int) -> np.ndarray:
    """Receiver side of one channel (op_util.py:216-235): returns the [S, F]
    sub-tensor in the sender's slice order (sub_remote_tensors)."""
    bits_assign = np.asarray(bits_assign)
    S = bits_assign.size
    out = np.zeros((S, F), np.float32)
    q_off = 0
    fp_off = 0
    for b, ids in bit_groups(bits_assign).items():
        n = ids.size
        qs = qsize(n, F, b)
        scale = from_bf16(params[0, fp_off:fp_off + n])
        rmin = from_bf16(params[1, fp_off:fp_off + n])
        out[ids] = unpack(qdata[q_off:q_off + qs], b, scale, rmin, n, F)
        q_off += qs
        fp_off += n
    return out


# --------------------------------------------------------------------------
# all-to-all halo exchange over W simulated ranks
# --------------------------------------------------------------------------
def exchange_fp(send_messages: List[np.ndarray], send_idx: List[Dict[int, Tuple[int, int]]],
                recv_idx: List[Dict[int, np.ndarray]], num_remote: List[int]) -> List[np.ndarray]:
    """fp32 exchange (op_util.py:156-171): remote[recv_idx[p]] = rows p sent."""
    W = len(send_messages)
    F = send_messages[0].shape[1]
    out = []
    for r in range(W):
        rem = np.zeros((num_remote[r], F), np.float32)
        for p, idx in recv_idx[r].items():
            lo, hi = send_idx[p][r]
            rem[idx] = send_messages[p][lo:hi]
        out.append(rem)
    return out


def exchange_quant(send_messages: List[np.ndarray], send_idx: List[Dict[int, Tuple[int, int]]],
                   recv_idx: List[Dict[int, np.ndarray]], num_remote: List[int],
                   assignment: List[Dict[int, np.ndarray]], seeds: List[int],
                   offsets: List[int], return_wire: bool = False):
    """Quantized exchange (op_util.py:173-236).  assignment[r][p] = int bits per
    row of rank r's slice for peer p.  Each rank's generator (seed, offset) is
    advanced peer by peer in send_idx dict order, bit by bit (2,4,8)."""
    W = len(send_messages)
    F = send_messages[0].shape[1]
    wire: List[Dict[int, tuple]] = [dict() for _ in range(W)]
    new_offsets = list(offsets)
    for r in range(W):
        off = offsets[r]
        for p, (lo, hi) in send_idx[r].items():
            q, prm, valid, off = mixed_quantize(send_messages[r][lo:hi], assignment[r][p], seeds[r], off)
            wire[r][p] = (q, prm, valid)
        new_offsets[r] = off
    out = []
    for r in range(W):
        rem = np.zeros((num_remote[r], F), np.float32)
        for p, idx in recv_idx[r].items():
            q, prm, _ = wire[p][r]
            rem[idx] = mixed_dequantize(q, prm, assignment[p][r], F)
        out.append(rem)
    if return_wire:
        return out, wire, new_offsets
    return out, new_offsets


# --------------------------------------------------------------------------
# aggregation
# --------------------------------------------------------------------------
def aggregate(indptr, indices, x, pre=None, post=None, mean: bool = False) -> np.ndarray:
    indptr = np.ascontiguousarray(indptr, np.int64)
    indices = np.ascontiguousarray(indices, np.int64)
    x = _f32(x)
    n_dst = indptr.size - 1
    F = x.shape[1]
    out = np.zeros((n_dst, F), np.float64)
    pre_p = post_p = None
    if pre is not None:
        pre = _f32(pre); pre_p = _p(pre, C.c_float)
    if post is not None:
        post = _f32(post); post_p = _p(post, C.c_float)
    lib().oracle_aggregate(_p(indptr, C.c_int64), _p(indices, C.c_int64), _p(x, C.c_float),
                           pre_p, post_p, n_dst, F, 1 if mean else 0, _p(out, C.c_double))
    return out


def _pow_clamped(deg, p: float) -> np.ndarray:
    """deg.float().clamp(min=1).pow(p) in fp32 (ops.py:21-25)."""
    d = np.maximum(np.asarray(deg, dtype=np.float32), np.float32(1.0))
    if p == -0.5:
        return (np.float32(1.0) / np.sqrt(d)).astype(np.float32)
    if p == -1:
        return (np.float32(1.0) / d).astype(np.float32)
    return np.power(d, np.float32(p)).astype(np.float32)


def gcn_aggregation(indptr, indices, feats, in_deg, out_deg, n_dst: int, backward: bool = False):
    """ops.py:17-32.  feats rows = all graph nodes (src side); in/out_deg are the
    GLOBAL degrees of those nodes; result rows = first n_dst nodes."""
    if not backward:
        norm1 = _pow_clamped(out_deg, -0.5)
        norm2 = _pow_clamped(in_deg, -0.5)
    else:
        norm1 = _pow_clamped(in_deg, -0.5)
        norm2 = _pow_clamped(out_deg, -0.5)
    return aggregate(indptr, indices, feats, pre=norm1, post=norm2[:n_dst])


def sage_aggregation(indptr, indices, feats, in_deg, out_deg, n_dst: int, backward: bool = False):
    """ops.py:34-67, aggregator_type='mean'."""
    if not backward:
        return aggregate(indptr, indices, feats, mean=True)
    norm = _pow_clamped(out_deg, -1)
    return aggregate(indptr, indices, feats, pre=norm)


def sage_gcn_aggregation(indptr, indices, feats, in_deg, out_deg, n_dst: int, backward: bool = False):
    """ops.py:34-67, aggregator_type='gcn' (the neighbourhood includes the node itself):
    forward  (sum_{u->v} x[u] + x[v]) / (clamp(in_deg[v], 1) + 1);
    backward sum_{u->v} x[u] / (clamp(out_deg[u], 1) + 1) + x[v] / (clamp(out_deg[v], 1) + 1).
    The norms are fp32 as in the reference (deg.float().clamp(min=1) + 1).pow(-1); the backward scales each
    row by its norm in fp32 before the float64 sum, as `aggregate` does."""
    x = _f32(feats)
    if not backward:
        post = _pow_clamped(np.maximum(np.asarray(in_deg, np.float32), np.float32(1.0)) + np.float32(1.0), -1)
        out = aggregate(indptr, indices, x) + x[:n_dst].astype(np.float64)
        return out * post[:n_dst, None].astype(np.float64)
    pre = _pow_clamped(np.maximum(np.asarray(out_deg, np.float32), np.float32(1.0)) + np.float32(1.0), -1)
    return aggregate(indptr, indices, x, pre=pre) + (x[:n_dst] * pre[:n_dst, None]).astype(np.float64)

"""Boundary-message exchange orchestration.

Mirror of AdaQP/model/op_util.py: the quantisation helpers (:20-83), the tracing /
stream decorators' behaviour (:91-130) and `msg_all2all_GLOO` (:137-153) keep their names
and signatures.  On the 'p2p' transport the whole chain

    gather -> per (peer, bit) min/max + pack + bf16 params -> D2H -> gloo -> H2D ->
    per (peer, bit) unpack -> scatter                      (op_util.py:156-236)

is two kernel launches (csrc/exchange.cu) driven by `halo_exchange`; the reference's loops
survive only on the 'gloo' transport (CPU plumbing / timed baseline).
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch
from torch import Tensor

from .. import quant as integer_quantizer
from ..assigner import Assigner as assigner
from ..communicator import Basic_Buffer_Type
from ..communicator import Communicator as comm
from ..communicator.p2p import layer_index
from ..helper import BitType
from ..manager import GraphEngine as engine


# ---------------------------------------------------------------- codec helpers (API parity)
def compute_minmax_params(input: Tensor) -> Tuple[Tensor, Tensor]:
    return torch.min(input, dim=1)[0], torch.max(input, dim=1)[0]


def integer_quantize(data: Tensor, bits: int, rmin: Tensor, rmax: Tensor, stochastic: bool = True):
    assert type(bits) == int
    scale = (2 ** bits - 1) / (rmax - rmin)
    q_data = integer_quantizer.pack_single_precision(data, rmin, rmax, scale.to(data.dtype), bits, stochastic)
    return q_data, scale


def integer_dequantize(q_data: Tensor, shape: torch.Size, bits: int, scale: Tensor, rmin: Tensor) -> Tensor:
    assert type(bits) == int
    return integer_quantizer.unpack_single_precision(q_data, bits, scale, rmin, shape[0], shape[1])


def message_quantization(input: Tensor, bits: int, stochastic: bool):
    rmin, rmax = compute_minmax_params(input)
    q_input, q_scale = integer_quantize(input, bits, rmin, rmax, stochastic=stochastic)
    if input.dtype == torch.float32:          # wire parameters travel as bf16 (op_util.py:72-74)
        return q_input, q_scale.to(torch.bfloat16), rmin.to(torch.bfloat16), input.shape
    return q_input, q_scale, rmin, input.shape


def message_dequantization(q_input: Tensor, q_scale: Tensor, rmin: Tensor, input_tempin_shape: torch.Size, bits):
    if q_scale.dtype == torch.bfloat16:
        q_scale, rmin = q_scale.to(torch.float32), rmin.to(torch.float32)
    return integer_dequantize(q_input, input_tempin_shape, bits, q_scale, rmin).contiguous()


# ---------------------------------------------------------------- fused p2p path
class PendingExchange(object):
    """Handle of an exchange whose kernels have been enqueued."""

    def __init__(self, key: str, halo: Tensor, fp: bool, stream):
        self.key, self.halo, self.fp, self.stream = key, halo, fp, stream

    def release(self, stream=None):
        """Enqueue the acks once the consumer of `halo` has been enqueued (fp32 path; the
        quantised receiver acks from inside its kernel)."""
        if self.fp:
            comm.ctx.comm_buffer.p2p.release_fp(self.key, stream)


def _trace_ptr(name: str, n_rows: int, device, stream=None) -> Optional[Tensor]:
    """trace_input (op_util.py:91-99) fused into the send kernel: the per-row
    (dim / 6) * (max - min)^2 accumulates into Assigner.traced_layer_data[name].
    The accumulator is allocated AND zero-filled on the stream the send kernel runs on, so the
    fill is ordered before the kernel's read-modify-write (the side stream in overlap modes)."""
    a = assigner.ctx
    if a is None or not a.is_tracing:
        return None
    cur = a.traced_layer_data.get(name)
    if not isinstance(cur, Tensor):
        with torch.cuda.stream(stream if stream is not None else torch.cuda.current_stream(device)):
            cur = torch.zeros(n_rows, dtype=torch.float32, device=device)
        a.traced_layer_data[name] = cur
    return cur


def halo_exchange(messages: Tensor, name: str, is_train: bool, gathered: bool = False, stream=None) -> PendingExchange:
    """Launch the exchange of one layer key on `stream` (current stream when None).
    `messages` is the local message matrix [num_inner, F], or send_messages when gathered."""
    ex = comm.ctx.comm_buffer.p2p
    quant = engine.ctx.bit_type == BitType.QUANT and is_train
    key = name if is_train else f"test{layer_index(name)}"
    if not quant:
        if assigner.ctx is not None and assigner.ctx.is_tracing:   # eval passes are traced too (op_util.py:91-99)
            _trace_rows(messages, name, gathered)
        ex.post_send_fp(key, messages, gathered=gathered, stream=stream)
        halo = ex.complete_recv_fp(key, stream=stream)
        return PendingExchange(key, halo, True, stream)
    plan = ex.quant_plans[key]
    seed, offset = integer_quantizer.philox_engine_inputs(messages.device, 0)
    # one philox_engine_inputs(F * 8/bits) per (peer, bit) pack call of the reference
    torch.cuda.default_generators[messages.device.index].set_offset(offset + plan.philox_increment)
    n_send = int(engine.ctx.total_send_idx.numel())
    ex.post_send_quant(key, messages, seed, offset, trace=_trace_ptr(name, n_send, messages.device, stream),
                       gathered=gathered, stream=stream)
    ex.wait_flags_quant(key, stream=stream)
    halo = ex.complete_recv_quant(key, stream=stream)
    return PendingExchange(key, halo, False, stream)


def _trace_rows(messages: Tensor, name: str, gathered: bool):
    rows = messages if gathered else messages[engine.ctx.total_send_idx]
    rmin, rmax = compute_minmax_params(rows)
    assigner.ctx.traced_layer_data[name] += (rows.shape[1] / 6) * (rmax - rmin) ** 2


# ---------------------------------------------------------------- reference entry point
def msg_all2all_GLOO(send_messages: Tensor, name: str, is_train: bool = True) -> Tensor:
    """All-to-all of already gathered boundary rows; returns remote_messages
    [num_remote, F] in halo order (op_util.py:137-153)."""
    assert comm.get_backend() == "gloo", "currently only gloo backend is supported"
    if comm.ctx.transport == "p2p":
        pend = halo_exchange(send_messages.contiguous(), name, is_train, gathered=True)
        out = pend.halo.clone()          # callers own the result; the slab row block is reused
        pend.release()
        return out
    if assigner.ctx is not None and assigner.ctx.is_tracing:
        _trace_rows(send_messages, name, True)
    msg_dim, msg_dtype = send_messages.shape[-1], send_messages.dtype
    if engine.ctx.bit_type == BitType.FULL or not is_train:
        return fp_msg_transfer_process(send_messages, engine.ctx.send_idx, engine.ctx.recv_idx, msg_dim,
                                       msg_dtype, engine.ctx.num_remove, name, is_train)
    return qt_msg_transfer_process(send_messages, engine.ctx.send_idx, engine.ctx.recv_idx, msg_dim,
                                   msg_dtype, engine.ctx.num_remove, name)


# ---------------------------------------------------------------- gloo transport (reference flow)
def fp_msg_transfer_process(send_messages, send_idx, recv_idx: Basic_Buffer_Type, msg_dim, msg_dtype,
                            num_remote, name, is_train) -> Tensor:
    buf = comm.ctx.comm_buffer
    recv_cpu, recv_gpu, send_cpu = buf.get_train_buffer(name) if is_train else buf.get_test_buffer(layer_index(name))
    with engine.ctx.timer.record(f"{name}_communication"):
        comm.ctx.fp_msg_exchange(recv_cpu, recv_gpu, send_cpu, send_idx, send_messages)
    remote = torch.zeros(num_remote, msg_dim, dtype=msg_dtype, device=comm.ctx.device)
    for pid, idx in recv_idx.items():
        remote[idx.to(remote.device)] = recv_gpu[pid]
    return remote


def qt_msg_transfer_process(send_messages, send_idx, recv_idx: Basic_Buffer_Type, msg_dim, msg_dtype,
                            num_remote, name) -> Tensor:
    buf = comm.ctx.comm_buffer
    recv_cpu, recv_gpu, send_cpu = buf.get_train_buffer(name)
    recv_orig_idx, recv_orig_size, send_orig_idx = buf.get_auxillary_buffer(name)
    with engine.ctx.timer.record(f"{name}_quantization"):
        mixed_msg_quantization(send_messages, send_idx, send_cpu, send_orig_idx)
    with engine.ctx.timer.record(f"{name}_communication"):
        comm.ctx.qt_msg_exchange(recv_cpu, recv_gpu, send_cpu)
    with engine.ctx.timer.record(f"{name}_de-quantization"):
        return mixed_msg_dequantization(recv_idx, recv_gpu, recv_orig_idx, recv_orig_size, msg_dim, msg_dtype, num_remote)


def mixed_msg_quantization(send_messages: Tensor, send_idx: Dict[int, Tuple[int, int]],
                           send_buffer_cpu: Basic_Buffer_Type, send_orig_idx_buffer: Dict[int, Dict[int, Tensor]]):
    """Per peer, per bit-width (2, 4, 8): quantise the rows of that group and append to the
    peer's byte stream; params stacked as bf16 [2, S] (op_util.py:189-209)."""
    for pid, (lo, hi) in send_idx.items():
        rows = send_messages[lo:hi]
        qs, scales, mins = [], [], []
        for bit, ids in send_orig_idx_buffer[pid].items():
            q, s, m, _ = message_quantization(rows[ids.to(rows.device)], bit, stochastic=True)
            qs.append(q)
            scales.append(s)
            mins.append(m)
        send_buffer_cpu[pid][0].copy_(torch.concat(qs), non_blocking=True)
        send_buffer_cpu[pid][1].copy_(torch.stack([torch.concat(scales), torch.concat(mins)], dim=0), non_blocking=True)
    if send_messages.is_cuda:
        torch.cuda.current_stream().synchronize()     # host buffers must be complete before isend


def mixed_msg_dequantization(recv_idx: Basic_Buffer_Type, recv_buffer_gpu: Basic_Buffer_Type,
                             recv_orig_idx_buffer, recv_orig_size_buffer, msg_dim: int, dtype: torch.dtype,
                             num_remote: int) -> Tensor:
    remote = torch.zeros(num_remote, msg_dim, dtype=dtype, device=comm.ctx.device)
    for pid, ids in recv_idx.items():
        q_all, prm = recv_buffer_gpu[pid]
        ids = ids.to(remote.device)
        sub = remote[ids]
        q_off = fp_off = 0
        for bit, (q_size, n_rows) in recv_orig_size_buffer[pid].items():
            orig = recv_orig_idx_buffer[pid][bit].to(remote.device)
            sub[orig] = message_dequantization(q_all[q_off:q_off + q_size].contiguous(), prm[0, fp_off:fp_off + n_rows].contiguous(),
                                               prm[1, fp_off:fp_off + n_rows].contiguous(), torch.Size((len(orig), msg_dim)), bit)
            q_off += q_size
            fp_off += n_rows
        remote[ids] = sub
    return remote

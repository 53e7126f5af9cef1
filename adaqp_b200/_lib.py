"""ctypes binding of libadaqp_b200.so (the C ABI in include/adaqp_b200.h).

There is NO fallback: if the CUDA library is missing or does not export every
symbol the header declares, importing the product path fails loudly.  Build it
with ``python -m adaqp_b200.build`` (or ``__graft_entry__.build()``).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libadaqp_b200.so")

c_void_p = C.c_void_p
i64 = C.c_int64
i32 = C.c_int32
u64 = C.c_uint64
u32 = C.c_uint32

ADAQP_ABI_VERSION = 9
MAX_PARTS = 64           # ADAQP_MAX_PARTS
LP_HUB_DEGREE = 256      # ADAQP_LP_HUB_DEGREE
IPC_HANDLE_BYTES = 64
ST_OK, ST_FLAG_TIMEOUT, ST_ACK_TIMEOUT = 0, 1, 2

# numpy mirrors of the plain-C structs (host-side table construction)
SEND_ITEM_DTYPE = np.dtype([
    ("src_row", np.int32, (4,)), ("send_pos", np.int32, (4,)), ("dst_off", np.int64),
    ("param_pos", np.int32), ("group", np.int32), ("rel_offset", np.uint32),
    ("chan", np.int16), ("bits", np.int8), ("nrows", np.int8), ("_pad", np.int32)],
    align=True)
RECV_ITEM_DTYPE = np.dtype([
    ("dst_row", np.int32, (4,)), ("src_off", np.int64), ("param_pos", np.int32),
    ("chan", np.int16), ("bits", np.int8), ("nrows", np.int8)], align=True)
FP_ITEM_DTYPE = np.dtype([("src_row", np.int32), ("chan", np.int32), ("dst_row", np.int64)],
                         align=True)
SEND_CHAN_DTYPE = np.dtype([
    ("qdata", np.uint64), ("params", np.uint64), ("fp_rows", np.uint64), ("flag", np.uint64),
    ("ack", np.uint64), ("S", np.int64)], align=True)
RECV_CHAN_DTYPE = np.dtype([
    ("qdata", np.uint64), ("params", np.uint64), ("flag", np.uint64), ("ack", np.uint64),
    ("S", np.int64)], align=True)
assert SEND_ITEM_DTYPE.itemsize == 64 and RECV_ITEM_DTYPE.itemsize == 32
assert FP_ITEM_DTYPE.itemsize == 16 and SEND_CHAN_DTYPE.itemsize == 48
assert RECV_CHAN_DTYPE.itemsize == 40

# symbol -> (restype, argtypes); this table IS the list of symbols the header declares
SYMBOLS = {
    "adaqp_abi_version": (C.c_int, []),
    "adaqp_last_error": (C.c_char_p, []),
    "adaqp_sm_count": (C.c_int, []),
    "adaqp_set_option": (C.c_int, [C.c_char_p, i64]),
    "adaqp_get_option": (C.c_int, [C.c_char_p, C.POINTER(i64)]),
    "adaqp_enable_peer_access": (C.c_int, [C.c_int]),
    "adaqp_packed_nbytes": (i64, [i64, i64, C.c_int]),
    "adaqp_qsize": (i64, [i64, i64, C.c_int]),
    "adaqp_pack_f32": (C.c_int, [c_void_p, c_void_p, c_void_p, i64, i64, C.c_int, u64, u64,
                                 c_void_p, c_void_p]),
    "adaqp_unpack_f32": (C.c_int, [c_void_p, c_void_p, c_void_p, i64, i64, C.c_int, c_void_p,
                                   c_void_p]),
    "adaqp_pack_f16": (C.c_int, [c_void_p, c_void_p, c_void_p, i64, i64, C.c_int, u64, u64, c_void_p, c_void_p]),
    "adaqp_unpack_f16": (C.c_int, [c_void_p, c_void_p, c_void_p, i64, i64, C.c_int, c_void_p, c_void_p]),
    "adaqp_row_minmax_f32": (C.c_int, [c_void_p, i64, i64, C.c_int, c_void_p, c_void_p, c_void_p,
                                       c_void_p]),
    "adaqp_slab_alloc": (C.c_int, [C.POINTER(c_void_p), C.c_size_t]),
    "adaqp_slab_free": (C.c_int, [c_void_p]),
    "adaqp_ipc_export": (C.c_int, [c_void_p, C.c_char_p]),
    "adaqp_ipc_open": (C.c_int, [C.c_char_p, C.POINTER(c_void_p)]),
    "adaqp_ipc_close": (C.c_int, [c_void_p]),
    "adaqp_can_access_peer": (C.c_int, [C.c_int]),
    "adaqp_send_quant": (C.c_int, [c_void_p, i64, i32, c_void_p, i64, c_void_p, i32, c_void_p,
                                   u64, u64, u32, c_void_p, c_void_p, u64, c_void_p]),
    "adaqp_recv_quant": (C.c_int, [c_void_p, i64, i32, c_void_p, i64, c_void_p, i32, u32,
                                   c_void_p, c_void_p, u64, c_void_p]),
    "adaqp_send_fp32": (C.c_int, [c_void_p, i64, i32, c_void_p, i64, c_void_p, i32, i64, u32,
                                  c_void_p, c_void_p, u64, c_void_p]),
    "adaqp_wait_flags": (C.c_int, [c_void_p, i32, u32, c_void_p, u64, c_void_p]),
    "adaqp_post_acks": (C.c_int, [c_void_p, i32, u32, c_void_p]),
    "adaqp_spmm_csr_f32": (C.c_int, [c_void_p, c_void_p, c_void_p, i64, i64, c_void_p, i64,
                                     c_void_p, c_void_p, C.c_int, C.c_int, i64, i64, i32,
                                     c_void_p, i64, c_void_p]),
    "adaqp_spmm_csr_seg_f32": (C.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, i64, i64, c_void_p,
                                         i64, c_void_p, c_void_p, C.c_int, C.c_int, C.c_int, i64, i64, i32,
                                         c_void_p, i64, c_void_p, c_void_p, i64, c_void_p]),
    "adaqp_row_live_f32": (C.c_int, [c_void_p, i64, i64, i32, c_void_p, c_void_p]),
    "adaqp_appnp_prop_f32": (C.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, i64, i64, c_void_p, i64,
                                       c_void_p, c_void_p, C.c_float, C.c_float, c_void_p, i64, c_void_p, i64, i32,
                                       C.c_int, i64, i64, i32, c_void_p, i64, c_void_p]),
    "adaqp_cs_prop_f32": (C.c_int, [c_void_p, c_void_p, c_void_p, i64, i64, c_void_p, i64, c_void_p, c_void_p,
                                    C.c_float, C.c_float, c_void_p, i64, c_void_p, c_void_p, i64, i32, C.c_float,
                                    C.c_float, i64, i64, i32, c_void_p, i64, c_void_p]),
    "adaqp_cs_init_f32": (C.c_int, [c_void_p, i64, c_void_p, i64, i32, c_void_p, i64, c_void_p, i64, c_void_p, i32,
                                    c_void_p]),
    "adaqp_cs_combine_f32": (C.c_int, [c_void_p, i64, c_void_p, i64, c_void_p, i64, i32, i32, C.c_double, c_void_p,
                                       i64, c_void_p]),
    "adaqp_gemm_tf32x3_supported": (C.c_int, [i64, i32, i32, i64, i64, i64]),
    "adaqp_gemm_tf32x3_f32": (C.c_int, [c_void_p, i64, c_void_p, c_void_p, i64, c_void_p, i64, i32, i32, c_void_p, i64, c_void_p]),
    "adaqp_wgrad_tf32x3_supported": (C.c_int, [i64, i32, i32, i64, i64]),
    "adaqp_wgrad_tf32x3_grid": (C.c_int, [i64]),
    "adaqp_wgrad_tf32x3_f32": (C.c_int, [c_void_p, i64, c_void_p, i64, i64, i32, i32, c_void_p, i32, c_void_p]),
    "adaqp_ln_relu_grid": (C.c_int, [i64]),
    "adaqp_ln_relu_fwd_f32": (C.c_int, [c_void_p, i64, c_void_p, c_void_p, C.c_float, i64, i32, c_void_p, i64, c_void_p, c_void_p, c_void_p]),
    "adaqp_ln_relu_bwd_f32": (C.c_int, [c_void_p, i64, c_void_p, i64, c_void_p, c_void_p, c_void_p, c_void_p, i64, i32, c_void_p, i64,
                                        c_void_p, i32, c_void_p]),
    "adaqp_gather_rows_f32": (C.c_int, [c_void_p, i64, c_void_p, i64, i32, c_void_p, i64,
                                        c_void_p]),
    "adaqp_lp_rate_clusters": (C.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, i64, c_void_p, c_void_p, i64,
                                         c_void_p, i64, c_void_p, i32, u64, u32, C.c_int, c_void_p, c_void_p,
                                         c_void_p, c_void_p]),
    "adaqp_lp_rate_blocks": (C.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, i64, c_void_p, c_void_p, i32, i64,
                                       u64, u32, C.c_int, C.c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "adaqp_lp_apply": (C.c_int, [c_void_p, i64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, i64, c_void_p,
                                 c_void_p]),
    "adaqp_lp_rebalance_select": (C.c_int, [c_void_p, i64, c_void_p, c_void_p, c_void_p, c_void_p, i64, c_void_p,
                                            c_void_p]),
    "adaqp_contract_edges": (C.c_int, [c_void_p, c_void_p, i64, c_void_p, c_void_p, c_void_p]),
    "adaqp_gat_scores_f32": (C.c_int, [c_void_p, i64, i64, i32, i32, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "adaqp_gat_fwd_f32": (C.c_int, [c_void_p, c_void_p, i64, c_void_p, i64, c_void_p, i64, c_void_p, c_void_p, c_void_p,
                                    i32, i32, i64, i64, c_void_p, i64, c_void_p, c_void_p]),
    "adaqp_gat_bwd_f32": (C.c_int, [c_void_p, c_void_p, i64, c_void_p, i64, c_void_p, i64, c_void_p, i64, c_void_p, i64,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, i32, i32, i64, i64,
                                    c_void_p, i64, c_void_p, c_void_p, c_void_p]),
    "adaqp_gatv2_fwd_f32": (C.c_int, [c_void_p, c_void_p, i64, c_void_p, i64, c_void_p, i64, c_void_p, i64, c_void_p,
                                      i32, i32, i64, i64, c_void_p, i64, c_void_p, c_void_p]),
    "adaqp_gatv2_bwd_inner_f32": (C.c_int, [c_void_p, c_void_p, i64, c_void_p, i64, c_void_p, i64, c_void_p, i64,
                                            c_void_p, i64, c_void_p, c_void_p, c_void_p, c_void_p, i64, c_void_p,
                                            c_void_p, i32, i32, i64, i64, c_void_p, i64, c_void_p, i64, c_void_p, i64,
                                            c_void_p]),
    "adaqp_gatv2_bwd_halo_f32": (C.c_int, [c_void_p, c_void_p, c_void_p, i64, c_void_p, i64, c_void_p, i64, c_void_p,
                                           c_void_p, c_void_p, i32, i32, i64, i64, c_void_p, i64, c_void_p]),
    "adaqp_sage_pool_fwd_f32": (C.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, i64, c_void_p, i64, c_void_p, i64,
                                          i32, i64, i64, C.c_int, c_void_p, i64, c_void_p, i64, c_void_p]),
    "adaqp_sage_pool_bwd_f32": (C.c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, i64, c_void_p, i64,
                                          c_void_p, i64, c_void_p, i64, c_void_p, i64, i32, i64, i64, C.c_int,
                                          c_void_p, i64, c_void_p]),
}

_lib = None


class AdaqpLibraryError(RuntimeError):
    pass


def load():
    """Load the shared library and bind every declared symbol (raises if any is missing)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise AdaqpLibraryError(
            f"{LIB_PATH} not found: the CUDA library is the product path and there is no "
            f"fallback. Build it with `python -m adaqp_b200.build`.")
    L = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        try:
            fn = getattr(L, name)
        except AttributeError as e:
            raise AdaqpLibraryError(f"{LIB_PATH} does not export {name}") from e
        fn.restype = res
        fn.argtypes = args
    v = L.adaqp_abi_version()
    if v != ADAQP_ABI_VERSION:
        raise AdaqpLibraryError(f"ABI version mismatch: library {v}, binding {ADAQP_ABI_VERSION}")
    _lib = L
    _apply_env_options(L)
    return L


# environment variable -> library option (read ONCE, here; the library itself never reads the environment)
ENV_OPTIONS = {"ADAQP_SPMM": "spmm_impl", "ADAQP_SPMM_GRAB": "spmm_rows_per_grab", "ADAQP_SPMM_CTAS": "spmm_ctas_per_sm",
               "ADAQP_SPMM_HINTS": "spmm_hints", "ADAQP_EXCH_SEND_CTAS": "exch_send_ctas",
               "ADAQP_EXCH_RECV_CTAS": "exch_recv_ctas", "ADAQP_GEMM_BLOCK_K": "gemm_block_k",
               "ADAQP_SPMM_SLICE_COLS": "spmm_slice_cols"}


def _apply_env_options(L):
    for env, name in ENV_OPTIONS.items():
        v = os.environ.get(env)
        if v is not None and v != "":
            set_option(name, int(v), L)


def set_option(name: str, value: int, L=None):
    L = L or load()
    rc = L.adaqp_set_option(name.encode(), int(value))
    if rc != 0:
        raise ValueError(L.adaqp_last_error().decode("utf-8", "replace"))


def get_option(name: str) -> int:
    L = load()
    out = i64(0)
    rc = L.adaqp_get_option(name.encode(), C.byref(out))
    if rc != 0:
        raise ValueError(L.adaqp_last_error().decode("utf-8", "replace"))
    return int(out.value)


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().adaqp_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"libadaqp_b200 {what} failed (rc={rc}): {msg}")


def stream_ptr(stream=None) -> int:
    """cudaStream_t of a torch stream (current stream when None)."""
    import torch
    if stream is None:
        stream = torch.cuda.current_stream()
    return stream.cuda_stream

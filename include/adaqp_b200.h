/*
 * adaqp_b200.h -- C ABI of libadaqp_b200.so (sm_90a).
 *
 * Drop-in boundary for AdaQP's per-layer boundary-message exchange + local
 * aggregation path.  The reference has no C/FFI plugin interface: its native
 * boundary is the pybind11 torch extension `quant_cuda` plus Python methods on
 * Communicator / CommBuffer (SURVEY.md 8b).  Every entry point below names the
 * reference interface it replaces (paths relative to the reference tree) and
 * takes plain pointers, sizes and a cudaStream_t passed as void*; no torch
 * types.  The Python side (adaqp_b200/_lib.py, ctypes) is the binding a
 * maintainer would add -- see INTEGRATION.md.
 *
 * Conventions: all pointers are DEVICE pointers unless the name says host;
 * every function returns 0 on success, a positive cudaError_t on a CUDA
 * failure, or a negative ADAQP_E* code on bad arguments.  Launches are
 * asynchronous on `stream` (NULL = legacy default stream).
 * adaqp_last_error() returns a thread-local message for the last failure.
 */
#ifndef ADAQP_B200_H
#define ADAQP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ADAQP_ABI_VERSION 9

#define ADAQP_EINVAL (-1)   /* bad argument (bits not in {1,2,4,8}, negative size ...) */
#define ADAQP_EALIGN (-2)   /* pointer alignment requirement violated */
#define ADAQP_ELIMIT (-3)   /* size outside what the kernels support */

/* status words written by the exchange kernels into `status` (device uint32[4]):
 * status[0] != 0 -> a flag/ack wait timed out (value = ADAQP_ST_*), status[1] = slot */
#define ADAQP_ST_OK 0u
#define ADAQP_ST_FLAG_TIMEOUT 1u
#define ADAQP_ST_ACK_TIMEOUT 2u

/* ---------------------------------------------------------------- runtime */
int adaqp_abi_version(void);
const char *adaqp_last_error(void);
/* number of SMs of the current device (grid sizing); <0 on error */
int adaqp_sm_count(void);
/* Process-wide tunables (the library never reads the environment; adaqp_b200/_lib.py maps ADAQP_*
 * variables onto these once at load).  Names: "spmm_impl" (1 register gather [default], 2 cp.async
 * ring, 3 TMA tile::gather4 ring, 4 TMA bulk-per-row ring), "spmm_rows_per_grab" (0 = default),
 * "spmm_ctas_per_sm", "spmm_hints" (bit 0 streaming output stores, bit 1 streaming index loads),
 * "gemm_block_k" (32 or 16: K block / swizzle width of the dense GEMM),
 * "exch_send_ctas" / "exch_recv_ctas" (0 = one resident wave over all SMs, n = at most n CTAs, so
 * that the exchange kernels leave the remaining SMs to the overlapped aggregation,
 * SURVEY.md 7 step 7 -- the reference instead serialises them, ops.py:119-130). */
int adaqp_set_option(const char *name, int64_t value);
int adaqp_get_option(const char *name, int64_t *value);

/* ------------------------------------------------------------ single codec
 * Replaces quant_cuda.pack_single_precision / unpack_single_precision
 * (AdaQP/util/quantization/src/quantization.cc:23-45,
 *  quantization_cuda_kernel.cu:34-52,106-122), fp32 instantiation.
 *
 * pack: packed[k = no*F + d] |= q(n = no*wpt + ni, d) << (ni*bits),
 *   q = rn(max(fma(data[n,d] - min[n], scale[n], U) - 0.5, 0)),
 *   U = curand_uniform of Philox4_32_10(seed, subsequence = k, offset), draw ni.
 * Writes exactly adaqp_packed_nbytes(N,F,bits) bytes.  The reference returns a
 * tensor one byte longer (adaqp_qsize) whose last byte is never written; the
 * host mirror allocates that size.  (seed, offset) are the values ATen's
 * philox_engine_inputs(F*8/bits) would hand the reference kernel; advancing
 * the generator is the host mirror's job (adaqp_b200/quant.py).
 */
int64_t adaqp_packed_nbytes(int64_t N, int64_t F, int bits);
int64_t adaqp_qsize(int64_t N, int64_t F, int bits);
int adaqp_pack_f32(const float *data, const float *min, const float *scale,
                   int64_t N, int64_t F, int bits, uint64_t seed, uint64_t offset,
                   uint8_t *packed, void *stream);
/* out[n,d] = float((packed[no*F+d] >> ni*bits) & mask) / scale[n] + min[n] */
int adaqp_unpack_f32(const uint8_t *packed, const float *scale, const float *min,
                     int64_t N, int64_t F, int bits, float *out, void *stream);

/* fp16 instantiation (the reference dispatches AT_DISPATCH_FLOATING_TYPES_AND_HALF, quantization_cuda_kernel.cu:81,138,
 * and check.h:22-27 admits float16): same layout and generator protocol, c10::Half arithmetic -- every Half (op) Half is
 * evaluated in float and rounded back to half.  data / min / scale / out are IEEE half arrays.  Not used by the hot
 * path (boundary messages are fp32); provided for API parity. */
int adaqp_pack_f16(const void *data, const void *min, const void *scale, int64_t N, int64_t F, int bits,
                   uint64_t seed, uint64_t offset, uint8_t *packed, void *stream);
int adaqp_unpack_f16(const uint8_t *packed, const void *scale, const void *min, int64_t N, int64_t F, int bits,
                     void *out, void *stream);

/* Row min / max / scale = (2^bits-1)/(max-min) in one pass
 * (AdaQP/model/op_util.py:20-22,41).  Any of rmin/rmax/scale may be NULL. */
int adaqp_row_minmax_f32(const float *data, int64_t N, int64_t F, int bits,
                         float *rmin, float *rmax, float *scale, void *stream);

/* ------------------------------------------------------------- P2P slabs
 * Replace the pinned-host staging buffers + gloo isend/irecv of
 * AdaQP/communicator/buffer.py:154-248 and comm.py:166-222: each rank owns one
 * device slab holding its receive regions, flags and acks; peers map it with
 * CUDA IPC and write into it directly over NVLink.  Handles travel through the
 * (gloo) control plane as 64 opaque bytes.
 */
#define ADAQP_IPC_HANDLE_BYTES 64
int adaqp_slab_alloc(void **ptr, size_t bytes);           /* cudaMalloc + zero fill */
int adaqp_slab_free(void *ptr);
int adaqp_ipc_export(void *ptr, unsigned char handle[ADAQP_IPC_HANDLE_BYTES]);
int adaqp_ipc_open(const unsigned char handle[ADAQP_IPC_HANDLE_BYTES], void **ptr);
int adaqp_ipc_close(void *ptr);
/* 1 if the current device can map `peer_device` memory */
int adaqp_can_access_peer(int peer_device);
/* cudaDeviceEnablePeerAccess(peer_device) for the current device (idempotent): lets ONE process
 * that drives several GPUs address their slabs directly (tools/bench_exchange.py --devices, the
 * single-process harness ncu can profile; multi-process runs map slabs with the IPC calls above). */
int adaqp_enable_peer_access(int peer_device);

/* --------------------------------------------------------- fused exchange
 * One channel = (this rank, one peer) for one layer key.
 */
typedef struct adaqp_send_chan {
    uint8_t *qdata;        /* peer-mapped: region receiving this rank's packed bytes   */
    uint16_t *params;      /* peer-mapped: bf16 [2, S] (row 0 scale, row 1 min)        */
    float *fp_rows;        /* peer-mapped: fp32 rows (fp32 exchange), else NULL        */
    uint32_t *flag;        /* peer-mapped: written with `seq` when the data is visible */
    const uint32_t *ack;   /* local: peer writes seq here after consuming              */
    int64_t S;             /* rows on this channel (params row stride)                 */
} adaqp_send_chan;

typedef struct adaqp_recv_chan {
    const uint8_t *qdata;  /* local region the peer writes                              */
    const uint16_t *params;
    const uint32_t *flag;  /* local flag the peer sets                                  */
    uint32_t *ack;         /* peer-mapped ack word                                      */
    int64_t S;
} adaqp_recv_chan;

/* One work item = one byte-row of a segment: 8/bits consecutive rows of one
 * (peer, bit-width) segment that share packed bytes. 64 bytes. */
typedef struct adaqp_send_item {
    int32_t src_row[4];    /* rows of the local message matrix (-1 = past the end)      */
    int32_t send_pos[4];   /* position in send_messages (total_send_idx order), tracing */
    int64_t dst_off;       /* byte offset of the item's F bytes inside chan.qdata       */
    int32_t param_pos;     /* column of the item's first row in chan.params             */
    int32_t group;         /* byte-row index inside its segment (Philox subsequence/F)  */
    uint32_t rel_offset;   /* Philox offset of the segment's pack call minus the base   */
    int16_t chan;          /* index into the channel table                              */
    int8_t bits;           /* 2, 4 or 8 (BITS_SET, buffer.py:20)                        */
    int8_t nrows;          /* valid rows (1..8/bits)                                    */
    int32_t _pad;
} adaqp_send_item;

typedef struct adaqp_recv_item {
    int32_t dst_row[4];    /* rows of the halo matrix to write (-1 = none)              */
    int64_t src_off;       /* byte offset of the item's F bytes inside chan.qdata       */
    int32_t param_pos;
    int16_t chan;
    int8_t bits;
    int8_t nrows;
} adaqp_recv_item;

/* fp32 exchange: one item per row sent. 16 bytes. */
typedef struct adaqp_fp_item {
    int32_t src_row;       /* row of the local message matrix                           */
    int32_t chan;
    int64_t dst_row;       /* row inside chan.fp_rows                                   */
} adaqp_fp_item;

/* Fused gather -> row min/max -> stochastic quantize -> bit-pack -> store into the
 * peers' slabs (+ bf16 params) -> publish flag.  Replaces, per layer key,
 * local_messages[total_send_idx] (ops.py:134,164), mixed_msg_quantization
 * (op_util.py:189-209), the D2H staging + isend half of qt_msg_exchange
 * (comm.py:193-222) and the tracing reductions of trace_input (op_util.py:91-99).
 * Byte-for-byte the reference wire format (SURVEY.md 3.6).
 *   x[n_rows, F] fp32 row-major (ld = row stride in floats);
 *   trace: optional [S_total] fp32 accumulator, trace[pos] += (F/6)(max-min)^2;
 *   (seed, base_offset): generator state the first pack call would have seen;
 *   seq: per-key exchange sequence number (>=1), written to every chan.flag;
 *   work: device uint32[2] scratch, zero on first use (kernel leaves it zero);
 *   status: device uint32[4], see ADAQP_ST_*; timeout_ns bounds every spin. */
int adaqp_send_quant(const float *x, int64_t ld, int32_t F,
                     const adaqp_send_item *items, int64_t n_items,
                     const adaqp_send_chan *chans, int32_t n_chans,
                     float *trace, uint64_t seed, uint64_t base_offset, uint32_t seq,
                     uint32_t *work, uint32_t *status, uint64_t timeout_ns, void *stream);

/* Wait flags -> unpack -> dequantize with the bf16 params -> scatter into the halo
 * matrix -> ack.  Replaces the irecv/H2D half of qt_msg_exchange and
 * mixed_msg_dequantization (op_util.py:211-236).  halo[n_remote, F], ld in floats. */
int adaqp_recv_quant(float *halo, int64_t ld, int32_t F,
                     const adaqp_recv_item *items, int64_t n_items,
                     const adaqp_recv_chan *chans, int32_t n_chans,
                     uint32_t seq, uint32_t *work, uint32_t *status,
                     uint64_t timeout_ns, void *stream);

/* fp32 exchange (Vanilla / AdaQP-p training and every eval forward): gather rows and
 * store them straight into the peers' halo rows, then publish flags.  Replaces
 * fp_msg_exchange (comm.py:166-191) + the scatter of fp_msg_transfer_process
 * (op_util.py:168-170): the sender already knows each row's halo position. */
int adaqp_send_fp32(const float *x, int64_t ld, int32_t F,
                    const adaqp_fp_item *items, int64_t n_items,
                    const adaqp_send_chan *chans, int32_t n_chans, int64_t dst_ld,
                    uint32_t seq, uint32_t *work, uint32_t *status,
                    uint64_t timeout_ns, void *stream);

/* Spin until every flags[i] >= seq (i < n).  Receiver half of the fp32 exchange. */
int adaqp_wait_flags(const uint32_t *const *flags, int32_t n, uint32_t seq,
                     uint32_t *status, uint64_t timeout_ns, void *stream);
/* Store seq into every acks[i]; launched after the consumer of a halo buffer. */
int adaqp_post_acks(uint32_t *const *acks, int32_t n, uint32_t seq, void *stream);

/* ------------------------------------------------------------ aggregation
 * Normalised CSR SpMM replacing DGL update_all(copy_src, sum|mean) plus the two
 * elementwise norm multiplies and the torch.cat of local and halo rows
 * (AdaQP/model/ops.py:17-67,137-147,169-185):
 *   out[v - row_begin] = post[v] * ( sum_{j in [indptr[v], indptr[v+1])} pre[u_j] x[u_j]
 *                                    (+ pre[v] x[v] if add_self) )      v in [row_begin,row_end)
 *   x[u] = u < n_split ? x0[u*ld0 ..] : x1[(u-n_split)*ld1 ..]   (local rows | halo rows)
 *   mean != 0: divide the sum by (indptr[v+1]-indptr[v]) (0-degree rows give 0).
 * pre (per source id, may be NULL) and post (per destination id, may be NULL) are fp32.
 * indices are int32 source ids; indptr is int64.  F <= 1024 (as the reference's codec). */
int adaqp_spmm_csr_f32(const int64_t *indptr, const int32_t *indices,
                       const float *x0, int64_t ld0, int64_t n_split,
                       const float *x1, int64_t ld1,
                       const float *pre, const float *post, int mean, int add_self,
                       int64_t row_begin, int64_t row_end, int32_t F,
                       float *out, int64_t ldo, void *stream);

/* Same aggregation over a per-row neighbour SEGMENT [seg_start[v], seg_end[v]) of the CSR row
 * (NULL = the row's own bounds), optionally accumulating into `out` (out += ...).  With the
 * columns of a row sorted, [indptr[v], split[v]) are the local sources and [split[v],
 * indptr[v+1]) the halo sources: the local part of the marginal rows can then run while the
 * exchange is still in flight and only the halo part waits for it (a finer overlap than the
 * reference's central / marginal split, ops.py:156-193).  `mean` still divides by the full
 * in-degree indptr[v+1] - indptr[v]; add_self belongs to exactly one of the two calls.
 * `live` (NULL = every source row is read): uint8 per local source row, 0 where the row of x0 is all
 * zeros (adaqp_row_live_f32).  The gather then skips the neighbours u < n_split with live[u] == 0 and a
 * finite pre[u]; they add exactly zero, so the result is the same (DESIGN §3).  Halo sources are always
 * read.  The opt-in spmm_impl variants 2-4 ignore `live`.
 * `rows` (NULL = every row of [row_begin, row_end)): a device list of n_list int32 destination row ids,
 * absolute CSR ids inside [row_begin, row_end), ascending and unique.  Only those rows are computed, each
 * exactly as without the list, into out + (row - row_begin) * ldo; the other output rows are neither read
 * nor written.  0 <= n_list <= row_end - row_begin (ADAQP_EINVAL otherwise); n_list == 0 launches nothing.
 * The ids themselves are the caller's to check (they live on the device).  `rows` and `live` cannot be
 * combined, and a list always takes the default kernels (spmm_impl 2-4 are not used with it). */
int adaqp_spmm_csr_seg_f32(const int64_t *indptr, const int64_t *seg_start, const int64_t *seg_end,
                           const int32_t *indices, const float *x0, int64_t ld0, int64_t n_split,
                           const float *x1, int64_t ld1, const float *pre, const float *post,
                           int mean, int add_self, int accumulate, int64_t row_begin,
                           int64_t row_end, int32_t F, float *out, int64_t ldo, const uint8_t *live,
                           const int32_t *rows, int64_t n_list, void *stream);

/* live[r] = 1 if some x[r, c] != 0 (a NaN counts as nonzero), else 0, for r < rows; x is [rows, F] fp32 with
 * pitch ld.  One coalesced read of x on `stream`. */
int adaqp_row_live_f32(const float *x, int64_t ld, int64_t rows, int32_t F, uint8_t *live, void *stream);

/* One APPNP personalized-PageRank step (DESIGN §13; host mirror adaqp_b200/appnp.py), with the same sources
 * (x0 | x1 split at n_split), per-row segments and accumulate mode as adaqp_spmm_csr_seg_f32:
 *   r[v] = (scale * post[v]) * sum_{u in seg(v)} pre[u] x[u]                v in [row_begin, row_end) <= n_split
 * forward (tele != NULL):  out[v] = r[v] + alpha * tele[v]            (scale = 1 - alpha, tele = z)
 * backward (acc_mode != 0, bit 0 set):  a[v] = alpha * x0[v] (+ acc[v] when bit 1 is set);
 *   without bit 2: out[v] = r[v], acc[v] = a[v];  with bit 2 (fold): out[v] = r[v] + a[v], acc is only read.
 * tele and acc_mode are exclusive; with neither, out[v] = r[v].  The once-per-row terms (tele, acc) belong
 * to the call with accumulate == 0: a call with accumulate != 0 (the halo segment of a split row) does
 * out[v] += r[v] only.  tele / acc / out rows are indexed v - row_begin (pitch ldt / lda / ldo).  fp32, the
 * __fmaf_rn chain of adaqp_spmm_csr_seg_f32 in CSR order, no float atomics: equal inputs give bitwise equal
 * outputs.  0 < F <= 1024; rows need only 4-byte alignment (odd F).  16-byte rows are aggregated in column slices
 * by the rule of adaqp_spmm_csr_seg_f32 (128 columns when F is a multiple of 128 above 128; option spmm_slice_cols
 * forces a width, a multiple of 4 up to 128, >= F = unsliced), with bitwise the same result (DESIGN §14). */
int adaqp_appnp_prop_f32(const int64_t *indptr, const int64_t *seg_start, const int64_t *seg_end,
                         const int32_t *indices, const float *x0, int64_t ld0, int64_t n_split, const float *x1,
                         int64_t ld1, const float *pre, const float *post, float scale, float alpha,
                         const float *tele, int64_t ldt, float *acc, int64_t lda, int32_t acc_mode, int accumulate,
                         int64_t row_begin, int64_t row_end, int32_t F, float *out, int64_t ldo, void *stream);

/* --------------------------------------------------------------- Correct & Smooth (DESIGN §16; host mirror
 * adaqp_b200/cs.py).  y is int32 per row: the row's label where it is fixed (a train row), else -1.  Bad arguments
 * (C outside [1, 1024], a bad row range or shape, null pointers, lo > hi, a bad scale) return ADAQP_EINVAL before any
 * CUDA call.
 *
 * One propagation step over whole CSR rows [row_begin, row_end) <= n_split, the sources of adaqp_appnp_prop_f32:
 *   r[v] = (scale * post[v]) * sum_{u in N(v)} pre[u] x[u]  (+ alpha * tele[v] in clamp mode, tele != NULL)
 *   post_mode 0 (clamp): out[v] = min(max(r[v], lo), hi)
 *   post_mode 1 (fix)  : out[v] = fix[v] where y[v] >= 0 (no gather for that row), else r[v]; tele is not read
 * tele / y / fix / out rows are indexed v - row_begin.  The sum and the epilogue's rounding are appnp_prop's: with
 * lo = -inf and hi = +inf the clamp step is bitwise adaqp_appnp_prop_f32's teleport step.  No segments: a clamp or a
 * fixed row cannot be applied to two partial sums. */
int adaqp_cs_prop_f32(const int64_t *indptr, const int32_t *indices, const float *x0, int64_t ld0, int64_t n_split,
                      const float *x1, int64_t ld1, const float *pre, const float *post, float scale, float alpha,
                      const float *tele, int64_t ldt, const int32_t *y, const float *fix, int64_t ldf,
                      int32_t post_mode, float lo, float hi, int64_t row_begin, int64_t row_end, int32_t F,
                      float *out, int64_t ldo, void *stream);

/* Set-up of rows [0, rows): yhat = softmax(z) (row maximum subtracted), e0 = onehot(y) - yhat where y >= 0 and 0
 * elsewhere, and partials[b] = the float64 sum of |e0| over the rows CTA b handles (the grid is n_partials CTAs; the
 * partials depend only on the input and n_partials). */
int adaqp_cs_init_f32(const float *z, int64_t ldz, const int32_t *y, int64_t rows, int32_t C, float *yhat,
                      int64_t ldy, float *e0, int64_t lde, double *partials, int32_t n_partials, void *stream);

/* Combine of rows [0, rows): g0[v] = onehot(y[v]) where y >= 0, else yhat[v] + s[v] e[v] with, for autoscale != 0,
 * s[v] = value / |e[v]|_1 (value = sigma >= 0; s[v] = 1 where |e[v]|_1 = 0 or s[v] > 1000, decided in float64), and
 * for autoscale == 0 s[v] = value (a finite scale > 0). */
int adaqp_cs_combine_f32(const float *yhat, int64_t ldy, const float *e, int64_t lde, const int32_t *y, int64_t rows,
                         int32_t C, int32_t autoscale, double value, float *g0, int64_t ldg, void *stream);

/* --------------------------------------------------------------- dense GEMM
 * C[M, N] = A[M, K] . Bt[N, K]^T (+ bias[N]) in fp32 on the Hopper tensor cores (wgmma) by 3xTF32 error-compensated
 * splitting (csrc/gemm.cu): replaces torch.matmul(rst, self.weight) (AdaQP/model/distGCN.py:45) and the Linear
 * layers of distSAGE.py:51-53 for tall-skinny shapes (M = inner nodes, N <= 256).  Bt_hi / Bt_lo are the
 * transposed weight split as b_hi = b & 0xFFFFE000, b_lo = b - b_hi (host mirror: adaqp_b200/dense.py).
 * lda / ldb multiples of 4 floats, 16-byte aligned bases; adaqp_gemm_tf32x3_supported tells whether a shape
 * qualifies (otherwise the caller keeps torch.matmul). */
int adaqp_gemm_tf32x3_supported(int64_t M, int32_t N, int32_t K, int64_t lda, int64_t ldb, int64_t ldc);
int adaqp_gemm_tf32x3_f32(const float *A, int64_t lda, const float *Bt_hi, const float *Bt_lo, int64_t ldb,
                          const float *bias, int64_t M, int32_t N, int32_t K, float *C, int64_t ldc, void *stream);

/* Weight gradient dW[N, K] = dY[M, N]^T . X[M, K] (the `X^T . dY` of the layers' backward), split over the M node rows:
 * CTA c writes its partial sum to partials[c] ([grid, N, K] fp32, grid = adaqp_wgrad_tf32x3_grid(M)); the caller adds the
 * slices.  Same 3xTF32 arithmetic; both operands are read straight from their row-major storage. */
int adaqp_wgrad_tf32x3_supported(int64_t M, int32_t N, int32_t K, int64_t ldy, int64_t ldx);
int adaqp_wgrad_tf32x3_grid(int64_t M);
int adaqp_wgrad_tf32x3_f32(const float *dY, int64_t ldy, const float *X, int64_t ldx, int64_t M, int32_t N, int32_t K,
                           float *partials, int32_t grid, void *stream);

/* ------------------------------------------------------ LayerNorm + ReLU
 * y = relu(LayerNorm(x) * gamma + beta) over the last dimension (biased variance, eps as nn.LayerNorm), forward and
 * backward in one pass each: the `self.norms[i](feats)` + `F.relu` between aggregations (AdaQP/model/distGCN.py:81-84,
 * distSAGE.py:93-96).  F % 4 == 0, F <= 1024, 16-byte aligned rows.  The backward writes per-CTA partial column sums
 * partials[grid][2][F] (dgamma, dbeta; grid = adaqp_ln_relu_grid(M)) that the caller adds.  Dropout stays torch's. */
int adaqp_ln_relu_grid(int64_t M);
int adaqp_ln_relu_fwd_f32(const float *x, int64_t ldx, const float *gamma, const float *beta, float eps, int64_t M,
                          int32_t F, float *y, int64_t ldy, float *mean, float *rstd, void *stream);
int adaqp_ln_relu_bwd_f32(const float *dy, int64_t lddy, const float *x, int64_t ldx, const float *mean,
                          const float *rstd, const float *gamma, const float *beta, int64_t M, int32_t F, float *dx,
                          int64_t lddx, float *partials, int32_t grid, void *stream);

/* Row gather out[i] = x[idx[i]] (copy-buffer fills of ops.py:159-164; API parity only). */
int adaqp_gather_rows_f32(const float *x, int64_t ld, const int64_t *idx, int64_t n,
                          int32_t F, float *out, int64_t ldo, void *stream);

/* ------------------------------------------------------------ graph attention (GAT)
 * DGL's GATConv aggregation (shared projection, negative slope 0.2, no attention dropout) over the halo exchange
 * (csrc/gat.cu, host mirror adaqp_b200/gat.py); an extension beyond the reference, whose models are GCN and SAGE.
 * Rows are F = H * D floats (H heads of width D); F <= 256, and when H > 1, D must be a multiple or a divisor of
 * 32.  Per-head scalars are [rows, H] row-major.  As in adaqp_spmm_csr_seg_f32, source ids < n_split are local rows
 * (z0, el0, ...) and ids >= n_split halo rows (z1, el1, ...; may be NULL when no row of the range has a halo
 * neighbour); a launch covers destination rows [row_begin, row_end) and writes output row v at v - row_begin.
 * No float atomics: equal inputs give bitwise equal outputs.
 *
 * scores: el[i,h] = <z[i,h,:], a_l[h,:]>, er[i,h] = <z[i,h,:], a_r[h,:]> for i < n_rows; a_l, a_r are [H * D]. */
int adaqp_gat_scores_f32(const float *z, int64_t ldz, int64_t n_rows, int32_t H, int32_t F, const float *a_l,
                         const float *a_r, float *el, float *er, void *stream);
/* forward: e[v,u,h] = LeakyReLU(el[u,h] + er[v,h]) over the CSR row of v, lse[v,h] = logsumexp_u e[v,u,h],
 * out[v,h,:] = sum_u exp(e[v,u,h] - lse[v,h]) z[u,h,:].  er covers the local rows (indexed by v). */
int adaqp_gat_fwd_f32(const int64_t *indptr, const int32_t *indices, int64_t n_split, const float *z0, int64_t ldz0,
                      const float *z1, int64_t ldz1, const float *el0, const float *el1, const float *er, int32_t H,
                      int32_t F, int64_t row_begin, int64_t row_end, float *out, int64_t ldo, float *lse,
                      void *stream);
/* backward for local rows u (row_end <= n_split) of a symmetric graph, g = dL/dout, aux rows [er | lse | s] (3H
 * floats, s[v,h] = <g[v,h,:], out[v,h,:]>):
 *   t[v,u,h] = alpha[v,u,h] (<g[v,h,:], z[u,h,:]> - s[v,h]) (1 if el[u,h] + er[v,h] > 0 else 0.2)
 *   del[u,h] = sum_{v in row u} t[v,u,h],  der[u,h] = sum_{w in row u} t[u,w,h]
 *   dz[u] = sum_{v in row u} alpha[v,u] g[v] + del[u] a_l + der[u] a_r  (per head). */
int adaqp_gat_bwd_f32(const int64_t *indptr, const int32_t *indices, int64_t n_split, const float *g0, int64_t ldg0,
                      const float *g1, int64_t ldg1, const float *z0, int64_t ldz0, const float *z1, int64_t ldz1,
                      const float *el0, const float *el1, const float *aux0, const float *aux1, const float *a_l,
                      const float *a_r, int32_t H, int32_t F, int64_t row_begin, int64_t row_end, float *dz,
                      int64_t lddz, float *del, float *der, void *stream);

/* ------------------------------------------------------------ GATv2 attention
 * DGL's GATv2Conv aggregation (share_weights=False, negative slope 0.2, no attention dropout) over the halo exchange
 * (csrc/gatv2.cu, host mirror adaqp_b200/gatv2.py).  Rows, head layouts, per-head scalars and the local / halo
 * source split are those of the GAT entry points; attn is [H * D].  zd, g, lse and S cover the local rows only.
 * No float atomics: equal inputs give bitwise equal outputs.
 *
 * forward: e[v,u,h] = sum_{c in head h} attn[h,c] LeakyReLU(zs[u,h,c] + zd[v,h,c]) over the CSR row of v,
 * lse[v,h] = logsumexp_u e[v,u,h], out[v,h,:] = sum_u exp(e[v,u,h] - lse[v,h]) zs[u,h,:]; rows are local. */
int adaqp_gatv2_fwd_f32(const int64_t *indptr, const int32_t *indices, int64_t n_split, const float *zs0,
                        int64_t ldzs0, const float *zs1, int64_t ldzs1, const float *zd, int64_t ldzd,
                        const float *attn, int32_t H, int32_t F, int64_t row_begin, int64_t row_end, float *out,
                        int64_t ldo, float *lse, void *stream);
/* backward of the inner rows u (row_end <= n_split) of a symmetric graph, g = dL/dout, S[v,h] = <g[v,h,:],
 * out[v,h,:]>, t[v,u,h] = alpha[v,u,h] (<g[v,h,:], zs[u,h,:]> - S[v,h]), s = zs[u] + zd[v]:
 *   dzs[u] = sum_{local v in row u} alpha[v,u] g[v] + t[v,u] attn . LeakyReLU'(s) + pushed rows of u
 *   dzd[u] = sum_{w in row u} t[u,w] attn . LeakyReLU'(zs[w] + zd[u])
 *   da[u]  = sum_{w in row u} t[u,w] LeakyReLU(zs[w] + zd[u])       (per-row shares; da is their column sum)
 * The pushed rows of u are push[fold_pos[k]] for k in [fold_indptr[u], fold_indptr[u+1]), added in that order;
 * push, fold_indptr and fold_pos are all NULL (no fold) or all given. */
int adaqp_gatv2_bwd_inner_f32(const int64_t *indptr, const int32_t *indices, int64_t n_split, const float *zs0,
                              int64_t ldzs0, const float *zs1, int64_t ldzs1, const float *zd, int64_t ldzd,
                              const float *g, int64_t ldg, const float *lse, const float *S, const float *attn,
                              const float *push, int64_t ldp, const int64_t *fold_indptr, const int32_t *fold_pos,
                              int32_t H, int32_t F, int64_t row_begin, int64_t row_end, float *dzs, int64_t lddzs,
                              float *dzd, int64_t lddzd, float *da, int64_t ldda, void *stream);
/* backward of the halo rows h in [row_begin, row_end): out[h - row_begin] = sum over the inner destinations v in
 * halo_dst[halo_indptr[h] .. halo_indptr[h+1]) of alpha[v,h] g[v] + t[v,h] attn . LeakyReLU'(zs1[h] + zd[v]): the
 * gradient of the received row, which its holder pushes back to the row's owner. */
int adaqp_gatv2_bwd_halo_f32(const int64_t *halo_indptr, const int32_t *halo_dst, const float *zs1, int64_t ldzs1,
                             const float *zd, int64_t ldzd, const float *g, int64_t ldg, const float *lse,
                             const float *S, const float *attn, int32_t H, int32_t F, int64_t row_begin,
                             int64_t row_end, float *out, int64_t ldo, void *stream);

/* ------------------------------------------------------------ GraphSAGE max-pool aggregation
 * DGL's SAGEConv(aggregator_type='pool') neighbourhood max over the halo exchange (csrc/sage_pool.cu, host mirror
 * adaqp_b200/sage_pool.py); an extension beyond the reference, whose aggregators are mean and gcn.  Rows are
 * 0 < F <= 1024 floats.  As in adaqp_spmm_csr_seg_f32, source ids < n_split are local rows (x0, g0, a0) and ids
 * >= n_split halo rows (x1, g1, a1; may be NULL when no visited entry is a halo source); seg_start / seg_end (NULL =
 * the row bounds) restrict each row to [seg_start[v], seg_end[v]); a launch covers rows [row_begin, row_end) and
 * writes row v at v - row_begin; accumulate != 0 continues from what the output already holds.  arg entries are
 * (source id - n_split), INT32_MIN for a row without sources (whose m is 0).  No float atomics: equal inputs give
 * bitwise equal outputs, and a local-segment launch followed by an accumulating halo-segment launch equals one
 * launch over whole rows bit for bit.
 *
 * forward: m[v,c] = max_u x[u,c] over the row of v, arg[v,c] = the first u in CSR order attaining it. */
int adaqp_sage_pool_fwd_f32(const int64_t *indptr, const int64_t *seg_start, const int64_t *seg_end,
                            const int32_t *indices, int64_t n_split, const float *x0, int64_t ld0, const float *x1,
                            int64_t ld1, int32_t F, int64_t row_begin, int64_t row_end, int accumulate, float *out,
                            int64_t ldo, int32_t *arg, int64_t lda, void *stream);
/* backward for local rows u (row_end <= n_split) of a symmetric graph, g = dL/dm, a = arg rows in their owner's
 * encoding, want[e] (aligned with indices) = row u in the encoding of the owner of indices[e]:
 *   dp[u,c] = sum_{e in row u} g[x_e,c] [a[x_e,c] == want[e]]   (sum in CSR order) */
int adaqp_sage_pool_bwd_f32(const int64_t *indptr, const int64_t *seg_start, const int64_t *seg_end,
                            const int32_t *indices, const int32_t *want, int64_t n_split, const float *g0,
                            int64_t ldg0, const float *g1, int64_t ldg1, const int32_t *a0, int64_t lda0,
                            const int32_t *a1, int64_t lda1, int32_t F, int64_t row_begin, int64_t row_end,
                            int accumulate, float *dp, int64_t ldd, void *stream);

/* ------------------------------------------------------------ graph partitioning
 * Multilevel label-propagation k-way partitioning (csrc/partition.cu, level driver and host initial
 * partition in adaqp_b200/partition.py): replaces dgl.distributed.partition_graph(graph, ..., num_hops=1,
 * balance_edges=False), i.e. METIS, at AdaQP/helper/partition.py:71-72.  Graphs are symmetric CSR without
 * self-loops: int64 indptr[n+1], int32 indices, int32 edge weights ew and vertex weights vw.  Labels are int32;
 * label weights (lw / bw) are int64.  One sub-round (round, sub) moves only the vertices v with
 * h(seed, round, v) & 1 == sub, h = splitmix64 mix (DESIGN.md, "Graph partitioning").  Every rating kernel
 * writes, per vertex, tgt[v] (proposed label, -1 = none), gain[v] = rho(tgt) - rho(label[v]) and
 * hkey[v] = h(seed, round, v) >> 1, the order key of the apply step. */
#define ADAQP_MAX_PARTS 64          /* the exchange's channel limit */
#define ADAQP_LP_HUB_DEGREE 256     /* clustering: vertices of larger degree are rated by the hub path */

/* Clustering sub-round rating: candidate labels are the neighbours' labels c with lw[c] + vw[v] <= cap;
 * only positive gains are proposed.  Labels are < n.  Vertices of degree > ADAQP_LP_HUB_DEGREE must all be listed
 * in hubs[n_hubs]; they are rated by min(n_hubs, hub_ctas) CTAs, CTA b counting in the dense row
 * hub_scratch[b * n .. (b + 1) * n), which must be zero on entry and is left zero. */
int adaqp_lp_rate_clusters(const int64_t *indptr, const int32_t *indices, const int32_t *ew, const int32_t *vw,
                           int64_t n, const int32_t *label, const int64_t *lw, int64_t cap, const int32_t *hubs,
                           int64_t n_hubs, uint32_t *hub_scratch, int32_t hub_ctas, uint64_t seed, uint32_t round, int sub,
                           int32_t *tgt, int64_t *gain, int64_t *hkey, void *stream);
/* k-way rating, 1 <= k <= ADAQP_MAX_PARTS.  mode 0: refinement sub-round (positive gains only);
 * mode 1: rebalancing, every vertex of a block with bw > cap proposes its best block with room, any gain. */
int adaqp_lp_rate_blocks(const int64_t *indptr, const int32_t *indices, const int32_t *ew, const int32_t *vw, int64_t n,
                         const int32_t *part, const int64_t *bw, int32_t k, int64_t cap, uint64_t seed, uint32_t round,
                         int sub, int mode, int32_t *tgt, int64_t *gain, int64_t *hkey, void *stream);
/* Apply: order[n_prop] = proposing vertices sorted by (tgt asc, gain desc, hkey asc, v asc); csum = inclusive
 * prefix sum of vw[order].  Per target b the longest prefix with lw[b] + prefix weight <= cap is accepted:
 * label[v] = b and dlw[b] += vw[v], dlw[old label] -= vw[v] (the caller adds dlw to lw). */
int adaqp_lp_apply(const int32_t *order, int64_t n_prop, const int64_t *csum, const int32_t *tgt, const int32_t *vw,
                   int32_t *label, const int64_t *lw, int64_t cap, int64_t *dlw, void *stream);
/* Rebalancing, source side: order = proposals of mode 1 sorted by (part asc, gain desc, hkey asc, v asc), csum as
 * above.  Per over-full block keeps the shortest prefix whose weight covers bw - cap and sets tgt[v] = -1 for the
 * rest; the kept proposals then go through adaqp_lp_apply. */
int adaqp_lp_rebalance_select(const int32_t *order, int64_t n_prop, const int64_t *csum, const int32_t *part,
                              const int32_t *vw, const int64_t *bw, int64_t cap, int32_t *tgt, void *stream);
/* Contraction: key[e] = (int64)cid[v] << 32 | cid[indices[e]] for every edge e of row v, INT64_MAX when both
 * ends are in the same cluster (the caller sorts the keys and sums the weights of equal keys). */
int adaqp_contract_edges(const int64_t *indptr, const int32_t *indices, int64_t n, const int32_t *cid, int64_t *key,
                         void *stream);

#ifdef __cplusplus
}
#endif
#endif /* ADAQP_B200_H */

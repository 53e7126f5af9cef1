// Normalised CSR SpMM for full-graph GNN aggregation (sm_90a).
//
// Replaces DGL update_all(copy_src, sum|mean) and the surrounding elementwise norm
// kernels / torch.cat copies of AdaQP/model/ops.py:17-67,137-147,169-185:
//   out[v] = post[v] * ( sum_{u in N_in(v)} pre[u] * x[u]  (+ pre[v] x[v]) )  [/ deg(v)]
// Source rows come from two matrices without concatenation: ids < n_split are local
// (inner) rows, ids >= n_split are halo rows written by the exchange kernels.  The
// central / marginal decomposition of the reference (conversion.py:114-172) is a row
// range [row_begin, row_end) of the same CSR: central rows have no halo in-neighbours
// by construction, so no copy buffers are needed.
//
// HBM/L2-bound gather: one warp per destination row, the row's F floats spread across
// lanes as VEC-wide vectors (CHUNKS per lane), neighbour ids fetched 32 at a time and
// broadcast by shuffle, 4 neighbour rows (4*CHUNKS vector loads per lane) in flight.
// fp32 accumulation in CSR order (DGL's order is unspecified: parity is to a stated
// tolerance against a float64 oracle, DESIGN.md).
#include <cuda.h>      // CUtensorMap (type only: the encoder is fetched with cudaGetDriverEntryPoint)

#include <mutex>
#include <unordered_map>

#include "common.cuh"

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kUnroll = 4;

// hint bits (option "spmm_hints"): the output rows and the index stream are touched once per launch,
// the gathered source rows are what should stay in L2
constexpr int kHintStoreStreaming = 1;   // st.global.cs for the output rows (evict-first)
constexpr int kHintIndexStreaming = 2;   // ld.global.cs for `indices`

template <int VEC> struct Vec;
template <> struct Vec<4> {
    static __device__ __forceinline__ void load(const float *p, float (&v)[4]) {
        const float4 t = __ldg(reinterpret_cast<const float4 *>(p)); v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    }
    static __device__ __forceinline__ void store(float *p, const float (&v)[4]) {
        *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]);
    }
    static __device__ __forceinline__ void store_cs(float *p, const float (&v)[4]) {
        __stcs(reinterpret_cast<float4 *>(p), make_float4(v[0], v[1], v[2], v[3]));
    }
};
template <> struct Vec<2> {
    static __device__ __forceinline__ void load(const float *p, float (&v)[2]) {
        const float2 t = __ldg(reinterpret_cast<const float2 *>(p)); v[0] = t.x; v[1] = t.y;
    }
    static __device__ __forceinline__ void store(float *p, const float (&v)[2]) {
        *reinterpret_cast<float2 *>(p) = make_float2(v[0], v[1]);
    }
    static __device__ __forceinline__ void store_cs(float *p, const float (&v)[2]) {
        __stcs(reinterpret_cast<float2 *>(p), make_float2(v[0], v[1]));
    }
};
template <> struct Vec<1> {
    static __device__ __forceinline__ void load(const float *p, float (&v)[1]) { v[0] = __ldg(p); }
    static __device__ __forceinline__ void store(float *p, const float (&v)[1]) { *p = v[0]; }
    static __device__ __forceinline__ void store_cs(float *p, const float (&v)[1]) { __stcs(p, v[0]); }
};

// Row liveness (DESIGN §3, "skipping all-zero source rows"): live[r] = 1 when row r of the local source matrix
// has an element that compares unequal to 0 (a NaN does), 0 when every element is +0 or -0.  A neighbour u whose
// row is dead adds __fmaf_rn(w, ±0, acc) == acc to every accumulator as long as w is finite: acc starts at +0 and
// the chain only produces -0 from a product that underflows to -0, so dropping the term leaves every output
// element unchanged (at most the sign of a zero result can differ, after such an underflow).
//
// compact_live_window: the warp's window of n (<= 32) neighbour ids u and weights w, one per lane, is compacted
// in place to the neighbours that are kept -- halo sources (u >= n_split, always kept), live local rows, and any
// neighbour whose weight is not finite (inf * 0 is NaN) -- keeping their CSR order.  Lane i takes the i-th kept
// neighbour; returns how many were kept.
__device__ __forceinline__ int compact_live_window(int lane, int n, int64_t n_split, const uint8_t *__restrict__ live,
                                                   int &u, float &w) {
    const bool keep = lane < n && ((int64_t)u >= n_split || __ldg(live + u) != 0 || !isfinite(w));
    const unsigned m = __ballot_sync(ADAQP_FULL_MASK, keep);
    const int kept = __popc(m);
    const int src = lane < kept ? (int)__fns(m, 0, lane + 1) : lane;
    u = __shfl_sync(ADAQP_FULL_MASK, u, src);
    w = __shfl_sync(ADAQP_FULL_MASK, w, src);
    return kept;
}

// One warp's weighted gather over the neighbour segment [b, e_) of a destination row:
// acc += pre[u] * x[u] in CSR order, one __fmaf_rn per element and neighbour, the row's F floats spread
// across lanes as VEC-wide vectors (CHUNKS per lane), neighbour ids fetched 32 at a time and broadcast by
// shuffle, UNROLL_ neighbour rows (UNROLL_ * CHUNKS vector loads per lane) in flight.  Expanded in
// spmm_csr_kernel and appnp_prop_kernel, so both sum in the same order.  A macro rather than an inlined
// function: expanded in place, spmm_csr_kernel compiles to the same SASS as before appnp_prop_kernel
// shared it (an inlined function changed its register allocation).  Reads acc, colok, lane, indices,
// b, e_, x0, ld0, n_split, x1, ld1, pre and hints from the enclosing scope.
// With SKIP_ (a constant) the 32-id window is first compacted to the neighbours compact_live_window keeps, in CSR
// order, reading the row-liveness array LIVE_; with SKIP_ false the expansion is the gather without liveness.
#define ADAQP_GATHER_SEGMENT(UNROLL_, SKIP_, LIVE_) \
        for (int64_t j0 = b; j0 < e_; j0 += 32) {                                                                       \
            int n = (e_ - j0) < 32 ? (int)(e_ - j0) : 32;                                                               \
            int u = 0;                                                                                                  \
            float w = 0.f;                                                                                              \
            if (lane < n) {                                                                                             \
                u = (hints & kHintIndexStreaming) ? __ldcs(indices + j0 + lane) : __ldg(indices + j0 + lane);           \
                w = pre ? __ldg(pre + u) : 1.f;                                                                         \
            }                                                                                                           \
            if constexpr (SKIP_) n = compact_live_window(lane, n, n_split, LIVE_, u, w);                                \
            for (int k = 0; k < n; k += UNROLL_) {                                                                      \
                float v[UNROLL_][CHUNKS][VEC];                                                                          \
                float ww[UNROLL_];                                                                                      \
_Pragma("unroll")                                                                                                       \
                for (int t = 0; t < UNROLL_; ++t) {                                                                     \
                    const int src = (k + t) & 31;                                                                       \
                    const int uu = __shfl_sync(ADAQP_FULL_MASK, u, src);                                                \
                    ww[t] = __shfl_sync(ADAQP_FULL_MASK, w, src);                                                       \
                    const bool live = (k + t) < n;                                                                      \
                    if (!live) ww[t] = 0.f;                                                                             \
                    const float *rp = (uu < n_split) ? (x0 + (int64_t)uu * ld0) : (x1 + ((int64_t)uu - n_split) * ld1); \
_Pragma("unroll")                                                                                                       \
                    for (int c = 0; c < CHUNKS; ++c) {                                                                  \
                        if (live && colok[c]) {                                                                         \
                            Vec<VEC>::load(rp + (c * 32 + lane) * VEC, v[t][c]);                                        \
                        } else {                                                                                        \
_Pragma("unroll")                                                                                                       \
                            for (int e = 0; e < VEC; ++e) v[t][c][e] = 0.f;                                             \
                        }                                                                                               \
                    }                                                                                                   \
                }                                                                                                       \
_Pragma("unroll")                                                                                                       \
                for (int t = 0; t < UNROLL_; ++t)                                                                       \
_Pragma("unroll")                                                                                                       \
                    for (int c = 0; c < CHUNKS; ++c)                                                                    \
_Pragma("unroll")                                                                                                       \
                        for (int e = 0; e < VEC; ++e) acc[c][e] = __fmaf_rn(ww[t], v[t][c][e], acc[c][e]);              \
            }                                                                                                           \
        }

// SKIP: the gather leaves out the local source rows that `live` marks all-zero (compact_live_window); the
// result is the same.  SKIP = false is the kernel without liveness (`live` unused).
// LIST: only the destination rows rows[0 .. n_list) are computed (absolute CSR row ids in [row_begin, row_end),
// ascending): the frontier numbers positions in the list instead of rows, and each listed row is computed and
// stored exactly as without the list; the other output rows are not touched.  LIST = false: `rows` unused.
template <int VEC, int CHUNKS, bool SKIP, bool LIST>
__global__ void __launch_bounds__(kThreads)
spmm_csr_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                const float *__restrict__ x0, int64_t ld0, int64_t n_split,
                const float *__restrict__ x1, int64_t ld1,
                const float *__restrict__ pre, const float *__restrict__ post,
                int mean, int add_self, int64_t row_begin, int64_t row_end, int F,
                float *__restrict__ out, int64_t ldo, unsigned long long *__restrict__ next_row, int rows_per_grab,
                const int64_t *__restrict__ seg_start, const int64_t *__restrict__ seg_end, int accumulate, int hints,
                const uint8_t *__restrict__ live, const int32_t *__restrict__ rows, int64_t n_list) {
    const int lane = threadIdx.x & 31;
    bool colok[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) colok[c] = ((c * 32 + lane) * VEC) < F;

    // Frontier scheduling: warps take the next `rows_per_grab` destination rows from a global
    // counter, so the rows in flight are always one contiguous window (~ #warps * rows_per_grab
    // rows) however uneven the degrees are.  With a static row -> warp map the warps drift
    // apart (power-law degrees) and the set of source rows being reused grows far beyond
    // L2, even on graphs where most edges stay inside small communities.
    // With LIST the counter walks list positions: position i is row rows[i].
    const int64_t n_rows = LIST ? n_list : row_end - row_begin;
    const int64_t pos_base = LIST ? 0 : row_begin;
    while (true) {
        unsigned long long grab = 0;
        if (lane == 0) grab = atomicAdd(next_row, (unsigned long long)rows_per_grab);
        grab = __shfl_sync(ADAQP_FULL_MASK, grab, 0);
        if ((int64_t)grab >= n_rows) break;
        const int64_t r_hi = ((int64_t)grab + rows_per_grab < n_rows) ? (int64_t)grab + rows_per_grab : n_rows;
    for (int64_t pos = pos_base + (int64_t)grab; pos < pos_base + r_hi; ++pos) {
        const int64_t row = LIST ? (int64_t)__ldg(rows + pos) : pos;
        float acc[CHUNKS][VEC];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c)
#pragma unroll
            for (int e = 0; e < VEC; ++e) acc[c][e] = 0.f;
        // neighbour segment of this launch: the whole row, or [seg_start[row], seg_end[row]) when the
        // caller splits a row into its local-source and halo-source parts (ops.py overlap)
        const int64_t row_b = __ldg(indptr + row), row_e = __ldg(indptr + row + 1);
        const int64_t b = seg_start ? __ldg(seg_start + row) : row_b;
        const int64_t e_ = seg_end ? __ldg(seg_end + row) : row_e;
        ADAQP_GATHER_SEGMENT(kUnroll, SKIP, live)
        if (add_self) {
            const float ws = pre ? __ldg(pre + row) : 1.f;
            const float *rp = (row < n_split) ? (x0 + row * ld0) : (x1 + (row - n_split) * ld1);
#pragma unroll
            for (int c = 0; c < CHUNKS; ++c) {
                if (colok[c]) {
                    float v[VEC];
                    Vec<VEC>::load(rp + (c * 32 + lane) * VEC, v);
#pragma unroll
                    for (int e = 0; e < VEC; ++e) acc[c][e] = __fmaf_rn(ws, v[e], acc[c][e]);
                }
            }
        }
        const float deg = (float)(row_e - row_b);       // mean divides by the full in-degree
        const float ps = post ? __ldg(post + row) : 1.f;
        float *orow = out + (row - row_begin) * ldo;
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            if (colok[c]) {
                float prev[VEC];
                if (accumulate) Vec<VEC>::load(orow + (c * 32 + lane) * VEC, prev);
#pragma unroll
                for (int e = 0; e < VEC; ++e) {
                    float r = acc[c][e];
                    if (mean && deg > 0.f) r = __fdiv_rn(r, deg);
                    if (post) r = __fmul_rn(r, ps);
                    if (accumulate) r = __fadd_rn(prev[e], r);
                    acc[c][e] = r;
                }
                if (hints & kHintStoreStreaming) Vec<VEC>::store_cs(orow + (c * 32 + lane) * VEC, acc[c]);
                else Vec<VEC>::store(orow + (c * 32 + lane) * VEC, acc[c]);
            }
        }
    }
    }
    frontier_release(next_row);
}

// ---------------------------------------------------------------------------------------
// APPNP teleport propagation (DESIGN §13): spmm_csr_kernel's gather with the step's teleport term in the
// epilogue, so a propagation step is one pass over [n, C] instead of an SpMM plus elementwise passes.
//   r[v] = (scale * post[v]) * sum_{u in seg(v)} pre[u] x[u]
//   EPI = kEpiTeleport: out[v] = r[v] + alpha * tele[v]                      (forward: tele = z)
//   EPI = kEpiAccum   : out[v] = r[v];  a = alpha * x[v] (+ acc[v] with kAccRead)  (backward: x = g_{k+1})
//                       acc[v] = a, or with kAccFold out[v] = r[v] + a and acc is only read (the last step writes dz)
// The once-per-row terms (tele, acc) belong to the non-accumulating call of a row; an accumulating call
// (the halo segment of a split row) adds only r[v] to what out holds.  The row's own operands (tele, acc and
// x[v], or the accumulated output) are loaded before the gather, so their latency hides behind it instead of
// following it (and acc[v] is written before the gather when it is not folded).  Rows of at most 4 floats per
// lane are held to 40 registers, 6 CTAs = 48 warps per SM, the occupancy of spmm_csr_kernel at these widths.
constexpr int kEpiTeleport = 0;
constexpr int kEpiAccum = 1;
constexpr int kAccRead = 2;    // acc_mode bits (bit 0: the acc term is on)
constexpr int kAccFold = 4;

template <int VEC, int CHUNKS, int EPI>
__global__ void __launch_bounds__(kThreads, VEC * CHUNKS <= 2 ? 6 : (VEC * CHUNKS <= 4 ? 5 : 1))
appnp_prop_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                  const float *__restrict__ x0, int64_t ld0, int64_t n_split,
                  const float *__restrict__ x1, int64_t ld1,
                  const float *__restrict__ pre, const float *__restrict__ post, float scale, float alpha,
                  const float *__restrict__ tele, int64_t ldt, float *__restrict__ accv, int64_t lda, int acc_mode,
                  int64_t row_begin, int64_t row_end, int F,
                  float *__restrict__ out, int64_t ldo, unsigned long long *__restrict__ next_row,
                  const int64_t *__restrict__ seg_start, const int64_t *__restrict__ seg_end, int accumulate) {
    const int lane = threadIdx.x & 31;
    bool colok[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) colok[c] = ((c * 32 + lane) * VEC) < F;
    const int64_t n_rows = row_end - row_begin;
    // what the epilogue adds to r: alpha * tele (teleport), a (folded acc term) or the accumulated output
    const bool once = !accumulate;
    const bool add_tele = EPI == kEpiTeleport && once && tele != nullptr;
    const bool acc_on = EPI == kEpiAccum && once && (acc_mode & 1);
    const bool fold = acc_on && (acc_mode & kAccFold);
    while (true) {
        unsigned long long grab = 0;
        if (lane == 0) grab = atomicAdd(next_row, 1ull);       // one row per grab, as spmm_csr_kernel's default
        grab = __shfl_sync(ADAQP_FULL_MASK, grab, 0);
        if ((int64_t)grab >= n_rows) break;
        const int64_t row = row_begin + (int64_t)grab;
        const int64_t o = row - row_begin;
        float *orow = out + o * ldo;
        float addend[CHUNKS][VEC];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            const int col = (c * 32 + lane) * VEC;
#pragma unroll
            for (int e = 0; e < VEC; ++e) addend[c][e] = 0.f;
            if (!colok[c]) continue;
            if (add_tele) {
                Vec<VEC>::load(tele + o * ldt + col, addend[c]);
            } else if (acc_on) {
                float own[VEC];
                Vec<VEC>::load(x0 + row * ld0 + col, own);
                if (acc_mode & kAccRead) Vec<VEC>::load(accv + o * lda + col, addend[c]);
#pragma unroll
                for (int e = 0; e < VEC; ++e) addend[c][e] = __fmaf_rn(alpha, own[e], addend[c][e]);
                if (!fold) Vec<VEC>::store(accv + o * lda + col, addend[c]);
            } else if (accumulate) {
                Vec<VEC>::load(orow + col, addend[c]);
            }
        }
        float acc[CHUNKS][VEC];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c)
#pragma unroll
            for (int e = 0; e < VEC; ++e) acc[c][e] = 0.f;
        const int64_t b = seg_start ? __ldg(seg_start + row) : __ldg(indptr + row);
        const int64_t e_ = seg_end ? __ldg(seg_end + row) : __ldg(indptr + row + 1);
        const int hints = 0;
        ADAQP_GATHER_SEGMENT(kUnroll, false, nullptr)
        const float s = post ? __fmul_rn(scale, __ldg(post + row)) : scale;
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            if (!colok[c]) continue;
            float r[VEC];
#pragma unroll
            for (int e = 0; e < VEC; ++e) {
                r[e] = __fmul_rn(acc[c][e], s);
                if (add_tele) r[e] = __fmaf_rn(alpha, addend[c][e], r[e]);
                else if (fold) r[e] = __fadd_rn(r[e], addend[c][e]);
                else if (accumulate) r[e] = __fadd_rn(addend[c][e], r[e]);
            }
            Vec<VEC>::store(orow + (c * 32 + lane) * VEC, r);
        }
    }
    frontier_release(next_row);
}

// ---------------------------------------------------------------------------------------
// Correct & Smooth propagation step (DESIGN §16): appnp_prop_kernel's teleport step, whole rows only (one pass per
// row, no segments), followed by a non-linear post-step that two partial sums of a row could not take:
//   r[v] = (scale * post[v]) * sum_{u in N(v)} pre[u] x[u]  (+ alpha * tele[v])
//   POST = kCsClamp: out[v] = fminf(fmaxf(r[v], lo), hi)
//   POST = kCsFix  : out[v] = fix[v] where y[v] >= 0 (the row's gather is skipped), else r[v]; tele is not read
//                    (the fixed rows are the only rows where the correct step's E0 is nonzero)
// tele, fix, y and out are indexed by v - row_begin.  The gather and the fmul / fmaf of the epilogue are those of
// appnp_prop_kernel, so with lo = -inf and hi = +inf the clamp step is bitwise its teleport step.  The row's own
// operands (tele; y and fix) are loaded before the gather.  Rows of at most 2 floats per lane are held to 40 registers
// (6 CTAs per SM) and <4, 1> to 48 (5 CTAs), as appnp_prop_kernel; <1, 4> and <2, 2> to 64 (4 CTAs): at 48 they spill.
constexpr int kCsClamp = 0;
constexpr int kCsFix = 1;

template <int VEC, int CHUNKS, int POST>
__global__ void __launch_bounds__(kThreads, VEC * CHUNKS <= 2 ? 6 : (VEC == 4 && CHUNKS == 1 ? 5 : (VEC * CHUNKS <= 4 ? 4 : 1)))
cs_prop_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
               const float *__restrict__ x0, int64_t ld0, int64_t n_split,
               const float *__restrict__ x1, int64_t ld1,
               const float *__restrict__ pre, const float *__restrict__ post, float scale, float alpha,
               const float *__restrict__ tele, int64_t ldt, const int32_t *__restrict__ y,
               const float *__restrict__ fix, int64_t ldf, float lo, float hi,
               int64_t row_begin, int64_t row_end, int F,
               float *__restrict__ out, int64_t ldo, unsigned long long *__restrict__ next_row) {
    const int lane = threadIdx.x & 31;
    bool colok[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) colok[c] = ((c * 32 + lane) * VEC) < F;
    const int64_t n_rows = row_end - row_begin;
    const bool add_tele = POST == kCsClamp && tele != nullptr;
    while (true) {
        unsigned long long grab = 0;
        if (lane == 0) grab = atomicAdd(next_row, 1ull);
        grab = __shfl_sync(ADAQP_FULL_MASK, grab, 0);
        if ((int64_t)grab >= n_rows) break;
        const int64_t row = row_begin + (int64_t)grab;
        const int64_t o = row - row_begin;
        float *orow = out + o * ldo;
        if (POST == kCsFix && __ldg(y + o) >= 0) {
            // a fixed row: its E0 row, no gather
#pragma unroll
            for (int c = 0; c < CHUNKS; ++c) {
                if (!colok[c]) continue;
                const int col = (c * 32 + lane) * VEC;
                float v[VEC];
                Vec<VEC>::load(fix + o * ldf + col, v);
                Vec<VEC>::store(orow + col, v);
            }
            continue;
        }
        float addend[CHUNKS][VEC];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
#pragma unroll
            for (int e = 0; e < VEC; ++e) addend[c][e] = 0.f;
            if (add_tele && colok[c]) Vec<VEC>::load(tele + o * ldt + (c * 32 + lane) * VEC, addend[c]);
        }
        float acc[CHUNKS][VEC];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c)
#pragma unroll
            for (int e = 0; e < VEC; ++e) acc[c][e] = 0.f;
        const int64_t b = __ldg(indptr + row);
        const int64_t e_ = __ldg(indptr + row + 1);
        const int hints = 0;
        ADAQP_GATHER_SEGMENT(kUnroll, false, nullptr)
        const float s = post ? __fmul_rn(scale, __ldg(post + row)) : scale;
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            if (!colok[c]) continue;
            float r[VEC];
#pragma unroll
            for (int e = 0; e < VEC; ++e) {
                r[e] = __fmul_rn(acc[c][e], s);
                if (add_tele) r[e] = __fmaf_rn(alpha, addend[c][e], r[e]);
                if (POST == kCsClamp) r[e] = fminf(fmaxf(r[e], lo), hi);
            }
            Vec<VEC>::store(orow + (c * 32 + lane) * VEC, r);
        }
    }
    frontier_release(next_row);
}

// ---------------------------------------------------------------------------------------
// Column-sliced gather (the default path for 16-byte rows of 256, 384, ... columns, DESIGN §3).
//
// The F columns are aggregated as ceil(F / slice_cols) slices of at most slice_cols <= 128 columns in
// one launch.  The frontier counter numbers the work (slice, row grab) slice-major, so every warp sweeps
// slice 0 over all rows before slice 1 starts: the source rows a slice touches are slice_cols * 4 bytes
// wide instead of F * 4, so the same L2 holds F / slice_cols times as many of the reused source rows.
// One warp per destination row, one float4 column of the slice per lane, kUnroll neighbour rows in
// flight per lane (the weights are shuffled after the loads are issued: 48 registers, no spills, the
// same occupancy as spmm_csr_kernel<4, 2>).  Every output element is
// the same __fmaf_rn chain in CSR order as spmm_csr_kernel's, followed by the same self term, mean,
// post norm and accumulate, so the results are bitwise those of the unsliced kernel.  SKIP and LIST as in
// spmm_csr_kernel; with LIST the units are (slice, list grab), slice-major.
template <bool SKIP, bool LIST>
__global__ void __launch_bounds__(kThreads)
spmm_csr_sliced_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                       const float *__restrict__ x0, int64_t ld0, int64_t n_split,
                       const float *__restrict__ x1, int64_t ld1,
                       const float *__restrict__ pre, const float *__restrict__ post,
                       int mean, int add_self, int64_t row_begin, int64_t row_end, int F, int slice_cols,
                       float *__restrict__ out, int64_t ldo, unsigned long long *__restrict__ next_row, int rows_per_grab,
                       const int64_t *__restrict__ seg_start, const int64_t *__restrict__ seg_end, int accumulate, int hints,
                       const uint8_t *__restrict__ live, const int32_t *__restrict__ rows, int64_t n_list) {
    const int lane = threadIdx.x & 31;
    const int64_t n_rows = LIST ? n_list : row_end - row_begin;
    const int64_t pos_begin = LIST ? 0 : row_begin, pos_end = LIST ? n_list : row_end;
    const int64_t n_grabs = (n_rows + rows_per_grab - 1) / rows_per_grab;
    const int64_t n_units = n_grabs * ((F + slice_cols - 1) / slice_cols);
    while (true) {
        unsigned long long unit = 0;
        if (lane == 0) unit = atomicAdd(next_row, 1ull);
        unit = __shfl_sync(ADAQP_FULL_MASK, unit, 0);
        if ((int64_t)unit >= n_units) break;
        const int64_t slice = (int64_t)unit / n_grabs, grab = (int64_t)unit % n_grabs;
        const int col = (int)slice * slice_cols + lane * 4;
        const bool colok = lane * 4 < slice_cols && col < F;
        const int64_t r_lo = pos_begin + grab * rows_per_grab;
        const int64_t r_hi = (r_lo + rows_per_grab < pos_end) ? r_lo + rows_per_grab : pos_end;
        for (int64_t pos = r_lo; pos < r_hi; ++pos) {
            const int64_t row = LIST ? (int64_t)__ldg(rows + pos) : pos;
            const int64_t row_b = __ldg(indptr + row), row_e = __ldg(indptr + row + 1);
            const int64_t b = seg_start ? __ldg(seg_start + row) : row_b;
            const int64_t e_ = seg_end ? __ldg(seg_end + row) : row_e;
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
            for (int64_t j0 = b; j0 < e_; j0 += 32) {
                int n = (e_ - j0) < 32 ? (int)(e_ - j0) : 32;
                int u = 0;
                float w = 0.f;
                if (lane < n) {
                    u = (hints & kHintIndexStreaming) ? __ldcs(indices + j0 + lane) : __ldg(indices + j0 + lane);
                    w = pre ? __ldg(pre + u) : 1.f;
                }
                if constexpr (SKIP) n = compact_live_window(lane, n, n_split, live, u, w);
                for (int k = 0; k < n; k += kUnroll) {
                    float v[kUnroll][4];
#pragma unroll
                    for (int t = 0; t < kUnroll; ++t) {
                        const int uu = __shfl_sync(ADAQP_FULL_MASK, u, (k + t) & 31);
                        const float *rs = (uu < n_split) ? (x0 + (int64_t)uu * ld0) : (x1 + ((int64_t)uu - n_split) * ld1);
                        if ((k + t) < n && colok) {
                            Vec<4>::load(rs + col, v[t]);
                        } else {
#pragma unroll
                            for (int e = 0; e < 4; ++e) v[t][e] = 0.f;
                        }
                    }
                    // the weights are shuffled once the loads are in flight: fewer live registers
#pragma unroll
                    for (int t = 0; t < kUnroll; ++t) {
                        float wt = __shfl_sync(ADAQP_FULL_MASK, w, (k + t) & 31);
                        if ((k + t) >= n) wt = 0.f;
#pragma unroll
                        for (int e = 0; e < 4; ++e) acc[e] = __fmaf_rn(wt, v[t][e], acc[e]);
                    }
                }
            }
            if (!colok) continue;
            if (add_self) {
                const float ws = pre ? __ldg(pre + row) : 1.f;
                const float *rs = (row < n_split) ? (x0 + row * ld0) : (x1 + (row - n_split) * ld1);
                float v[4];
                Vec<4>::load(rs + col, v);
#pragma unroll
                for (int e = 0; e < 4; ++e) acc[e] = __fmaf_rn(ws, v[e], acc[e]);
            }
            const float deg = (float)(row_e - row_b);       // mean divides by the full in-degree
            const float ps = post ? __ldg(post + row) : 1.f;
            float *orow = out + (row - row_begin) * ldo + col;
            float prev[4];
            if (accumulate) Vec<4>::load(orow, prev);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                float r = acc[e];
                if (mean && deg > 0.f) r = __fdiv_rn(r, deg);
                if (post) r = __fmul_rn(r, ps);
                if (accumulate) r = __fadd_rn(prev[e], r);
                acc[e] = r;
            }
            if (hints & kHintStoreStreaming) Vec<4>::store_cs(orow, acc);
            else Vec<4>::store(orow, acc);
        }
    }
    frontier_release(next_row);
}

// Row liveness of a [rows, F] fp32 matrix with pitch ld: live[r] = 1 when some x[r, c] != 0 (NaN included), else 0.
// One warp per row (grid-stride), VEC-wide coalesced loads: one read of the matrix, the answer by warp vote.
template <int VEC>
__global__ void __launch_bounds__(kThreads)
row_live_kernel(const float *__restrict__ x, int64_t ld, int64_t rows, int F, uint8_t *__restrict__ live) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = (int64_t)gridDim.x * kWarps;
    for (int64_t r = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); r < rows; r += nwarps) {
        const float *rp = x + r * ld;
        bool nz = false;
#pragma unroll 4
        for (int c = lane * VEC; c < F; c += 32 * VEC) {
            float v[VEC];
            Vec<VEC>::load(rp + c, v);
#pragma unroll
            for (int e = 0; e < VEC; ++e) nz |= v[e] != 0.f;
        }
        nz = __any_sync(ADAQP_FULL_MASK, nz);
        if (lane == 0) live[r] = nz ? 1 : 0;
    }
}

// ---------------------------------------------------------------------------------------
// Column-sliced propagation step (GCNII's hidden-width rows, DESIGN §14): spmm_csr_sliced_kernel's slice-major
// schedule and gather with appnp_prop_kernel's epilogue, applied per slice to that slice's columns of tele / acc /
// x[v] / out.  One destination row per unit (unit = slice * n_rows + row), one float4 of the slice per lane, kUnroll
// neighbour rows in flight, the weights shuffled after the loads are issued.  The row's own operands are loaded
// before the gather, and the once-per-row terms belong to the non-accumulating call, as in appnp_prop_kernel.
// Every output element is the same __fmaf_rn chain in CSR order, followed by the same __fmul_rn(acc, scale * post)
// and epilogue ops, so the result is bitwise that of appnp_prop_kernel.
template <int EPI>
__global__ void __launch_bounds__(kThreads)
appnp_prop_sliced_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                         const float *__restrict__ x0, int64_t ld0, int64_t n_split,
                         const float *__restrict__ x1, int64_t ld1,
                         const float *__restrict__ pre, const float *__restrict__ post, float scale, float alpha,
                         const float *__restrict__ tele, int64_t ldt, float *__restrict__ accv, int64_t lda, int acc_mode,
                         int64_t row_begin, int64_t row_end, int F, int slice_cols,
                         float *__restrict__ out, int64_t ldo, unsigned long long *__restrict__ next_row,
                         const int64_t *__restrict__ seg_start, const int64_t *__restrict__ seg_end, int accumulate) {
    const int lane = threadIdx.x & 31;
    const int64_t n_rows = row_end - row_begin;
    const int64_t n_units = n_rows * ((F + slice_cols - 1) / slice_cols);
    const bool once = !accumulate;
    const bool add_tele = EPI == kEpiTeleport && once && tele != nullptr;
    const bool acc_on = EPI == kEpiAccum && once && (acc_mode & 1);
    const bool fold = acc_on && (acc_mode & kAccFold);
    while (true) {
        unsigned long long unit = 0;
        if (lane == 0) unit = atomicAdd(next_row, 1ull);
        unit = __shfl_sync(ADAQP_FULL_MASK, unit, 0);
        if ((int64_t)unit >= n_units) break;
        const int64_t slice = (int64_t)unit / n_rows, o = (int64_t)unit % n_rows;
        const int col = (int)slice * slice_cols + lane * 4;
        const bool colok = lane * 4 < slice_cols && col < F;
        const int64_t row = row_begin + o;
        float *orow = out + o * ldo + col;
        float addend[4] = {0.f, 0.f, 0.f, 0.f};
        if (colok) {
            if (add_tele) {
                Vec<4>::load(tele + o * ldt + col, addend);
            } else if (acc_on) {
                float own[4];
                Vec<4>::load(x0 + row * ld0 + col, own);
                if (acc_mode & kAccRead) Vec<4>::load(accv + o * lda + col, addend);
#pragma unroll
                for (int e = 0; e < 4; ++e) addend[e] = __fmaf_rn(alpha, own[e], addend[e]);
                if (!fold) Vec<4>::store(accv + o * lda + col, addend);
            } else if (accumulate) {
                Vec<4>::load(orow, addend);
            }
        }
        const int64_t b = seg_start ? __ldg(seg_start + row) : __ldg(indptr + row);
        const int64_t e_ = seg_end ? __ldg(seg_end + row) : __ldg(indptr + row + 1);
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int64_t j0 = b; j0 < e_; j0 += 32) {
            const int n = (e_ - j0) < 32 ? (int)(e_ - j0) : 32;
            int u = 0;
            float w = 0.f;
            if (lane < n) {
                u = __ldg(indices + j0 + lane);
                w = pre ? __ldg(pre + u) : 1.f;
            }
            for (int k = 0; k < n; k += kUnroll) {
                float v[kUnroll][4];
#pragma unroll
                for (int t = 0; t < kUnroll; ++t) {
                    const int uu = __shfl_sync(ADAQP_FULL_MASK, u, (k + t) & 31);
                    const float *rs = (uu < n_split) ? (x0 + (int64_t)uu * ld0) : (x1 + ((int64_t)uu - n_split) * ld1);
                    if ((k + t) < n && colok) {
                        Vec<4>::load(rs + col, v[t]);
                    } else {
#pragma unroll
                        for (int e = 0; e < 4; ++e) v[t][e] = 0.f;
                    }
                }
#pragma unroll
                for (int t = 0; t < kUnroll; ++t) {
                    float wt = __shfl_sync(ADAQP_FULL_MASK, w, (k + t) & 31);
                    if ((k + t) >= n) wt = 0.f;
#pragma unroll
                    for (int e = 0; e < 4; ++e) acc[e] = __fmaf_rn(wt, v[t][e], acc[e]);
                }
            }
        }
        if (!colok) continue;
        const float s = post ? __fmul_rn(scale, __ldg(post + row)) : scale;
        float r[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            r[e] = __fmul_rn(acc[e], s);
            if (add_tele) r[e] = __fmaf_rn(alpha, addend[e], r[e]);
            else if (fold) r[e] = __fadd_rn(r[e], addend[e]);
            else if (accumulate) r[e] = __fadd_rn(addend[e], r[e]);
        }
        Vec<4>::store(orow, r);
    }
    frontier_release(next_row);
}

// ---------------------------------------------------------------------------------------
// v2: asynchronous row gather through a lane-private shared-memory ring (cp.async / LDGSTS).
//
// v1 stages gathered rows in registers: bytes in flight per SM are bounded by the register
// file and the load -> wait -> consume phases do not overlap.  Here every lane copies its own 16-byte column chunks of
// each neighbour row with cp.async into a ring of kStages row slots per warp and consumes
// the oldest slot (LDS.128 + FFMA) while the next kStages-1 rows are still in flight:
// a continuous software pipeline with no register cost per in-flight row and no cross-lane
// synchronisation (a lane only ever reads the bytes it copied; completion is tracked by
// per-thread cp.async groups).  Neighbour ids and their norm weights travel in
// lane-distributed register windows that are prefetched one and two windows ahead.  Rows
// are handed to warps as contiguous nnz-balanced chunks, so the pipeline stays full across
// row boundaries and a hub row costs one warp its own length, not a whole CTA's.
//
// Requires F % 4 == 0 and 16-byte aligned rows (F = 100, 200, 256, 300 ...); anything else
// (F = 602) uses v1.
constexpr int kStages = 8;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// first row r in [lo, hi] with indptr[r] >= target
__device__ __forceinline__ int64_t row_lower_bound(const int64_t *__restrict__ indptr, int64_t lo, int64_t hi, int64_t target) {
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(indptr + mid) < target) lo = mid + 1; else hi = mid;
    }
    return lo;
}

template <int CHUNKS>
__global__ void __launch_bounds__(kThreads)
spmm_csr_ring_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                     const float *__restrict__ x0, int64_t ld0, int64_t n_split,
                     const float *__restrict__ x1, int64_t ld1,
                     const float *__restrict__ pre, const float *__restrict__ post,
                     int mean, int add_self, int64_t row_begin, int64_t row_end, int F,
                     float *__restrict__ out, int64_t ldo, int64_t chunk_nnz) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    // ring[warp][stage][chunk][lane] of 16 bytes: a lane's chunk is contiguous with its
    // neighbours' (conflict-free LDS.128 / LDGSTS.128)
    const uint32_t ring_u = smem_u32(smem_raw) + (uint32_t)wib * kStages * CHUNKS * 512u + (uint32_t)lane * 16u;
    const float4 *ring = reinterpret_cast<const float4 *>(smem_raw) + (size_t)wib * kStages * CHUNKS * 32 + lane;

    bool colok[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) colok[c] = ((c * 32 + lane) * 4) < F;
    const int64_t nnz_base = __ldg(indptr + row_begin);
    const int64_t nnz_end_all = __ldg(indptr + row_end);
    int64_t n_chunks = (nnz_end_all - nnz_base + chunk_nnz - 1) / chunk_nnz;
    if (n_chunks < 1) n_chunks = 1;   // rows without edges still produce output

    const int64_t warp = (int64_t)blockIdx.x * kWarps + wib;
    const int64_t nwarps = (int64_t)gridDim.x * kWarps;
    for (int64_t chunk = warp; chunk < n_chunks; chunk += nwarps) {
        // rows whose first nnz falls into this chunk's nnz window
        const int64_t lo_nnz = nnz_base + chunk * chunk_nnz;
        const bool last = (chunk == n_chunks - 1);
        const int64_t r0 = (chunk == 0) ? row_begin : row_lower_bound(indptr, row_begin, row_end, lo_nnz);
        const int64_t r1 = last ? row_end : row_lower_bound(indptr, row_begin, row_end, lo_nnz + chunk_nnz);
        if (r0 >= r1) continue;
        int64_t pc = __ldg(indptr + r0);                       // consume cursor
        const int64_t pend = last ? nnz_end_all : __ldg(indptr + r1);
        int64_t pi = pc;                                       // issue cursor
        // lane-distributed windows of 32 neighbour ids / weights: [cur | nxt | nx2 (ids only)]
        int64_t wb = pc;
        int idx_cur = (wb + lane < pend) ? __ldg(indices + wb + lane) : 0;
        int idx_nxt = (wb + 32 + lane < pend) ? __ldg(indices + wb + 32 + lane) : 0;
        int idx_nx2 = (wb + 64 + lane < pend) ? __ldg(indices + wb + 64 + lane) : 0;
        float w_cur = (pre && wb + lane < pend) ? __ldg(pre + idx_cur) : 1.f;
        float w_nxt = (pre && wb + 32 + lane < pend) ? __ldg(pre + idx_nxt) : 1.f;
        float w_prev = 1.f;   // the consume side lags the issue side by < kStages <= 32 ids
        int64_t row = r0;
        int64_t rend = __ldg(indptr + row + 1);
        float acc[CHUNKS][4];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) { acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = 0.f; }
        uint32_t si = 0, sc = 0;                               // ring positions

        auto issue_one = [&]() {
            if (pi < pend) {
                if (pi >= wb + 32) {                           // slide the issue windows
                    wb += 32;
                    idx_cur = idx_nxt; idx_nxt = idx_nx2;
                    idx_nx2 = (wb + 64 + lane < pend) ? __ldg(indices + wb + 64 + lane) : 0;
                    w_prev = w_cur;
                    w_cur = w_nxt;
                    w_nxt = (pre && wb + 32 + lane < pend) ? __ldg(pre + idx_nxt) : 1.f;
                }
                const int u = __shfl_sync(ADAQP_FULL_MASK, idx_cur, (int)(pi - wb));
                const float *src = (u < n_split) ? (x0 + (int64_t)u * ld0) : (x1 + ((int64_t)u - n_split) * ld1);
                const uint32_t dst = ring_u + (si % kStages) * (CHUNKS * 512u);
#pragma unroll
                for (int c = 0; c < CHUNKS; ++c)
                    if (colok[c]) cp_async_16(dst + c * 512u, src + (c * 32 + lane) * 4);
                ++pi;
                ++si;
            }
            cp_async_commit();                                 // empty groups keep the queue depth constant
        };

#pragma unroll 1
        for (int k = 0; k < kStages - 1; ++k) issue_one();     // prologue: fill the pipeline

        while (true) {
            // ---- finish every row that is complete (also rows without in-edges)
            while (row < r1 && pc == rend) {
                const int64_t rb = __ldg(indptr + row);
                if (add_self) {
                    const float ws = pre ? __ldg(pre + row) : 1.f;
                    const float *rp = (row < n_split) ? (x0 + row * ld0) : (x1 + (row - n_split) * ld1);
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c) if (colok[c]) {
                        const float4 t = __ldg(reinterpret_cast<const float4 *>(rp + (c * 32 + lane) * 4));
                        acc[c][0] = __fmaf_rn(ws, t.x, acc[c][0]); acc[c][1] = __fmaf_rn(ws, t.y, acc[c][1]);
                        acc[c][2] = __fmaf_rn(ws, t.z, acc[c][2]); acc[c][3] = __fmaf_rn(ws, t.w, acc[c][3]);
                    }
                }
                const float deg = (float)(rend - rb);
                const float ps = post ? __ldg(post + row) : 1.f;
                float *orow = out + (row - row_begin) * ldo;
#pragma unroll
                for (int c = 0; c < CHUNKS; ++c) if (colok[c]) {
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        float r = acc[c][e];
                        if (mean && deg > 0.f) r = __fdiv_rn(r, deg);
                        if (post) r = __fmul_rn(r, ps);
                        acc[c][e] = r;
                    }
                    *reinterpret_cast<float4 *>(orow + (c * 32 + lane) * 4) = make_float4(acc[c][0], acc[c][1], acc[c][2], acc[c][3]);
                    acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = 0.f;
                }
                ++row;
                if (row < r1) rend = __ldg(indptr + row + 1);
            }
            if (pc >= pend) break;
            issue_one();                                       // one more row in flight ...
            cp_async_wait<kStages - 1>();                      // ... and the oldest has landed (for this lane)
            const float wa = __shfl_sync(ADAQP_FULL_MASK, w_cur, (int)((pc - wb) & 31));
            const float wp = __shfl_sync(ADAQP_FULL_MASK, w_prev, (int)((pc - wb + 32) & 31));
            const float w = (pc >= wb) ? wa : wp;
            const float4 *slot = ring + (size_t)(sc % kStages) * (CHUNKS * 32);
#pragma unroll
            for (int c = 0; c < CHUNKS; ++c) if (colok[c]) {
                const float4 t = slot[c * 32];
                acc[c][0] = __fmaf_rn(w, t.x, acc[c][0]); acc[c][1] = __fmaf_rn(w, t.y, acc[c][1]);
                acc[c][2] = __fmaf_rn(w, t.z, acc[c][2]); acc[c][3] = __fmaf_rn(w, t.w, acc[c][3]);
            }
            ++sc;
            ++pc;
        }
        cp_async_wait<0>();
    }
}

// ---------------------------------------------------------------------------------------
// v3 / v4: TMA row gather into a per-warp shared-memory ring (opt-in, option spmm_impl = 3 / 4).
//
// v3 gathers through a 2-D tensor map over the source matrix with a one-row box {F, 1}: per group
// of up to four neighbour rows, one `cp.async.bulk.tensor.2d ... tile` (SASS UTMALDG) per row, all
// completing on the slot's mbarrier.  v4 issues one plain `cp.async.bulk` (UBLKCP) per neighbour row
// into the same ring, with no tensor map.  Scheduling is the frontier scheme of v1 (rows from a global
// counter, so the source rows being reused stay inside L2); the ring pipelines across the rows
// of one grab.  A group never mixes local and halo sources (two tensor maps): the columns of a
// row are sorted, so every 32-id window splits into a local prefix and a halo suffix.
// Rows sit 128-byte aligned in a slot (the alignment a tensor copy's destination needs).
// Needs 16-byte rows and F <= 256 (one TMA box); anything else runs v1.
constexpr int kRingWarps = 16;
constexpr int kRingThreads = kRingWarps * 32;

struct __align__(16) RingMeta {
    float w[4];     // pre-norm weights of the slot's rows
    int cnt;        // valid rows in the slot (0..4)
    int last;       // 1: the destination row is complete after this slot
    int pad[2];
};

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void tma_row(uint32_t dst, const CUtensorMap *map, int row, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst), "l"(map), "r"(0), "r"(row), "r"(bar) : "memory");
}

// bytes between the rows of a ring slot
__host__ __device__ __forceinline__ uint32_t ring_row_stride(int F) { return ((uint32_t)F * 4u + 127u) & ~127u; }

template <int CHUNKS, bool TENSOR_MAP>
__global__ void __launch_bounds__(kRingThreads, 1)
spmm_csr_tma_kernel(const __grid_constant__ CUtensorMap map0, const __grid_constant__ CUtensorMap map1,
                    const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                    const float *__restrict__ x0, int64_t ld0, int64_t n_split,
                    const float *__restrict__ x1, int64_t ld1,
                    const float *__restrict__ pre, const float *__restrict__ post,
                    int mean, int add_self, int64_t row_begin, int64_t row_end, int F,
                    float *__restrict__ out, int64_t ldo, unsigned long long *__restrict__ next_row, int rows_per_grab,
                    const int64_t *__restrict__ seg_start, const int64_t *__restrict__ seg_end, int accumulate,
                    int stages) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    const int lane = threadIdx.x & 31;
    const int wib = threadIdx.x >> 5;
    const uint32_t rowbytes = (uint32_t)F * 4u;
    const uint32_t rowstride = ring_row_stride(F);
    const uint32_t slot_bytes = 4u * rowstride;
    uint8_t *ring = smem_raw + (size_t)wib * stages * slot_bytes;
    uint8_t *aux = smem_raw + (size_t)kRingWarps * stages * slot_bytes;
    RingMeta *metas = reinterpret_cast<RingMeta *>(aux) + wib * stages;
    const uint32_t bars_u = smem_u32(aux + (size_t)kRingWarps * stages * sizeof(RingMeta)) + (uint32_t)(wib * stages) * 8u;
    const uint32_t ring_u = smem_u32(ring);
    if (lane == 0)
        for (int st = 0; st < stages; ++st) mbar_init(bars_u + 8u * st, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncwarp();

    bool colok[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) colok[c] = ((c * 32 + lane) * 4) < F;
    const int64_t n_rows = row_end - row_begin;
    int si = 0, sc = 0;                 // issue / consume slot
    uint32_t pc = 0;                    // parity of the consume side's current lap
    int inflight = 0;

    while (true) {
        unsigned long long grab = 0;
        if (lane == 0) grab = atomicAdd(next_row, (unsigned long long)rows_per_grab);
        grab = __shfl_sync(ADAQP_FULL_MASK, grab, 0);
        if ((int64_t)grab >= n_rows) break;
        const int64_t r_hi = ((int64_t)grab + rows_per_grab < n_rows) ? (int64_t)grab + rows_per_grab : n_rows;
        int64_t rc = row_begin + (int64_t)grab;          // row the consume side is accumulating
        float acc[CHUNKS][4];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = 0.f;

        auto consume_one = [&]() {
            mbar_wait(bars_u + 8u * sc, pc);
            const RingMeta m = metas[sc];
            const float4 *slot = reinterpret_cast<const float4 *>(ring + (size_t)sc * slot_bytes);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                if (k < m.cnt) {
                    const float w = m.w[k];
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c) {
                        if (colok[c]) {
                            const float4 t = slot[k * (rowstride >> 4) + c * 32 + lane];
                            acc[c][0] = __fmaf_rn(w, t.x, acc[c][0]); acc[c][1] = __fmaf_rn(w, t.y, acc[c][1]);
                            acc[c][2] = __fmaf_rn(w, t.z, acc[c][2]); acc[c][3] = __fmaf_rn(w, t.w, acc[c][3]);
                        }
                    }
                }
            }
            if (++sc == stages) { sc = 0; pc ^= 1u; }
            --inflight;
            if (m.last) {               // destination row rc is complete
                const int64_t row = rc;
                if (add_self) {
                    const float ws = pre ? __ldg(pre + row) : 1.f;
                    const float *rp = (row < n_split) ? (x0 + row * ld0) : (x1 + (row - n_split) * ld1);
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c) if (colok[c]) {
                        const float4 t = __ldg(reinterpret_cast<const float4 *>(rp + (c * 32 + lane) * 4));
                        acc[c][0] = __fmaf_rn(ws, t.x, acc[c][0]); acc[c][1] = __fmaf_rn(ws, t.y, acc[c][1]);
                        acc[c][2] = __fmaf_rn(ws, t.z, acc[c][2]); acc[c][3] = __fmaf_rn(ws, t.w, acc[c][3]);
                    }
                }
                const float deg = (float)(__ldg(indptr + row + 1) - __ldg(indptr + row));
                const float ps = post ? __ldg(post + row) : 1.f;
                float *orow = out + (row - row_begin) * ldo;
#pragma unroll
                for (int c = 0; c < CHUNKS; ++c) if (colok[c]) {
                    float4 prev = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (accumulate) prev = *reinterpret_cast<const float4 *>(orow + (c * 32 + lane) * 4);
                    const float pv[4] = {prev.x, prev.y, prev.z, prev.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        float r = acc[c][e];
                        if (mean && deg > 0.f) r = __fdiv_rn(r, deg);
                        if (post) r = __fmul_rn(r, ps);
                        if (accumulate) r = __fadd_rn(pv[e], r);
                        acc[c][e] = r;
                    }
                    *reinterpret_cast<float4 *>(orow + (c * 32 + lane) * 4) = make_float4(acc[c][0], acc[c][1], acc[c][2], acc[c][3]);
                    acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = 0.f;
                }
                ++rc;
            }
            __syncwarp();               // every lane is done with the slot before it is refilled
        };

        for (int64_t row = row_begin + (int64_t)grab; row < row_begin + r_hi; ++row) {
            const int64_t b = seg_start ? __ldg(seg_start + row) : __ldg(indptr + row);
            const int64_t e_ = seg_end ? __ldg(seg_end + row) : __ldg(indptr + row + 1);
            if (b >= e_) {              // no neighbours in this launch's segment: an empty, final slot
                while (inflight >= stages) consume_one();
                if (lane == 0) {
                    metas[si].cnt = 0;
                    metas[si].last = 1;
                    mbar_arrive(bars_u + 8u * si);
                }
                __syncwarp();
                if (++si == stages) si = 0;
                ++inflight;
                continue;
            }
            for (int64_t j0 = b; j0 < e_; j0 += 32) {
                const int n = (e_ - j0) < 32 ? (int)(e_ - j0) : 32;
                int u = 0;
                float w = 0.f;
                if (lane < n) {
                    u = __ldg(indices + j0 + lane);
                    w = pre ? __ldg(pre + u) : 1.f;
                }
                const int nl = __popc(__ballot_sync(ADAQP_FULL_MASK, lane < n && u < n_split));   // sorted: local prefix
                const int gl = (nl + 3) >> 2;
                const int ng = gl + ((n - nl + 3) >> 2);
                for (int g = 0; g < ng; ++g) {
                    while (inflight >= stages) consume_one();
                    const bool halo = g >= gl;
                    const int base = halo ? nl + 4 * (g - gl) : 4 * g;
                    const int lim = halo ? n : nl;
                    const int cnt = (lim - base) < 4 ? (lim - base) : 4;
                    const int srcl = (base + (lane & 3)) & 31;
                    int uv = __shfl_sync(ADAQP_FULL_MASK, u, srcl);
                    const float wv = __shfl_sync(ADAQP_FULL_MASK, w, srcl);
                    const int ufirst = __shfl_sync(ADAQP_FULL_MASK, u, base & 31);
                    if ((lane & 3) >= cnt) uv = ufirst;          // pad with the group's first row (never fetched)
                    const int r1 = __shfl_sync(ADAQP_FULL_MASK, uv, 1), r2 = __shfl_sync(ADAQP_FULL_MASK, uv, 2),
                              r3 = __shfl_sync(ADAQP_FULL_MASK, uv, 3);
                    if (lane < 4) metas[si].w[lane] = wv;
                    if (lane == 0) {
                        metas[si].cnt = cnt;
                        metas[si].last = (j0 + 32 >= e_ && g == ng - 1) ? 1 : 0;
                        const uint32_t bar = bars_u + 8u * si;
                        const uint32_t dst = ring_u + (uint32_t)si * slot_bytes;
                        const int off = halo ? (int)n_split : 0;
                        const int rr[4] = {uv - off, r1 - off, r2 - off, r3 - off};
                        mbar_arrive_expect_tx(bar, (uint32_t)cnt * rowbytes);
                        if (TENSOR_MAP) {
                            const CUtensorMap *map = halo ? &map1 : &map0;
#pragma unroll
                            for (int k = 0; k < 4; ++k)
                                if (k < cnt) tma_row(dst + (uint32_t)k * rowstride, map, rr[k], bar);
                        } else {
                            const float *sb = halo ? x1 : x0;
                            const int64_t ld = halo ? ld1 : ld0;
#pragma unroll
                            for (int k = 0; k < 4; ++k)
                                if (k < cnt) bulk_g2s(dst + (uint32_t)k * rowstride, sb + (int64_t)rr[k] * ld, rowbytes, bar);
                        }
                    }
                    __syncwarp();
                    if (++si == stages) si = 0;
                    ++inflight;
                }
            }
        }
        while (inflight > 0) consume_one();
    }
    frontier_release(next_row);
}

inline bool aligned(const void *p, int vec) { return ((uintptr_t)p & ((uintptr_t)vec * 4 - 1)) == 0; }

// Slice width the default path picks for 16-byte rows when spmm_slice_cols is 0 (0 = unsliced): 128-column
// slices when F is a multiple of 128 above 128, so every slice keeps all 32 lanes busy.  Slices with idle
// lanes measured slower than the unsliced kernel (F = 200 as 2 x 100, F = 256 as 3 x 88 or 4 x 64; DESIGN §3).
int auto_slice_cols(int F) { return (F > 128 && F % 128 == 0) ? 128 : 0; }

}  // namespace

namespace {

typedef CUresult (*TensorMapEncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                           const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                           CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// libcuda is not linked: the encoder comes from the driver the process already runs on
TensorMapEncodeTiledFn tensor_map_encoder() {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess) return nullptr;
    return q == cudaDriverEntryPointSuccess ? (TensorMapEncodeTiledFn)fn : nullptr;
}

// 2-D fp32 map {F, rows} with box {F, 1}: one tensor copy fetches one source row
int make_row_map(CUtensorMap *m, const float *base, int64_t rows, int F, int64_t ld) {
    TensorMapEncodeTiledFn enc = tensor_map_encoder();
    ADAQP_REQUIRE(enc != nullptr, ADAQP_EINVAL, "cuTensorMapEncodeTiled not available from the driver");
    const cuuint64_t dims[2] = {(cuuint64_t)F, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
    const cuuint32_t box[2] = {(cuuint32_t)F, 1};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void *)base, dims, strides, box, estr,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    ADAQP_REQUIRE(r == CUDA_SUCCESS, ADAQP_EINVAL, "cuTensorMapEncodeTiled failed (%d)", (int)r);
    return 0;
}

// One {next_row, finished} pair per (device, stream): launches on one stream are serialised and the
// kernel zeroes the pair when it finishes, so the pair is never shared by two live launches.
unsigned long long *frontier_counter(int dev, cudaStream_t s) {
    static std::mutex mu;
    static std::unordered_map<uint64_t, unsigned long long *> pairs;
    std::lock_guard<std::mutex> lock(mu);
    const uint64_t key = ((uint64_t)(uintptr_t)s << 6) ^ (uint64_t)dev;
    auto it = pairs.find(key);
    if (it != pairs.end()) return it->second;
    unsigned long long *p = nullptr;
    if (cudaMalloc(&p, 2 * sizeof(unsigned long long)) != cudaSuccess) return nullptr;
    if (cudaMemset(p, 0, 2 * sizeof(unsigned long long)) != cudaSuccess) return nullptr;
    pairs.emplace(key, p);
    return p;
}

}  // namespace

unsigned long long *adaqp_frontier_counter(int dev, cudaStream_t s) { return frontier_counter(dev, s); }

extern "C" {

int adaqp_spmm_csr_seg_f32(const int64_t *indptr, const int64_t *seg_start, const int64_t *seg_end,
                           const int32_t *indices, const float *x0, int64_t ld0,
                           int64_t n_split, const float *x1, int64_t ld1, const float *pre,
                           const float *post, int mean, int add_self, int accumulate, int64_t row_begin,
                           int64_t row_end, int32_t F, float *out, int64_t ldo, const uint8_t *live,
                           const int32_t *rows, int64_t n_list, void *stream) {
    ADAQP_REQUIRE(F > 0 && F <= 1024, ADAQP_ELIMIT, "adaqp_spmm_csr_f32: F=%d outside (0,1024]", F);
    ADAQP_REQUIRE(row_end >= row_begin && row_begin >= 0, ADAQP_EINVAL, "adaqp_spmm_csr_f32: bad row range");
    ADAQP_REQUIRE(!rows || (n_list >= 0 && n_list <= row_end - row_begin), ADAQP_EINVAL,
                  "adaqp_spmm_csr_seg_f32: row list of %lld ids for a range of %lld rows", (long long)n_list,
                  (long long)(row_end - row_begin));
    ADAQP_REQUIRE(!(rows && live), ADAQP_EINVAL, "adaqp_spmm_csr_seg_f32: a row list and row liveness together");
    if (row_end == row_begin) return 0;
    if (rows && n_list == 0) return 0;      // nothing listed: no launch (a grid of 0 is an error), counter untouched
    ADAQP_REQUIRE(indptr && indices && x0 && out, ADAQP_EINVAL, "adaqp_spmm_csr_f32: null pointer");
    int vec = 4;
    auto fits = [&](int v) {
        if (F % v || ld0 % v || ldo % v) return false;
        if (!aligned(x0, v) || !aligned(out, v)) return false;
        if (x1 && (!aligned(x1, v) || (ld1 % v))) return false;
        return true;
    };
    while (vec > 1 && !fits(vec)) vec >>= 1;
    const int nchunks = (F + 32 * vec - 1) / (32 * vec);
    const int64_t n_rows = row_end - row_begin;
    const int sms = adaqp_sm_count() > 0 ? adaqp_sm_count() : 132;
    const AdaqpOptions &opt = adaqp_options();
    cudaStream_t s = (cudaStream_t)stream;
    const int impl = opt.spmm_impl;
    // v2 (cp.async ring) needs 16-byte rows: F % 4 == 0, strides % 4 == 0, 16-byte aligned bases
    if (impl == 2 && !rows && vec == 4 && nchunks <= 8 && !seg_start && !seg_end && !accumulate) {
        auto launch = [&](auto kernel, int C) {
            const size_t smem = (size_t)kWarps * kStages * C * 512;
            int ctas_per_sm = (int)((200 * 1024) / (smem + 1024));
            if (ctas_per_sm > 4) ctas_per_sm = 4;
            if (ctas_per_sm < 1) ctas_per_sm = 1;
            int64_t g2 = (int64_t)sms * ctas_per_sm;
            const int64_t max_ctas = (n_rows + kWarps - 1) / kWarps;
            if (g2 > max_ctas) g2 = max_ctas;
            const int64_t chunk_nnz = 2048;   // nnz-balanced work units, many per warp
            cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
            kernel<<<(unsigned)g2, kThreads, smem, s>>>(indptr, indices, x0, ld0, n_split, x1, ld1, pre, post, mean,
                                                        add_self, row_begin, row_end, F, out, ldo, chunk_nnz);
        };
        if (nchunks <= 1) launch(spmm_csr_ring_kernel<1>, 1);
        else if (nchunks <= 2) launch(spmm_csr_ring_kernel<2>, 2);
        else if (nchunks <= 3) launch(spmm_csr_ring_kernel<3>, 3);
        else if (nchunks <= 4) launch(spmm_csr_ring_kernel<4>, 4);
        else if (nchunks <= 6) launch(spmm_csr_ring_kernel<6>, 6);
        else launch(spmm_csr_ring_kernel<8>, 8);
        return adaqp_check_launch("spmm_csr_ring_kernel");
    }
    int dev = 0;
    ADAQP_CUDA(cudaGetDevice(&dev));
    unsigned long long *counter = frontier_counter(dev, s);
    ADAQP_REQUIRE(counter != nullptr, ADAQP_EINVAL, "adaqp_spmm_csr_seg_f32: row counter allocation failed");
    // v3 / v4 (TMA ring): one TMA box per row -> F <= 256, 16-byte rows
    if ((impl == 3 || impl == 4) && !rows && vec == 4 && F <= 256 && nchunks <= 2) {
        CUtensorMap map0, map1;
        memset(&map0, 0, sizeof(map0));
        memset(&map1, 0, sizeof(map1));
        if (impl == 3) {
            // x0 holds the ids below n_split; the halo matrix's row count is not part of the ABI, the
            // map only bounds-checks coordinates, so give it the largest extent a row coordinate can have
            const int64_t rows0 = n_split > 0 ? n_split : 1;
            int rc = make_row_map(&map0, x0, rows0, F, ld0);
            if (rc) return rc;
            if (x1) { rc = make_row_map(&map1, x1, (int64_t)1 << 31, F, ld1); if (rc) return rc; }
        }
        const uint32_t slot_bytes = 4u * ring_row_stride(F);
        int stages = (int)((200u * 1024u) / ((size_t)kRingWarps * (slot_bytes + sizeof(RingMeta) + 8)));
        if (stages > 8) stages = 8;
        ADAQP_REQUIRE(stages >= 2, ADAQP_ELIMIT, "adaqp_spmm_csr_seg_f32: ring does not fit shared memory");
        const size_t smem = (size_t)kRingWarps * stages * (slot_bytes + sizeof(RingMeta) + 8);
        int64_t grid = (n_rows + kRingWarps - 1) / kRingWarps;
        if (grid > sms) grid = sms;
        const int grab = opt.spmm_rows_per_grab > 0 ? opt.spmm_rows_per_grab : 4;
        auto launch = [&](auto kernel) {
            cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            kernel<<<(unsigned)grid, kRingThreads, smem, s>>>(map0, map1, indptr, indices, x0, ld0, n_split, x1, ld1, pre, post,
                                                             mean, add_self, row_begin, row_end, F, out, ldo, counter, grab,
                                                             seg_start, seg_end, accumulate, stages);
        };
        if (impl == 3) { if (nchunks <= 1) launch(spmm_csr_tma_kernel<1, true>); else launch(spmm_csr_tma_kernel<2, true>); }
        else { if (nchunks <= 1) launch(spmm_csr_tma_kernel<1, false>); else launch(spmm_csr_tma_kernel<2, false>); }
        return adaqp_check_launch("spmm_csr_tma_kernel");
    }
    const int64_t cta_cap = (int64_t)sms * (opt.spmm_ctas_per_sm > 0 ? opt.spmm_ctas_per_sm : 8);
    const int hints = opt.spmm_hints;
    // column slices of 16-byte rows (spmm_csr_sliced_kernel); rows that are not 16-byte aligned stay unsliced
    int slice = 0;
    if (vec == 4) {
        slice = opt.spmm_slice_cols > 0 ? opt.spmm_slice_cols : auto_slice_cols(F);
        if (slice >= F) slice = 0;
        ADAQP_REQUIRE(slice == 0 || (slice % 4 == 0 && slice <= 128), ADAQP_EINVAL,
                      "adaqp_spmm_csr_seg_f32: slice width %d is not a multiple of 4 in [4, 128]", slice);
    }
    // one row per grab (option spmm_rows_per_grab overrides): the narrowest window of rows in flight, so most
    // of the reused source rows stay in L2 (DESIGN §3: 1 row beat 2 by 4 % at F = 256 sliced, 3 % at F = 100)
    const int grab_rows = opt.spmm_rows_per_grab > 0 ? opt.spmm_rows_per_grab : 1;
    // the rows the launch computes: the list, or the whole range; the grid comes from them
    const int64_t work_rows = rows ? n_list : n_rows;
    if (slice > 0) {
        const int grab = grab_rows;
        const int64_t units = ((work_rows + grab - 1) / grab) * ((F + slice - 1) / slice);
        int64_t grid = (units + kWarps - 1) / kWarps;
        if (grid > cta_cap) grid = cta_cap;
        auto launch_sliced = [&](auto kernel) {
            kernel<<<(unsigned)grid, kThreads, 0, s>>>(indptr, indices, x0, ld0, n_split, x1, ld1, pre, post, mean, add_self,
                                                       row_begin, row_end, F, slice, out, ldo, counter, grab, seg_start, seg_end,
                                                       accumulate, hints, live, rows, n_list);
        };
        if (rows) launch_sliced(spmm_csr_sliced_kernel<false, true>);
        else if (live) launch_sliced(spmm_csr_sliced_kernel<true, false>);
        else launch_sliced(spmm_csr_sliced_kernel<false, false>);
        return adaqp_check_launch("spmm_csr_sliced_kernel");
    }
    int64_t grid = (work_rows + kWarps - 1) / kWarps;
    const int grab_now = grab_rows;
    if (grid > cta_cap) grid = cta_cap;
#define CALL_SPMM(V, C)                                                                                                  \
    do {                                                                                                                 \
        if (rows) spmm_csr_kernel<V, C, false, true><<<(unsigned)grid, kThreads, 0, s>>>(                                \
            indptr, indices, x0, ld0, n_split, x1, ld1, pre, post, mean, add_self, row_begin, row_end, F, out, ldo,      \
            counter, grab_now, seg_start, seg_end, accumulate, hints, nullptr, rows, n_list);                            \
        else if (live) spmm_csr_kernel<V, C, true, false><<<(unsigned)grid, kThreads, 0, s>>>(                           \
            indptr, indices, x0, ld0, n_split, x1, ld1, pre, post, mean, add_self, row_begin, row_end, F, out, ldo,      \
            counter, grab_now, seg_start, seg_end, accumulate, hints, live, nullptr, 0);                                 \
        else spmm_csr_kernel<V, C, false, false><<<(unsigned)grid, kThreads, 0, s>>>(                                    \
            indptr, indices, x0, ld0, n_split, x1, ld1, pre, post, mean, add_self, row_begin, row_end, F, out, ldo,      \
            counter, grab_now, seg_start, seg_end, accumulate, hints, nullptr, nullptr, 0);                              \
    } while (0)
    if (vec == 4) {
        if (nchunks <= 1) CALL_SPMM(4, 1);
        else if (nchunks <= 2) CALL_SPMM(4, 2);
        else if (nchunks <= 3) CALL_SPMM(4, 3);
        else if (nchunks <= 4) CALL_SPMM(4, 4);
        else if (nchunks <= 6) CALL_SPMM(4, 6);
        else CALL_SPMM(4, 8);
    } else if (vec == 2) {
        if (nchunks <= 2) CALL_SPMM(2, 2);
        else if (nchunks <= 4) CALL_SPMM(2, 4);
        else if (nchunks <= 6) CALL_SPMM(2, 6);
        else if (nchunks <= 10) CALL_SPMM(2, 10);
        else CALL_SPMM(2, 16);
    } else {
        if (nchunks <= 4) CALL_SPMM(1, 4);
        else if (nchunks <= 8) CALL_SPMM(1, 8);
        else if (nchunks <= 16) CALL_SPMM(1, 16);
        else CALL_SPMM(1, 32);
    }
#undef CALL_SPMM
    return adaqp_check_launch("spmm_csr_kernel");
}


int adaqp_spmm_csr_f32(const int64_t *indptr, const int32_t *indices, const float *x0, int64_t ld0,
                       int64_t n_split, const float *x1, int64_t ld1, const float *pre,
                       const float *post, int mean, int add_self, int64_t row_begin,
                       int64_t row_end, int32_t F, float *out, int64_t ldo, void *stream) {
    return adaqp_spmm_csr_seg_f32(indptr, nullptr, nullptr, indices, x0, ld0, n_split, x1, ld1, pre, post, mean,
                                  add_self, 0, row_begin, row_end, F, out, ldo, nullptr, nullptr, 0, stream);
}

int adaqp_row_live_f32(const float *x, int64_t ld, int64_t rows, int32_t F, uint8_t *live, void *stream) {
    ADAQP_REQUIRE(F > 0 && rows >= 0 && ld >= F, ADAQP_EINVAL, "adaqp_row_live_f32: bad shape rows=%lld F=%d ld=%lld",
                  (long long)rows, F, (long long)ld);
    if (rows == 0) return 0;
    ADAQP_REQUIRE(x && live, ADAQP_EINVAL, "adaqp_row_live_f32: null pointer");
    const int sms = adaqp_sm_count() > 0 ? adaqp_sm_count() : 132;
    int64_t grid = (rows + kWarps - 1) / kWarps;
    if (grid > (int64_t)sms * 8) grid = (int64_t)sms * 8;
    cudaStream_t s = (cudaStream_t)stream;
    if (F % 4 == 0 && ld % 4 == 0 && aligned(x, 4))
        row_live_kernel<4><<<(unsigned)grid, kThreads, 0, s>>>(x, ld, rows, F, live);
    else
        row_live_kernel<1><<<(unsigned)grid, kThreads, 0, s>>>(x, ld, rows, F, live);
    return adaqp_check_launch("row_live_kernel");
}

int adaqp_appnp_prop_f32(const int64_t *indptr, const int64_t *seg_start, const int64_t *seg_end,
                         const int32_t *indices, const float *x0, int64_t ld0, int64_t n_split, const float *x1,
                         int64_t ld1, const float *pre, const float *post, float scale, float alpha,
                         const float *tele, int64_t ldt, float *acc, int64_t lda, int32_t acc_mode, int accumulate,
                         int64_t row_begin, int64_t row_end, int32_t F, float *out, int64_t ldo, void *stream) {
    ADAQP_REQUIRE(F > 0 && F <= 1024, ADAQP_ELIMIT, "adaqp_appnp_prop_f32: F=%d outside (0,1024]", F);
    ADAQP_REQUIRE(row_end >= row_begin && row_begin >= 0 && row_end <= n_split, ADAQP_EINVAL,
                  "adaqp_appnp_prop_f32: bad row range [%lld, %lld) for n_split=%lld", (long long)row_begin,
                  (long long)row_end, (long long)n_split);
    ADAQP_REQUIRE(acc_mode >= 0 && acc_mode <= 7 && (acc_mode == 0 || (acc_mode & 1)), ADAQP_EINVAL,
                  "adaqp_appnp_prop_f32: bad acc_mode %d", acc_mode);
    ADAQP_REQUIRE(!(tele && acc_mode), ADAQP_EINVAL, "adaqp_appnp_prop_f32: tele and acc_mode are exclusive");
    if (row_end == row_begin) return 0;
    ADAQP_REQUIRE(indptr && indices && x0 && out, ADAQP_EINVAL, "adaqp_appnp_prop_f32: null pointer");
    const bool need_acc = (acc_mode & kAccRead) || (acc_mode && !(acc_mode & kAccFold));
    ADAQP_REQUIRE(!need_acc || acc, ADAQP_EINVAL, "adaqp_appnp_prop_f32: null acc for acc_mode %d", acc_mode);
    // halo rows arrive as the exchange leaves them ([num_remote, F] contiguous): 4-byte aligned for odd F
    int vec = 4;
    auto fits = [&](int v) {
        if (F % v || ld0 % v || ldo % v) return false;
        if (!aligned(x0, v) || !aligned(out, v)) return false;
        if (x1 && (!aligned(x1, v) || (ld1 % v))) return false;
        if (tele && (!aligned(tele, v) || (ldt % v))) return false;
        if (acc && (!aligned(acc, v) || (lda % v))) return false;
        return true;
    };
    while (vec > 1 && !fits(vec)) vec >>= 1;
    const int nchunks = (F + 32 * vec - 1) / (32 * vec);
    int dev = 0;
    ADAQP_CUDA(cudaGetDevice(&dev));
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long *counter = frontier_counter(dev, s);
    ADAQP_REQUIRE(counter != nullptr, ADAQP_EINVAL, "adaqp_appnp_prop_f32: row counter allocation failed");
    const bool fwd = tele != nullptr || acc_mode == 0;
    // column slices of 16-byte rows by the SpMM's rule (auto_slice_cols, or option spmm_slice_cols: >= F = unsliced)
    int slice = 0;
    if (vec == 4) {
        const AdaqpOptions &opt = adaqp_options();
        slice = opt.spmm_slice_cols > 0 ? opt.spmm_slice_cols : auto_slice_cols(F);
        if (slice >= F) slice = 0;
        ADAQP_REQUIRE(slice == 0 || (slice % 4 == 0 && slice <= 128), ADAQP_EINVAL,
                      "adaqp_appnp_prop_f32: slice width %d is not a multiple of 4 in [4, 128]", slice);
    }
    if (slice > 0) {
        const int64_t units = (row_end - row_begin) * ((F + slice - 1) / slice);
        const int64_t sgrid = adaqp_frontier_grid(units, kWarps);
        auto launch_sliced = [&](auto kernel) {
            kernel<<<(unsigned)sgrid, kThreads, 0, s>>>(indptr, indices, x0, ld0, n_split, x1, ld1, pre, post, scale,
                                                        alpha, tele, ldt, acc, lda, acc_mode, row_begin, row_end, F,
                                                        slice, out, ldo, counter, seg_start, seg_end, accumulate);
        };
        if (fwd) launch_sliced(appnp_prop_sliced_kernel<kEpiTeleport>);
        else launch_sliced(appnp_prop_sliced_kernel<kEpiAccum>);
        return adaqp_check_launch("appnp_prop_sliced_kernel");
    }
    const int64_t grid = adaqp_frontier_grid(row_end - row_begin, kWarps);
    auto launch = [&](auto kernel) {
        kernel<<<(unsigned)grid, kThreads, 0, s>>>(indptr, indices, x0, ld0, n_split, x1, ld1, pre, post, scale, alpha,
                                                   tele, ldt, acc, lda, acc_mode, row_begin, row_end, F, out, ldo,
                                                   counter, seg_start, seg_end, accumulate);
    };
#define APPNP_PICK(V, C)                                                                                    \
    do {                                                                                                    \
        if (fwd) launch(appnp_prop_kernel<V, C, kEpiTeleport>);                                             \
        else launch(appnp_prop_kernel<V, C, kEpiAccum>);                                                    \
    } while (0)
    // the narrowest instantiation that holds the row: C = 47 is <1, 2>, C = 100 <4, 1>, C = 107 <1, 4>
    if (vec == 4) {
        if (nchunks <= 1) APPNP_PICK(4, 1);
        else if (nchunks <= 2) APPNP_PICK(4, 2);
        else if (nchunks <= 4) APPNP_PICK(4, 4);
        else APPNP_PICK(4, 8);
    } else if (vec == 2) {
        if (nchunks <= 1) APPNP_PICK(2, 1);
        else if (nchunks <= 2) APPNP_PICK(2, 2);
        else if (nchunks <= 4) APPNP_PICK(2, 4);
        else if (nchunks <= 8) APPNP_PICK(2, 8);
        else APPNP_PICK(2, 16);
    } else {
        if (nchunks <= 1) APPNP_PICK(1, 1);
        else if (nchunks <= 2) APPNP_PICK(1, 2);
        else if (nchunks <= 4) APPNP_PICK(1, 4);
        else if (nchunks <= 8) APPNP_PICK(1, 8);
        else if (nchunks <= 16) APPNP_PICK(1, 16);
        else APPNP_PICK(1, 32);
    }
#undef APPNP_PICK
    return adaqp_check_launch("appnp_prop_kernel");
}

int adaqp_cs_prop_f32(const int64_t *indptr, const int32_t *indices, const float *x0, int64_t ld0, int64_t n_split,
                      const float *x1, int64_t ld1, const float *pre, const float *post, float scale, float alpha,
                      const float *tele, int64_t ldt, const int32_t *y, const float *fix, int64_t ldf,
                      int32_t post_mode, float lo, float hi, int64_t row_begin, int64_t row_end, int32_t F,
                      float *out, int64_t ldo, void *stream) {
    ADAQP_REQUIRE(F > 0 && F <= 1024, ADAQP_EINVAL, "adaqp_cs_prop_f32: C=%d outside [1, 1024]", F);
    ADAQP_REQUIRE(row_end >= row_begin && row_begin >= 0 && row_end <= n_split, ADAQP_EINVAL,
                  "adaqp_cs_prop_f32: bad row range [%lld, %lld) for n_split=%lld", (long long)row_begin,
                  (long long)row_end, (long long)n_split);
    ADAQP_REQUIRE(post_mode == kCsClamp || post_mode == kCsFix, ADAQP_EINVAL, "adaqp_cs_prop_f32: bad post_mode %d",
                  post_mode);
    ADAQP_REQUIRE(post_mode != kCsClamp || lo <= hi, ADAQP_EINVAL, "adaqp_cs_prop_f32: clamp bounds lo=%g > hi=%g",
                  (double)lo, (double)hi);
    if (row_end == row_begin) return 0;
    ADAQP_REQUIRE(indptr && indices && x0 && out, ADAQP_EINVAL, "adaqp_cs_prop_f32: null pointer");
    ADAQP_REQUIRE(post_mode != kCsFix || (y && fix), ADAQP_EINVAL, "adaqp_cs_prop_f32: null pointer (y / fix)");
    if (post_mode == kCsFix) tele = nullptr;
    int vec = 4;
    auto fits = [&](int v) {
        if (F % v || ld0 % v || ldo % v) return false;
        if (!aligned(x0, v) || !aligned(out, v)) return false;
        if (x1 && (!aligned(x1, v) || (ld1 % v))) return false;
        if (tele && (!aligned(tele, v) || (ldt % v))) return false;
        if (fix && (!aligned(fix, v) || (ldf % v))) return false;
        return true;
    };
    while (vec > 1 && !fits(vec)) vec >>= 1;
    const int nchunks = (F + 32 * vec - 1) / (32 * vec);
    int dev = 0;
    ADAQP_CUDA(cudaGetDevice(&dev));
    cudaStream_t s = (cudaStream_t)stream;
    unsigned long long *counter = frontier_counter(dev, s);
    ADAQP_REQUIRE(counter != nullptr, ADAQP_EINVAL, "adaqp_cs_prop_f32: row counter allocation failed");
    const int64_t grid = adaqp_frontier_grid(row_end - row_begin, kWarps);
    auto launch = [&](auto kernel) {
        kernel<<<(unsigned)grid, kThreads, 0, s>>>(indptr, indices, x0, ld0, n_split, x1, ld1, pre, post, scale, alpha,
                                                   tele, ldt, y, fix, ldf, lo, hi, row_begin, row_end, F, out, ldo,
                                                   counter);
    };
#define CS_PICK(V, C)                                                                                       \
    do {                                                                                                    \
        if (post_mode == kCsClamp) launch(cs_prop_kernel<V, C, kCsClamp>);                                  \
        else launch(cs_prop_kernel<V, C, kCsFix>);                                                          \
    } while (0)
    // the ladder of appnp_prop_kernel: the narrowest instantiation that holds the row
    if (vec == 4) {
        if (nchunks <= 1) CS_PICK(4, 1);
        else if (nchunks <= 2) CS_PICK(4, 2);
        else if (nchunks <= 4) CS_PICK(4, 4);
        else CS_PICK(4, 8);
    } else if (vec == 2) {
        if (nchunks <= 1) CS_PICK(2, 1);
        else if (nchunks <= 2) CS_PICK(2, 2);
        else if (nchunks <= 4) CS_PICK(2, 4);
        else if (nchunks <= 8) CS_PICK(2, 8);
        else CS_PICK(2, 16);
    } else {
        if (nchunks <= 1) CS_PICK(1, 1);
        else if (nchunks <= 2) CS_PICK(1, 2);
        else if (nchunks <= 4) CS_PICK(1, 4);
        else if (nchunks <= 8) CS_PICK(1, 8);
        else if (nchunks <= 16) CS_PICK(1, 16);
        else CS_PICK(1, 32);
    }
#undef CS_PICK
    return adaqp_check_launch("cs_prop_kernel");
}

}  // extern "C"

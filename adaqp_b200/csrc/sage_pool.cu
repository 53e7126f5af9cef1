// GraphSAGE max-pool aggregation over the halo exchange (sm_90a).
//
// DGL's SAGEConv(aggregator_type='pool'): the pooled rows p = relu(x W_pool^T + b_pool) come from the dense GEMM;
// this file owns the neighbourhood max and its gradient:
//   m[v,c]   = max_{u in N_in(v)} p[u,c]        (CSR row v, self-loop included)
//   arg[v,c] = the first u in CSR order that attains it (strict '>' while scanning)
//   dp[u,c]  = sum_{v : u in N_in(v)} gm[v,c] [arg[v,c] = u]        (gm = dL/dm)
// The graphs are symmetric, so the destinations of an inner row u are exactly the entries of its CSR row: dp[u] is
// a pull over row u (one warp, sums in CSR order, no atomics).
//
// Sources split as in spmm.cu: ids < n_split are local rows, ids >= n_split halo rows.  arg is stored as
// (source id - n_split): a halo position (>= 0) for halo sources, a negative value for local ones, kNoArg for a row
// without sources.  That is the encoding the rows travel in, so the owner of a destination can send its arg rows
// as they are; the backward pass then compares arg[x,c] with want[e], the precomputed encoding of row u as seen by
// the owner of x (adaqp_b200/sage_pool.py, pool_want).
//
// seg_start / seg_end (optional, per row) restrict a launch to part of each CSR row -- the local-source segment
// [indptr[v], halo_split[v]) or the halo-source segment [halo_split[v], indptr[v+1]) -- and `accumulate` continues
// from what a previous launch wrote (forward: running max and arg; backward: the fp32 sum).  Local sources come
// first in every row (columns are sorted, halo ids >= n_split), so the two-pass form visits the sources in the
// same order as one pass and gives bitwise equal results.
//
// One warp per row from the frontier row scheduler; lane l owns columns c * 32 + l (c < CHUNKS), so a row gather
// is CHUNKS coalesced 128-byte loads.  fp32, no float atomics: repeated launches are bitwise equal.
#include <math.h>

#include "common.cuh"

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int32_t kNoArg = INT32_MIN;

// neighbour rows gathered per step: more for narrow rows, where one row is few loads
template <int CHUNKS>
struct Unroll {
    static constexpr int value = CHUNKS <= 4 ? 4 : CHUNKS <= 8 ? 2 : 1;
};

template <int CHUNKS>
__global__ void __launch_bounds__(kThreads)
sage_pool_fwd_kernel(const int64_t *__restrict__ indptr, const int64_t *__restrict__ seg_start,
                     const int64_t *__restrict__ seg_end, const int32_t *__restrict__ indices, int64_t n_split,
                     const float *__restrict__ x0, int64_t ld0, const float *__restrict__ x1, int64_t ld1, int F,
                     int64_t row_begin, int64_t row_end, int accumulate, float *__restrict__ out, int64_t ldo,
                     int32_t *__restrict__ arg, int64_t lda, unsigned long long *__restrict__ next_row) {
    constexpr int U = Unroll<CHUNKS>::value;
    const int lane = threadIdx.x & 31;
    bool ok[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) ok[c] = c * 32 + lane < F;
    const int64_t n_rows = row_end - row_begin;
    while (true) {
        unsigned long long grab = 0;
        if (lane == 0) grab = atomicAdd(next_row, 1ull);
        grab = __shfl_sync(ADAQP_FULL_MASK, grab, 0);
        if ((int64_t)grab >= n_rows) break;
        const int64_t row = row_begin + (int64_t)grab;
        float *orow = out + (int64_t)grab * ldo;
        int32_t *arow = arg + (int64_t)grab * lda;
        float m[CHUNKS];
        int32_t a[CHUNKS];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            m[c] = -INFINITY;
            a[c] = kNoArg;
            if (accumulate && ok[c]) {
                a[c] = arow[c * 32 + lane];
                if (a[c] != kNoArg) m[c] = orow[c * 32 + lane];
            }
        }
        const int64_t b = seg_start ? __ldg(seg_start + row) : __ldg(indptr + row);
        const int64_t e = seg_end ? __ldg(seg_end + row) : __ldg(indptr + row + 1);
        for (int64_t j0 = b; j0 < e; j0 += 32) {
            const int n = (e - j0) < 32 ? (int)(e - j0) : 32;
            int u = 0;
            if (lane < n) u = __ldg(indices + j0 + lane);
            for (int k = 0; k < n; k += U) {
                float v[U][CHUNKS];
                int32_t enc[U];
#pragma unroll
                for (int t = 0; t < U; ++t) {
                    const int uu = __shfl_sync(ADAQP_FULL_MASK, u, (k + t) & 31);
                    const bool live = (k + t) < n;
                    const bool local = uu < n_split;
                    const float *r = local ? x0 + (int64_t)uu * ld0 : x1 + ((int64_t)uu - n_split) * ld1;
                    enc[t] = (int32_t)((int64_t)uu - n_split);
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c) v[t][c] = (live && ok[c]) ? __ldg(r + c * 32 + lane) : -INFINITY;
                }
#pragma unroll
                for (int t = 0; t < U; ++t) {
                    if (k + t >= n) break;                      // warp-uniform
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c) {
                        if (v[t][c] > m[c]) {
                            m[c] = v[t][c];
                            a[c] = enc[t];
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            if (!ok[c]) continue;
            orow[c * 32 + lane] = a[c] == kNoArg ? 0.f : m[c];       // DGL: 0 for a row without sources
            arow[c * 32 + lane] = a[c];
        }
    }
    frontier_release(next_row);
}

// One warp per local row u; entry e = (u, x) of its CSR row routes gm[x,c] to u where arg[x,c] == want[e].
// The arg row is read first and the gradient column only where it matches (about 1 / deg(x) of the columns).
template <int CHUNKS>
__global__ void __launch_bounds__(kThreads)
sage_pool_bwd_kernel(const int64_t *__restrict__ indptr, const int64_t *__restrict__ seg_start,
                     const int64_t *__restrict__ seg_end, const int32_t *__restrict__ indices,
                     const int32_t *__restrict__ want, int64_t n_split, const float *__restrict__ g0, int64_t ldg0,
                     const float *__restrict__ g1, int64_t ldg1, const int32_t *__restrict__ a0, int64_t lda0,
                     const int32_t *__restrict__ a1, int64_t lda1, int F, int64_t row_begin, int64_t row_end,
                     int accumulate, float *__restrict__ dp, int64_t ldd, unsigned long long *__restrict__ next_row) {
    constexpr int U = Unroll<CHUNKS>::value;
    const int lane = threadIdx.x & 31;
    bool ok[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) ok[c] = c * 32 + lane < F;
    const int64_t n_rows = row_end - row_begin;
    while (true) {
        unsigned long long grab = 0;
        if (lane == 0) grab = atomicAdd(next_row, 1ull);
        grab = __shfl_sync(ADAQP_FULL_MASK, grab, 0);
        if ((int64_t)grab >= n_rows) break;
        const int64_t row = row_begin + (int64_t)grab;
        float *drow = dp + (int64_t)grab * ldd;
        float acc[CHUNKS];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) acc[c] = (accumulate && ok[c]) ? drow[c * 32 + lane] : 0.f;
        const int64_t b = seg_start ? __ldg(seg_start + row) : __ldg(indptr + row);
        const int64_t e = seg_end ? __ldg(seg_end + row) : __ldg(indptr + row + 1);
        for (int64_t j0 = b; j0 < e; j0 += 32) {
            const int n = (e - j0) < 32 ? (int)(e - j0) : 32;
            int xi = 0;
            int32_t wi = 0;
            if (lane < n) {
                xi = __ldg(indices + j0 + lane);
                wi = __ldg(want + j0 + lane);
            }
            for (int k = 0; k < n; k += U) {
                bool hit[U][CHUNKS];
                const float *gr[U];
#pragma unroll
                for (int t = 0; t < U; ++t) {
                    const int x = __shfl_sync(ADAQP_FULL_MASK, xi, (k + t) & 31);
                    const int32_t w = __shfl_sync(ADAQP_FULL_MASK, wi, (k + t) & 31);
                    const bool live = (k + t) < n;
                    const bool local = x < n_split;
                    const int64_t xr = local ? (int64_t)x : (int64_t)x - n_split;
                    const int32_t *ar = local ? a0 + xr * lda0 : a1 + xr * lda1;
                    gr[t] = local ? g0 + xr * ldg0 : g1 + xr * ldg1;
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c) hit[t][c] = live && ok[c] && __ldg(ar + c * 32 + lane) == w;
                }
#pragma unroll
                for (int t = 0; t < U; ++t) {
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c)
                        if (hit[t][c]) acc[c] = __fadd_rn(acc[c], __ldg(gr[t] + c * 32 + lane));
                }
            }
        }
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c)
            if (ok[c]) drow[c * 32 + lane] = acc[c];
    }
    frontier_release(next_row);
}

int pool_chunks(int F) {
    const int c = (F + 31) / 32;
    return c <= 1 ? 1 : c <= 2 ? 2 : c <= 4 ? 4 : c <= 8 ? 8 : c <= 12 ? 12 : c <= 16 ? 16 : c <= 24 ? 24 : 32;
}

}  // namespace

extern "C" {

int adaqp_sage_pool_fwd_f32(const int64_t *indptr, const int64_t *seg_start, const int64_t *seg_end,
                            const int32_t *indices, int64_t n_split, const float *x0, int64_t ld0, const float *x1,
                            int64_t ld1, int32_t F, int64_t row_begin, int64_t row_end, int accumulate, float *out,
                            int64_t ldo, int32_t *arg, int64_t lda, void *stream) {
    ADAQP_REQUIRE(F > 0 && F <= 1024, ADAQP_ELIMIT, "adaqp_sage_pool_fwd_f32: F=%d outside (0,1024]", F);
    ADAQP_REQUIRE(row_end >= row_begin && row_begin >= 0, ADAQP_EINVAL, "adaqp_sage_pool_fwd_f32: bad row range");
    ADAQP_REQUIRE(n_split >= 0, ADAQP_EINVAL, "adaqp_sage_pool_fwd_f32: n_split=%lld", (long long)n_split);
    ADAQP_REQUIRE(ld0 >= F && ldo >= F && lda >= F && (!x1 || ld1 >= F), ADAQP_EINVAL,
                  "adaqp_sage_pool_fwd_f32: row pitch < F");
    if (row_end == row_begin) return 0;
    ADAQP_REQUIRE(indptr && indices && x0 && out && arg, ADAQP_EINVAL, "adaqp_sage_pool_fwd_f32: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    int dev = 0;
    ADAQP_CUDA(cudaGetDevice(&dev));
    unsigned long long *counter = adaqp_frontier_counter(dev, s);
    ADAQP_REQUIRE(counter != nullptr, ADAQP_EINVAL, "adaqp_sage_pool_fwd_f32: row counter allocation failed");
    const int64_t grid = adaqp_frontier_grid(row_end - row_begin, kWarps);
#define CALL_FWD(C)                                                                                                 \
    sage_pool_fwd_kernel<C><<<(unsigned)grid, kThreads, 0, s>>>(indptr, seg_start, seg_end, indices, n_split, x0, ld0, \
                                                                x1, ld1, F, row_begin, row_end, accumulate, out, ldo, \
                                                                arg, lda, counter)
    switch (pool_chunks(F)) {
        case 1: CALL_FWD(1); break;
        case 2: CALL_FWD(2); break;
        case 4: CALL_FWD(4); break;
        case 8: CALL_FWD(8); break;
        case 12: CALL_FWD(12); break;
        case 16: CALL_FWD(16); break;
        case 24: CALL_FWD(24); break;
        default: CALL_FWD(32); break;
    }
#undef CALL_FWD
    return adaqp_check_launch("sage_pool_fwd_kernel");
}

int adaqp_sage_pool_bwd_f32(const int64_t *indptr, const int64_t *seg_start, const int64_t *seg_end,
                            const int32_t *indices, const int32_t *want, int64_t n_split, const float *g0,
                            int64_t ldg0, const float *g1, int64_t ldg1, const int32_t *a0, int64_t lda0,
                            const int32_t *a1, int64_t lda1, int32_t F, int64_t row_begin, int64_t row_end,
                            int accumulate, float *dp, int64_t ldd, void *stream) {
    ADAQP_REQUIRE(F > 0 && F <= 1024, ADAQP_ELIMIT, "adaqp_sage_pool_bwd_f32: F=%d outside (0,1024]", F);
    ADAQP_REQUIRE(row_end >= row_begin && row_begin >= 0, ADAQP_EINVAL, "adaqp_sage_pool_bwd_f32: bad row range");
    ADAQP_REQUIRE(row_end <= n_split, ADAQP_EINVAL,
                  "adaqp_sage_pool_bwd_f32: rows must be local (row_end %lld > n_split %lld)", (long long)row_end,
                  (long long)n_split);
    ADAQP_REQUIRE(ldg0 >= F && lda0 >= F && ldd >= F && (!g1 || ldg1 >= F) && (!a1 || lda1 >= F), ADAQP_EINVAL,
                  "adaqp_sage_pool_bwd_f32: row pitch < F");
    if (row_end == row_begin) return 0;
    ADAQP_REQUIRE(indptr && indices && want && g0 && a0 && dp, ADAQP_EINVAL, "adaqp_sage_pool_bwd_f32: null pointer");
    ADAQP_REQUIRE((g1 == nullptr) == (a1 == nullptr), ADAQP_EINVAL,
                  "adaqp_sage_pool_bwd_f32: halo g1 and a1 must be given together");
    cudaStream_t s = (cudaStream_t)stream;
    int dev = 0;
    ADAQP_CUDA(cudaGetDevice(&dev));
    unsigned long long *counter = adaqp_frontier_counter(dev, s);
    ADAQP_REQUIRE(counter != nullptr, ADAQP_EINVAL, "adaqp_sage_pool_bwd_f32: row counter allocation failed");
    const int64_t grid = adaqp_frontier_grid(row_end - row_begin, kWarps);
#define CALL_BWD(C)                                                                                                 \
    sage_pool_bwd_kernel<C><<<(unsigned)grid, kThreads, 0, s>>>(indptr, seg_start, seg_end, indices, want, n_split, \
                                                                g0, ldg0, g1, ldg1, a0, lda0, a1, lda1, F, row_begin, \
                                                                row_end, accumulate, dp, ldd, counter)
    switch (pool_chunks(F)) {
        case 1: CALL_BWD(1); break;
        case 2: CALL_BWD(2); break;
        case 4: CALL_BWD(4); break;
        case 8: CALL_BWD(8); break;
        case 12: CALL_BWD(12); break;
        case 16: CALL_BWD(16); break;
        case 24: CALL_BWD(24); break;
        default: CALL_BWD(32); break;
    }
#undef CALL_BWD
    return adaqp_check_launch("sage_pool_bwd_kernel");
}

}  // extern "C"

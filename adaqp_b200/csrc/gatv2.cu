// GATv2 attention aggregation over the halo exchange (sm_90a).
//
// DGL's GATv2Conv with share_weights=False: zs = x W_s + b_s, zd = x W_d + b_d (the dense GEMM), H heads of width D,
// F = H * D columns per row, negative slope 0.2:
//   e[v,u,h] = sum_{c in head h} a[h,c] LeakyReLU(zs[u,h,c] + zd[v,h,c])     u in N_in(v) (CSR row v, self-loop)
//   lse[v,h] = logsumexp_u e[v,u,h]          alpha[v,u,h] = exp(e[v,u,h] - lse[v,h])
//   out[v,h,:] = sum_u alpha[v,u,h] zs[u,h,:]
// Backward, with g = dL/dout and S[v,h] = <g[v,h,:], out[v,h,:]>, for every edge u -> v:
//   t[v,u,h] = alpha[v,u,h] (<g[v,h,:], zs[u,h,:]> - S[v,h])
//   dzs[u]  += alpha[v,u] g[v] + t[v,u] a . LeakyReLU'(zs[u] + zd[v])      (the source side of the edge)
//   dzd[v]  += t[v,u] a . LeakyReLU'(zs[u] + zd[v])                         (the destination side)
//   da      += t[v,u] LeakyReLU(zs[u] + zd[v])
// The logit does not split into per-row scalars, so only the rank of v can evaluate an edge u -> v.  For a halo
// source u that rank computes the source-side term against the received copy of zs[u] (gatv2_bwd_halo_kernel) and
// pushes the row back to u's owner, which folds the pushed rows into dzs[u] (gatv2_bwd_inner_kernel's epilogue).
// The graph is symmetric, so one pass over the CSR row of an inner row u serves u as a destination (every entry)
// and as a source (its local entries).
//
// Sources split as in spmm.cu: ids < n_split are local rows, ids >= n_split halo rows.  Launches take a row range.
// Column layout and per-head reductions as in gat.cu (attn.cuh).  fp32 throughout, no atomics on data: every row
// is reduced by one warp in CSR order and the pushed rows are folded in a fixed order, so repeated launches are
// bitwise equal.
#include <math.h>

#include "attn.cuh"

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kUnroll = 4;
constexpr float kSlope = 0.2f;

__device__ __forceinline__ float leaky(float x) { return x > 0.f ? x : kSlope * x; }

template <int CHUNKS>
__device__ __forceinline__ void load_row(float (&v)[CHUNKS], const float *r, const Cols<CHUNKS> &cols, int lane) {
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) v[c] = cols.ok[c] ? __ldg(r + c * 32 + lane) : 0.f;
}

// One warp per destination row, rows from the frontier counter.  zd[v] is loaded once; for each source the per-head
// logit sum_c a LeakyReLU(zs[u] + zd[v]) feeds the single-pass online softmax of gat_fwd_kernel, so every source row
// is gathered once and any in-degree is exact.
template <int CHUNKS>
__global__ void __launch_bounds__(kThreads)
gatv2_fwd_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices, int64_t n_split,
                 const float *__restrict__ zs0, int64_t ldzs0, const float *__restrict__ zs1, int64_t ldzs1,
                 const float *__restrict__ zd, int64_t ldzd, const float *__restrict__ attn, int H, int F, int mode,
                 int D, int cpg, int64_t row_begin, int64_t row_end, float *__restrict__ out, int64_t ldo,
                 float *__restrict__ lse, unsigned long long *__restrict__ next_row) {
    const int lane = threadIdx.x & 31;
    const Cols<CHUNKS> cols(lane, F, D);
    float a[CHUNKS];
    load_row(a, attn, cols, lane);
    const int64_t n_rows = row_end - row_begin;
    while (true) {
        unsigned long long grab = 0;
        if (lane == 0) grab = atomicAdd(next_row, 1ull);
        grab = __shfl_sync(ADAQP_FULL_MASK, grab, 0);
        if ((int64_t)grab >= n_rows) break;
        const int64_t row = row_begin + (int64_t)grab;
        float zdv[CHUNKS], m[CHUNKS], ssum[CHUNKS], acc[CHUNKS];
        load_row(zdv, zd + row * ldzd, cols, lane);
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            m[c] = -INFINITY;
            ssum[c] = 0.f;
            acc[c] = 0.f;
        }
        const int64_t b = __ldg(indptr + row), e = __ldg(indptr + row + 1);
        for (int64_t j0 = b; j0 < e; j0 += 32) {
            const int n = (e - j0) < 32 ? (int)(e - j0) : 32;
            int u = 0;
            if (lane < n) u = __ldg(indices + j0 + lane);
            for (int k = 0; k < n; k += kUnroll) {
                float v[kUnroll][CHUNKS];
#pragma unroll
                for (int t = 0; t < kUnroll; ++t) {
                    const int uu = __shfl_sync(ADAQP_FULL_MASK, u, (k + t) & 31);
                    const bool live = (k + t) < n;
                    const bool local = uu < n_split;
                    const float *zr = local ? zs0 + (int64_t)uu * ldzs0 : zs1 + ((int64_t)uu - n_split) * ldzs1;
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c) v[t][c] = (live && cols.ok[c]) ? __ldg(zr + c * 32 + lane) : 0.f;
                }
#pragma unroll
                for (int t = 0; t < kUnroll; ++t) {
                    if (k + t >= n) break;                   // warp-uniform
                    float p[CHUNKS];
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c) p[c] = __fmul_rn(a[c], leaky(__fadd_rn(v[t][c], zdv[c])));
                    head_reduce<CHUNKS>(p, mode, D, cpg);
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c) {
                        if (!cols.ok[c]) continue;
                        const float x = p[c];
                        if (x > m[c]) {
                            const float r = expf(m[c] - x);     // exp(-inf) = 0 on the first neighbour
                            ssum[c] = __fmaf_rn(ssum[c], r, 1.f);
                            acc[c] = __fmaf_rn(acc[c], r, v[t][c]);
                            m[c] = x;
                        } else {
                            const float q = expf(x - m[c]);
                            ssum[c] = __fadd_rn(ssum[c], q);
                            acc[c] = __fmaf_rn(q, v[t][c], acc[c]);
                        }
                    }
                }
            }
        }
        float *orow = out + (row - row_begin) * ldo;
        float *lrow = lse + (row - row_begin) * H;
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            if (!cols.ok[c]) continue;
            orow[c * 32 + lane] = ssum[c] > 0.f ? __fdiv_rn(acc[c], ssum[c]) : 0.f;
            if (cols.lead[c]) lrow[cols.hid[c]] = ssum[c] > 0.f ? __fadd_rn(m[c], logf(ssum[c])) : -INFINITY;
        }
    }
    frontier_release(next_row);
}

// Source side of the edge u -> x (x a local destination): acc += alpha[x,u] g[x] + t[x,u] a . LeakyReLU'(zs[u] + zd[x]).
// Shared by the inner rows (u local) and the halo rows (u the received copy of a remote row).
template <int CHUNKS>
__device__ __forceinline__ void source_term(const float (&zsu)[CHUNKS], const float (&a)[CHUNKS], const float *zdr,
                                            const float *gr, const float *lser, const float *sr,
                                            const Cols<CHUNKS> &cols, int lane, int mode, int D, int cpg,
                                            float (&acc)[CHUNKS]) {
    float gx[CHUNKS], s[CHUNKS], p[CHUNKS], q[CHUNKS], lx[CHUNKS], sx[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
        const bool ok = cols.ok[c];
        const int h = cols.hid[c];
        gx[c] = ok ? __ldg(gr + c * 32 + lane) : 0.f;
        const float zdx = ok ? __ldg(zdr + c * 32 + lane) : 0.f;
        lx[c] = ok ? __ldg(lser + h) : 0.f;
        sx[c] = ok ? __ldg(sr + h) : 0.f;
        s[c] = __fadd_rn(zsu[c], zdx);
        p[c] = __fmul_rn(a[c], leaky(s[c]));
        q[c] = __fmul_rn(gx[c], zsu[c]);
    }
    head_reduce<CHUNKS>(p, mode, D, cpg);
    head_reduce<CHUNKS>(q, mode, D, cpg);
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
        if (!cols.ok[c]) continue;
        const float al = expf(__fsub_rn(p[c], lx[c]));
        const float t = __fmul_rn(al, __fsub_rn(q[c], sx[c]));
        acc[c] = __fmaf_rn(al, gx[c], acc[c]);
        acc[c] = __fmaf_rn(__fmul_rn(t, a[c]), s[c] > 0.f ? 1.f : kSlope, acc[c]);
    }
}

// One warp per inner row u.  Entry x of the CSR row of u is a source of u (every x, local or halo: dzd[u] and the
// row's share of da) and, when local, a destination of u (dzs[u]).  The epilogue adds the rows pushed back for u by
// the peers holding u as a halo row, at push rows fold_pos[fold_indptr[u] .. fold_indptr[u+1]) in that order.
template <int CHUNKS>
__global__ void __launch_bounds__(kThreads)
gatv2_bwd_inner_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices, int64_t n_split,
                       const float *__restrict__ zs0, int64_t ldzs0, const float *__restrict__ zs1, int64_t ldzs1,
                       const float *__restrict__ zd, int64_t ldzd, const float *__restrict__ g, int64_t ldg,
                       const float *__restrict__ lse, const float *__restrict__ S, const float *__restrict__ attn,
                       const float *__restrict__ push, int64_t ldp, const int64_t *__restrict__ fold_indptr,
                       const int32_t *__restrict__ fold_pos, int H, int F, int mode, int D, int cpg,
                       int64_t row_begin, int64_t row_end, float *__restrict__ dzs, int64_t lddzs,
                       float *__restrict__ dzd, int64_t lddzd, float *__restrict__ da, int64_t ldda,
                       unsigned long long *__restrict__ next_row) {
    const int lane = threadIdx.x & 31;
    const Cols<CHUNKS> cols(lane, F, D);
    float a[CHUNKS];
    load_row(a, attn, cols, lane);
    const int64_t n_rows = row_end - row_begin;
    while (true) {
        unsigned long long grab = 0;
        if (lane == 0) grab = atomicAdd(next_row, 1ull);
        grab = __shfl_sync(ADAQP_FULL_MASK, grab, 0);
        if ((int64_t)grab >= n_rows) break;
        const int64_t u = row_begin + (int64_t)grab;
        float zsu[CHUNKS], zdu[CHUNKS], gu[CHUNKS], lseu[CHUNKS], su[CHUNKS];
        float acc_s[CHUNKS], acc_d[CHUNKS], acc_a[CHUNKS];
        load_row(zsu, zs0 + u * ldzs0, cols, lane);
        load_row(zdu, zd + u * ldzd, cols, lane);
        load_row(gu, g + u * ldg, cols, lane);
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            lseu[c] = cols.ok[c] ? __ldg(lse + u * H + cols.hid[c]) : 0.f;
            su[c] = cols.ok[c] ? __ldg(S + u * H + cols.hid[c]) : 0.f;
            acc_s[c] = acc_d[c] = acc_a[c] = 0.f;
        }
        const int64_t b = __ldg(indptr + u), e = __ldg(indptr + u + 1);
        for (int64_t j0 = b; j0 < e; j0 += 32) {
            const int n = (e - j0) < 32 ? (int)(e - j0) : 32;
            int xi = 0;
            if (lane < n) xi = __ldg(indices + j0 + lane);
            for (int k = 0; k < n; ++k) {
                const int x = __shfl_sync(ADAQP_FULL_MASK, xi, k);
                const bool local = x < n_split;                         // warp-uniform
                const int64_t xr = local ? (int64_t)x : (int64_t)x - n_split;
                float zsx[CHUNKS], s[CHUNKS], lk[CHUNKS], p[CHUNKS], q[CHUNKS];
                load_row(zsx, local ? zs0 + xr * ldzs0 : zs1 + xr * ldzs1, cols, lane);
#pragma unroll
                for (int c = 0; c < CHUNKS; ++c) {
                    s[c] = __fadd_rn(zsx[c], zdu[c]);
                    lk[c] = leaky(s[c]);
                    p[c] = __fmul_rn(a[c], lk[c]);
                    q[c] = __fmul_rn(gu[c], zsx[c]);
                }
                head_reduce<CHUNKS>(p, mode, D, cpg);
                head_reduce<CHUNKS>(q, mode, D, cpg);
#pragma unroll
                for (int c = 0; c < CHUNKS; ++c) {
                    if (!cols.ok[c]) continue;
                    const float al = expf(__fsub_rn(p[c], lseu[c]));
                    const float t = __fmul_rn(al, __fsub_rn(q[c], su[c]));
                    acc_d[c] = __fmaf_rn(__fmul_rn(t, a[c]), s[c] > 0.f ? 1.f : kSlope, acc_d[c]);
                    acc_a[c] = __fmaf_rn(t, lk[c], acc_a[c]);
                }
                if (local)
                    source_term<CHUNKS>(zsu, a, zd + xr * ldzd, g + xr * ldg, lse + xr * H, S + xr * H, cols, lane,
                                        mode, D, cpg, acc_s);
            }
        }
        if (push != nullptr) {
            const int64_t fb = __ldg(fold_indptr + u), fe = __ldg(fold_indptr + u + 1);
            for (int64_t k = fb; k < fe; ++k) {
                const float *pr = push + (int64_t)__ldg(fold_pos + k) * ldp;
#pragma unroll
                for (int c = 0; c < CHUNKS; ++c)
                    if (cols.ok[c]) acc_s[c] = __fadd_rn(acc_s[c], __ldg(pr + c * 32 + lane));
            }
        }
        const int64_t o = u - row_begin;
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            if (!cols.ok[c]) continue;
            const int col = c * 32 + lane;
            dzs[o * lddzs + col] = acc_s[c];
            dzd[o * lddzd + col] = acc_d[c];
            da[o * ldda + col] = acc_a[c];
        }
    }
    frontier_release(next_row);
}

// One warp per halo row h: the source-side gradient of the received copy zs1[h] over its inner destinations
// halo_dst[halo_indptr[h] .. halo_indptr[h+1]), which the holder pushes back to the row's owner.
template <int CHUNKS>
__global__ void __launch_bounds__(kThreads)
gatv2_bwd_halo_kernel(const int64_t *__restrict__ halo_indptr, const int32_t *__restrict__ halo_dst,
                      const float *__restrict__ zs1, int64_t ldzs1, const float *__restrict__ zd, int64_t ldzd,
                      const float *__restrict__ g, int64_t ldg, const float *__restrict__ lse,
                      const float *__restrict__ S, const float *__restrict__ attn, int H, int F, int mode, int D,
                      int cpg, int64_t row_begin, int64_t row_end, float *__restrict__ out, int64_t ldo,
                      unsigned long long *__restrict__ next_row) {
    const int lane = threadIdx.x & 31;
    const Cols<CHUNKS> cols(lane, F, D);
    float a[CHUNKS];
    load_row(a, attn, cols, lane);
    const int64_t n_rows = row_end - row_begin;
    while (true) {
        unsigned long long grab = 0;
        if (lane == 0) grab = atomicAdd(next_row, 1ull);
        grab = __shfl_sync(ADAQP_FULL_MASK, grab, 0);
        if ((int64_t)grab >= n_rows) break;
        const int64_t h = row_begin + (int64_t)grab;
        float zsu[CHUNKS], acc[CHUNKS];
        load_row(zsu, zs1 + h * ldzs1, cols, lane);
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) acc[c] = 0.f;
        const int64_t b = __ldg(halo_indptr + h), e = __ldg(halo_indptr + h + 1);
        for (int64_t j0 = b; j0 < e; j0 += 32) {
            const int n = (e - j0) < 32 ? (int)(e - j0) : 32;
            int vi = 0;
            if (lane < n) vi = __ldg(halo_dst + j0 + lane);
            for (int k = 0; k < n; ++k) {
                const int64_t v = __shfl_sync(ADAQP_FULL_MASK, vi, k);
                source_term<CHUNKS>(zsu, a, zd + v * ldzd, g + v * ldg, lse + v * H, S + v * H, cols, lane, mode, D,
                                    cpg, acc);
            }
        }
        float *orow = out + (h - row_begin) * ldo;
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c)
            if (cols.ok[c]) orow[c * 32 + lane] = acc[c];
    }
    frontier_release(next_row);
}

int64_t frontier_grid(int64_t rows) { return adaqp_frontier_grid(rows, kWarps); }

}  // namespace

extern "C" {

int adaqp_gatv2_fwd_f32(const int64_t *indptr, const int32_t *indices, int64_t n_split, const float *zs0,
                        int64_t ldzs0, const float *zs1, int64_t ldzs1, const float *zd, int64_t ldzd,
                        const float *attn, int32_t H, int32_t F, int64_t row_begin, int64_t row_end, float *out,
                        int64_t ldo, float *lse, void *stream) {
    int mode, D, cpg, chunks;
    int rc = head_layout("adaqp_gatv2_fwd_f32", H, F, &mode, &D, &cpg, &chunks);
    if (rc) return rc;
    ADAQP_REQUIRE(row_end >= row_begin && row_begin >= 0, ADAQP_EINVAL, "adaqp_gatv2_fwd_f32: bad row range");
    ADAQP_REQUIRE(row_end <= n_split, ADAQP_EINVAL,
                  "adaqp_gatv2_fwd_f32: rows must be local (row_end %lld > n_split %lld)", (long long)row_end,
                  (long long)n_split);
    ADAQP_REQUIRE(ldzs0 >= F && ldzd >= F && ldo >= F && (!zs1 || ldzs1 >= F), ADAQP_EINVAL,
                  "adaqp_gatv2_fwd_f32: row pitch < F");
    if (row_end == row_begin) return 0;
    ADAQP_REQUIRE(indptr && indices && zs0 && zd && attn && out && lse, ADAQP_EINVAL,
                  "adaqp_gatv2_fwd_f32: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    int dev = 0;
    ADAQP_CUDA(cudaGetDevice(&dev));
    unsigned long long *counter = adaqp_frontier_counter(dev, s);
    ADAQP_REQUIRE(counter != nullptr, ADAQP_EINVAL, "adaqp_gatv2_fwd_f32: row counter allocation failed");
    const int64_t grid = frontier_grid(row_end - row_begin);
#define CALL_FWD(C)                                                                                                 \
    gatv2_fwd_kernel<C><<<(unsigned)grid, kThreads, 0, s>>>(indptr, indices, n_split, zs0, ldzs0, zs1, ldzs1, zd,  \
                                                            ldzd, attn, H, F, mode, D, cpg, row_begin, row_end, out, \
                                                            ldo, lse, counter)
    if (chunks == 1) CALL_FWD(1);
    else if (chunks == 2) CALL_FWD(2);
    else if (chunks == 4) CALL_FWD(4);
    else CALL_FWD(8);
#undef CALL_FWD
    return adaqp_check_launch("gatv2_fwd_kernel");
}

int adaqp_gatv2_bwd_inner_f32(const int64_t *indptr, const int32_t *indices, int64_t n_split, const float *zs0,
                              int64_t ldzs0, const float *zs1, int64_t ldzs1, const float *zd, int64_t ldzd,
                              const float *g, int64_t ldg, const float *lse, const float *S, const float *attn,
                              const float *push, int64_t ldp, const int64_t *fold_indptr, const int32_t *fold_pos,
                              int32_t H, int32_t F, int64_t row_begin, int64_t row_end, float *dzs, int64_t lddzs,
                              float *dzd, int64_t lddzd, float *da, int64_t ldda, void *stream) {
    int mode, D, cpg, chunks;
    int rc = head_layout("adaqp_gatv2_bwd_inner_f32", H, F, &mode, &D, &cpg, &chunks);
    if (rc) return rc;
    ADAQP_REQUIRE(row_end >= row_begin && row_begin >= 0, ADAQP_EINVAL, "adaqp_gatv2_bwd_inner_f32: bad row range");
    ADAQP_REQUIRE(row_end <= n_split, ADAQP_EINVAL,
                  "adaqp_gatv2_bwd_inner_f32: rows must be local (row_end %lld > n_split %lld)", (long long)row_end,
                  (long long)n_split);
    ADAQP_REQUIRE(ldzs0 >= F && ldzd >= F && ldg >= F && lddzs >= F && lddzd >= F && ldda >= F &&
                      (!zs1 || ldzs1 >= F) && (!push || ldp >= F),
                  ADAQP_EINVAL, "adaqp_gatv2_bwd_inner_f32: row pitch < F");
    ADAQP_REQUIRE((push == nullptr) == (fold_indptr == nullptr) && (fold_indptr == nullptr) == (fold_pos == nullptr),
                  ADAQP_EINVAL, "adaqp_gatv2_bwd_inner_f32: push, fold_indptr and fold_pos must be given together");
    if (row_end == row_begin) return 0;
    ADAQP_REQUIRE(indptr && indices && zs0 && zd && g && lse && S && attn && dzs && dzd && da, ADAQP_EINVAL,
                  "adaqp_gatv2_bwd_inner_f32: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    int dev = 0;
    ADAQP_CUDA(cudaGetDevice(&dev));
    unsigned long long *counter = adaqp_frontier_counter(dev, s);
    ADAQP_REQUIRE(counter != nullptr, ADAQP_EINVAL, "adaqp_gatv2_bwd_inner_f32: row counter allocation failed");
    const int64_t grid = frontier_grid(row_end - row_begin);
#define CALL_BWD(C)                                                                                                  \
    gatv2_bwd_inner_kernel<C><<<(unsigned)grid, kThreads, 0, s>>>(                                                   \
        indptr, indices, n_split, zs0, ldzs0, zs1, ldzs1, zd, ldzd, g, ldg, lse, S, attn, push, ldp, fold_indptr,    \
        fold_pos, H, F, mode, D, cpg, row_begin, row_end, dzs, lddzs, dzd, lddzd, da, ldda, counter)
    if (chunks == 1) CALL_BWD(1);
    else if (chunks == 2) CALL_BWD(2);
    else if (chunks == 4) CALL_BWD(4);
    else CALL_BWD(8);
#undef CALL_BWD
    return adaqp_check_launch("gatv2_bwd_inner_kernel");
}

int adaqp_gatv2_bwd_halo_f32(const int64_t *halo_indptr, const int32_t *halo_dst, const float *zs1, int64_t ldzs1,
                             const float *zd, int64_t ldzd, const float *g, int64_t ldg, const float *lse,
                             const float *S, const float *attn, int32_t H, int32_t F, int64_t row_begin,
                             int64_t row_end, float *out, int64_t ldo, void *stream) {
    int mode, D, cpg, chunks;
    int rc = head_layout("adaqp_gatv2_bwd_halo_f32", H, F, &mode, &D, &cpg, &chunks);
    if (rc) return rc;
    ADAQP_REQUIRE(row_end >= row_begin && row_begin >= 0, ADAQP_EINVAL, "adaqp_gatv2_bwd_halo_f32: bad row range");
    ADAQP_REQUIRE(ldzs1 >= F && ldzd >= F && ldg >= F && ldo >= F, ADAQP_EINVAL,
                  "adaqp_gatv2_bwd_halo_f32: row pitch < F");
    if (row_end == row_begin) return 0;
    ADAQP_REQUIRE(halo_indptr && halo_dst && zs1 && zd && g && lse && S && attn && out, ADAQP_EINVAL,
                  "adaqp_gatv2_bwd_halo_f32: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    int dev = 0;
    ADAQP_CUDA(cudaGetDevice(&dev));
    unsigned long long *counter = adaqp_frontier_counter(dev, s);
    ADAQP_REQUIRE(counter != nullptr, ADAQP_EINVAL, "adaqp_gatv2_bwd_halo_f32: row counter allocation failed");
    const int64_t grid = frontier_grid(row_end - row_begin);
#define CALL_HALO(C)                                                                                                \
    gatv2_bwd_halo_kernel<C><<<(unsigned)grid, kThreads, 0, s>>>(halo_indptr, halo_dst, zs1, ldzs1, zd, ldzd, g,   \
                                                                 ldg, lse, S, attn, H, F, mode, D, cpg, row_begin, \
                                                                 row_end, out, ldo, counter)
    if (chunks == 1) CALL_HALO(1);
    else if (chunks == 2) CALL_HALO(2);
    else if (chunks == 4) CALL_HALO(4);
    else CALL_HALO(8);
#undef CALL_HALO
    return adaqp_check_launch("gatv2_bwd_halo_kernel");
}

}  // extern "C"

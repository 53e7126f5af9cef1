// Graph attention (GAT) aggregation over the halo exchange (sm_90a).
//
// DGL's GATConv with one shared projection z = x W (computed by the dense GEMM), H heads of width D,
// F = H * D columns per row, negative slope 0.2:
//   el[i,h] = <z[i,h,:], a_l[h,:]>      er[i,h] = <z[i,h,:], a_r[h,:]>
//   e[v,u,h] = LeakyReLU(el[u,h] + er[v,h])   for u in N_in(v) (CSR row v, self-loop included)
//   lse[v,h] = logsumexp_u e[v,u,h]          alpha[v,u,h] = exp(e[v,u,h] - lse[v,h])
//   out[v,h,:] = sum_u alpha[v,u,h] z[u,h,:]
// Backward, with g = dL/dout and s[v,h] = <g[v,h,:], out[v,h,:]>:
//   t[v,u,h]  = alpha[v,u,h] (<g[v,h,:], z[u,h,:]> - s[v,h]) LeakyReLU'(el[u,h] + er[v,h])
//   dz[u]     = sum_{u->v} (alpha[v,u] g[v] + t[v,u] a_l) + (sum_{w->u} t[u,w]) a_r
//   del[u,h]  = sum_{u->v} t[v,u,h]          der[u,h] = sum_{w->u} t[u,w,h]
// The graph is symmetric, so the destinations of an inner row u are exactly the entries of its CSR row: one
// pass over row u serves u as a destination (der) and as a source (dz, del).
//
// Sources split as in spmm.cu: ids < n_split are local rows, ids >= n_split are halo rows (received from their
// owners).  Launches take a destination row range of the one CSR, so the central / marginal split of the
// overlapped path is two launches.  One warp per row; the column layout and the per-head reductions are those of
// attn.cuh.  fp32 throughout, no atomics on data: a row is always reduced by one warp in CSR order, so repeated
// launches are bitwise equal.
#include <math.h>

#include "attn.cuh"

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;
constexpr int kUnroll = 4;
constexpr float kSlope = 0.2f;

__device__ __forceinline__ float leaky(float x) { return x > 0.f ? x : kSlope * x; }

template <int CHUNKS>
__global__ void __launch_bounds__(kThreads)
gat_scores_kernel(const float *__restrict__ z, int64_t ldz, int64_t n_rows, const float *__restrict__ a_l,
                  const float *__restrict__ a_r, int H, int F, int mode, int D, int cpg, float *__restrict__ el,
                  float *__restrict__ er) {
    const int lane = threadIdx.x & 31;
    const Cols<CHUNKS> cols(lane, F, D);
    float al[CHUNKS], ar[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
        al[c] = cols.ok[c] ? __ldg(a_l + c * 32 + lane) : 0.f;
        ar[c] = cols.ok[c] ? __ldg(a_r + c * 32 + lane) : 0.f;
    }
    const int64_t warps = (int64_t)gridDim.x * kWarps;
    for (int64_t row = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); row < n_rows; row += warps) {
        float p[CHUNKS], q[CHUNKS];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            const float x = cols.ok[c] ? __ldg(z + row * ldz + c * 32 + lane) : 0.f;
            p[c] = x * al[c];
            q[c] = x * ar[c];
        }
        head_reduce<CHUNKS>(p, mode, D, cpg);
        head_reduce<CHUNKS>(q, mode, D, cpg);
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            if (cols.lead[c]) {
                el[row * H + cols.hid[c]] = p[c];
                er[row * H + cols.hid[c]] = q[c];
            }
        }
    }
}

// One warp per destination row, rows from the frontier counter.  Single-pass online softmax per head: the
// running maximum m and the rescaled sum / accumulator (one exp per column and neighbour), so every neighbour
// row z[u] is gathered once and any in-degree is exact.
template <int CHUNKS>
__global__ void __launch_bounds__(kThreads)
gat_fwd_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices, int64_t n_split,
               const float *__restrict__ z0, int64_t ldz0, const float *__restrict__ z1, int64_t ldz1,
               const float *__restrict__ el0, const float *__restrict__ el1, const float *__restrict__ er,
               int H, int F, int D, int64_t row_begin, int64_t row_end, float *__restrict__ out, int64_t ldo,
               float *__restrict__ lse, unsigned long long *__restrict__ next_row) {
    const int lane = threadIdx.x & 31;
    const Cols<CHUNKS> cols(lane, F, D);
    const int64_t n_rows = row_end - row_begin;
    while (true) {
        unsigned long long grab = 0;
        if (lane == 0) grab = atomicAdd(next_row, 1ull);
        grab = __shfl_sync(ADAQP_FULL_MASK, grab, 0);
        if ((int64_t)grab >= n_rows) break;
        const int64_t row = row_begin + (int64_t)grab;
        float erv[CHUNKS], m[CHUNKS], ssum[CHUNKS], acc[CHUNKS];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            erv[c] = cols.ok[c] ? __ldg(er + row * H + cols.hid[c]) : 0.f;
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
                float v[kUnroll][CHUNKS], sc[kUnroll][CHUNKS];
#pragma unroll
                for (int t = 0; t < kUnroll; ++t) {
                    const int uu = __shfl_sync(ADAQP_FULL_MASK, u, (k + t) & 31);
                    const bool live = (k + t) < n;
                    const bool local = uu < n_split;
                    const float *zr = local ? z0 + (int64_t)uu * ldz0 : z1 + ((int64_t)uu - n_split) * ldz1;
                    const float *lr = local ? el0 + (int64_t)uu * H : el1 + ((int64_t)uu - n_split) * H;
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c) {
                        if (live && cols.ok[c]) {
                            v[t][c] = __ldg(zr + c * 32 + lane);
                            sc[t][c] = __ldg(lr + cols.hid[c]);
                        } else {
                            v[t][c] = 0.f;
                            sc[t][c] = 0.f;
                        }
                    }
                }
#pragma unroll
                for (int t = 0; t < kUnroll; ++t) {
                    const bool live = (k + t) < n;           // warp-uniform
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c) {
                        if (!live || !cols.ok[c]) continue;
                        const float x = leaky(__fadd_rn(sc[t][c], erv[c]));
                        if (x > m[c]) {
                            const float r = expf(m[c] - x);     // exp(-inf) = 0 on the first neighbour
                            ssum[c] = __fmaf_rn(ssum[c], r, 1.f);
                            acc[c] = __fmaf_rn(acc[c], r, v[t][c]);
                            m[c] = x;
                        } else {
                            const float p = expf(x - m[c]);
                            ssum[c] = __fadd_rn(ssum[c], p);
                            acc[c] = __fmaf_rn(p, v[t][c], acc[c]);
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

// One warp per inner row u.  Neighbour x of u in the CSR row is both a destination of u (gather g[x] and
// er / lse / s of x: dz and del terms) and a source of u (gather z[x] and el[x]: der term).
// aux rows are [er | lse | s] (3H floats), local (aux0) or received with the halo (aux1).
template <int CHUNKS>
__global__ void __launch_bounds__(kThreads)
gat_bwd_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices, int64_t n_split,
               const float *__restrict__ g0, int64_t ldg0, const float *__restrict__ g1, int64_t ldg1,
               const float *__restrict__ z0, int64_t ldz0, const float *__restrict__ z1, int64_t ldz1,
               const float *__restrict__ el0, const float *__restrict__ el1, const float *__restrict__ aux0,
               const float *__restrict__ aux1, const float *__restrict__ a_l, const float *__restrict__ a_r,
               int H, int F, int mode, int D, int cpg, int64_t row_begin, int64_t row_end,
               float *__restrict__ dz, int64_t lddz, float *__restrict__ del, float *__restrict__ der,
               unsigned long long *__restrict__ next_row) {
    const int lane = threadIdx.x & 31;
    const Cols<CHUNKS> cols(lane, F, D);
    const int64_t n_rows = row_end - row_begin;
    const int ldx = 3 * H;
    while (true) {
        unsigned long long grab = 0;
        if (lane == 0) grab = atomicAdd(next_row, 1ull);
        grab = __shfl_sync(ADAQP_FULL_MASK, grab, 0);
        if ((int64_t)grab >= n_rows) break;
        const int64_t u = row_begin + (int64_t)grab;
        float zu[CHUNKS], gu[CHUNKS], elu[CHUNKS], eru[CHUNKS], lseu[CHUNKS], su[CHUNKS];
        float acc[CHUNKS], dl[CHUNKS], dr[CHUNKS];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            const bool ok = cols.ok[c];
            const int h = cols.hid[c];
            zu[c] = ok ? __ldg(z0 + u * ldz0 + c * 32 + lane) : 0.f;
            gu[c] = ok ? __ldg(g0 + u * ldg0 + c * 32 + lane) : 0.f;
            elu[c] = ok ? __ldg(el0 + u * H + h) : 0.f;
            eru[c] = ok ? __ldg(aux0 + u * ldx + h) : 0.f;
            lseu[c] = ok ? __ldg(aux0 + u * ldx + H + h) : 0.f;
            su[c] = ok ? __ldg(aux0 + u * ldx + 2 * H + h) : 0.f;
            acc[c] = dl[c] = dr[c] = 0.f;
        }
        const int64_t b = __ldg(indptr + u), e = __ldg(indptr + u + 1);
        for (int64_t j0 = b; j0 < e; j0 += 32) {
            const int n = (e - j0) < 32 ? (int)(e - j0) : 32;
            int xi = 0;
            if (lane < n) xi = __ldg(indices + j0 + lane);
            for (int k = 0; k < n; ++k) {
                const int x = __shfl_sync(ADAQP_FULL_MASK, xi, k);
                const bool local = x < n_split;
                const int64_t xr = local ? (int64_t)x : (int64_t)x - n_split;
                const float *gr = local ? g0 + xr * ldg0 : g1 + xr * ldg1;
                const float *zr = local ? z0 + xr * ldz0 : z1 + xr * ldz1;
                const float *lr = local ? el0 + xr * H : el1 + xr * H;
                const float *ar = local ? aux0 + xr * ldx : aux1 + xr * ldx;
                float gx[CHUNKS], p1[CHUNKS], p2[CHUNKS], elx[CHUNKS], erx[CHUNKS], lsex[CHUNKS], sx[CHUNKS];
#pragma unroll
                for (int c = 0; c < CHUNKS; ++c) {
                    const bool ok = cols.ok[c];
                    const int h = cols.hid[c];
                    gx[c] = ok ? __ldg(gr + c * 32 + lane) : 0.f;
                    const float zx = ok ? __ldg(zr + c * 32 + lane) : 0.f;
                    elx[c] = ok ? __ldg(lr + h) : 0.f;
                    erx[c] = ok ? __ldg(ar + h) : 0.f;
                    lsex[c] = ok ? __ldg(ar + H + h) : 0.f;
                    sx[c] = ok ? __ldg(ar + 2 * H + h) : 0.f;
                    p1[c] = __fmul_rn(gx[c], zu[c]);     // <g[x], z[u]>: u as a source of x
                    p2[c] = __fmul_rn(gu[c], zx);        // <g[u], z[x]>: x as a source of u
                }
                head_reduce<CHUNKS>(p1, mode, D, cpg);
                head_reduce<CHUNKS>(p2, mode, D, cpg);
#pragma unroll
                for (int c = 0; c < CHUNKS; ++c) {
                    if (!cols.ok[c]) continue;
                    const float e1 = __fadd_rn(elu[c], erx[c]);
                    const float a1 = expf(__fsub_rn(leaky(e1), lsex[c]));
                    const float t1 = __fmul_rn(__fmul_rn(a1, __fsub_rn(p1[c], sx[c])), e1 > 0.f ? 1.f : kSlope);
                    acc[c] = __fmaf_rn(a1, gx[c], acc[c]);
                    dl[c] = __fadd_rn(dl[c], t1);
                    const float e2 = __fadd_rn(elx[c], eru[c]);
                    const float a2 = expf(__fsub_rn(leaky(e2), lseu[c]));
                    const float t2 = __fmul_rn(__fmul_rn(a2, __fsub_rn(p2[c], su[c])), e2 > 0.f ? 1.f : kSlope);
                    dr[c] = __fadd_rn(dr[c], t2);
                }
            }
        }
        float *drow = dz + (u - row_begin) * lddz;
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            if (!cols.ok[c]) continue;
            const int col = c * 32 + lane;
            drow[col] = __fmaf_rn(dr[c], __ldg(a_r + col), __fmaf_rn(dl[c], __ldg(a_l + col), acc[c]));
            if (cols.lead[c]) {
                del[(u - row_begin) * H + cols.hid[c]] = dl[c];
                der[(u - row_begin) * H + cols.hid[c]] = dr[c];
            }
        }
    }
    frontier_release(next_row);
}

int64_t frontier_grid(int64_t rows) { return adaqp_frontier_grid(rows, kWarps); }

}  // namespace

extern "C" {

int adaqp_gat_scores_f32(const float *z, int64_t ldz, int64_t n_rows, int32_t H, int32_t F, const float *a_l,
                         const float *a_r, float *el, float *er, void *stream) {
    int mode, D, cpg, chunks;
    int rc = head_layout("adaqp_gat_scores_f32", H, F, &mode, &D, &cpg, &chunks);
    if (rc) return rc;
    ADAQP_REQUIRE(n_rows >= 0, ADAQP_EINVAL, "adaqp_gat_scores_f32: n_rows=%lld", (long long)n_rows);
    ADAQP_REQUIRE(ldz >= F, ADAQP_EINVAL, "adaqp_gat_scores_f32: ldz=%lld < F=%d", (long long)ldz, F);
    if (n_rows == 0) return 0;
    ADAQP_REQUIRE(z && a_l && a_r && el && er, ADAQP_EINVAL, "adaqp_gat_scores_f32: null pointer");
    cudaStream_t s = (cudaStream_t)stream;
    const int64_t grid = frontier_grid(n_rows);
#define CALL_SCORES(C) \
    gat_scores_kernel<C><<<(unsigned)grid, kThreads, 0, s>>>(z, ldz, n_rows, a_l, a_r, H, F, mode, D, cpg, el, er)
    if (chunks == 1) CALL_SCORES(1);
    else if (chunks == 2) CALL_SCORES(2);
    else if (chunks == 4) CALL_SCORES(4);
    else CALL_SCORES(8);
#undef CALL_SCORES
    return adaqp_check_launch("gat_scores_kernel");
}

int adaqp_gat_fwd_f32(const int64_t *indptr, const int32_t *indices, int64_t n_split, const float *z0, int64_t ldz0,
                      const float *z1, int64_t ldz1, const float *el0, const float *el1, const float *er, int32_t H,
                      int32_t F, int64_t row_begin, int64_t row_end, float *out, int64_t ldo, float *lse,
                      void *stream) {
    int mode, D, cpg, chunks;
    int rc = head_layout("adaqp_gat_fwd_f32", H, F, &mode, &D, &cpg, &chunks);
    if (rc) return rc;
    ADAQP_REQUIRE(row_end >= row_begin && row_begin >= 0, ADAQP_EINVAL, "adaqp_gat_fwd_f32: bad row range");
    ADAQP_REQUIRE(ldz0 >= F && ldo >= F && (!z1 || ldz1 >= F), ADAQP_EINVAL, "adaqp_gat_fwd_f32: row pitch < F");
    ADAQP_REQUIRE(n_split >= 0, ADAQP_EINVAL, "adaqp_gat_fwd_f32: n_split=%lld", (long long)n_split);
    if (row_end == row_begin) return 0;
    ADAQP_REQUIRE(indptr && indices && z0 && el0 && er && out && lse, ADAQP_EINVAL, "adaqp_gat_fwd_f32: null pointer");
    ADAQP_REQUIRE((z1 == nullptr) == (el1 == nullptr), ADAQP_EINVAL,
                  "adaqp_gat_fwd_f32: halo z1 and el1 must be given together");
    cudaStream_t s = (cudaStream_t)stream;
    int dev = 0;
    ADAQP_CUDA(cudaGetDevice(&dev));
    unsigned long long *counter = adaqp_frontier_counter(dev, s);
    ADAQP_REQUIRE(counter != nullptr, ADAQP_EINVAL, "adaqp_gat_fwd_f32: row counter allocation failed");
    const int64_t grid = frontier_grid(row_end - row_begin);
#define CALL_FWD(C)                                                                                              \
    gat_fwd_kernel<C><<<(unsigned)grid, kThreads, 0, s>>>(indptr, indices, n_split, z0, ldz0, z1, ldz1, el0, el1, \
                                                          er, H, F, D, row_begin, row_end, out, ldo, lse, counter)
    if (chunks == 1) CALL_FWD(1);
    else if (chunks == 2) CALL_FWD(2);
    else if (chunks == 4) CALL_FWD(4);
    else CALL_FWD(8);
#undef CALL_FWD
    return adaqp_check_launch("gat_fwd_kernel");
}

int adaqp_gat_bwd_f32(const int64_t *indptr, const int32_t *indices, int64_t n_split, const float *g0, int64_t ldg0,
                      const float *g1, int64_t ldg1, const float *z0, int64_t ldz0, const float *z1, int64_t ldz1,
                      const float *el0, const float *el1, const float *aux0, const float *aux1, const float *a_l,
                      const float *a_r, int32_t H, int32_t F, int64_t row_begin, int64_t row_end, float *dz,
                      int64_t lddz, float *del, float *der, void *stream) {
    int mode, D, cpg, chunks;
    int rc = head_layout("adaqp_gat_bwd_f32", H, F, &mode, &D, &cpg, &chunks);
    if (rc) return rc;
    ADAQP_REQUIRE(row_end >= row_begin && row_begin >= 0, ADAQP_EINVAL, "adaqp_gat_bwd_f32: bad row range");
    ADAQP_REQUIRE(row_end <= n_split, ADAQP_EINVAL, "adaqp_gat_bwd_f32: rows must be local (row_end %lld > n_split %lld)",
                  (long long)row_end, (long long)n_split);
    ADAQP_REQUIRE(ldg0 >= F && ldz0 >= F && lddz >= F && (!g1 || ldg1 >= F) && (!z1 || ldz1 >= F), ADAQP_EINVAL,
                  "adaqp_gat_bwd_f32: row pitch < F");
    if (row_end == row_begin) return 0;
    ADAQP_REQUIRE(indptr && indices && g0 && z0 && el0 && aux0 && a_l && a_r && dz && del && der, ADAQP_EINVAL,
                  "adaqp_gat_bwd_f32: null pointer");
    ADAQP_REQUIRE((g1 == nullptr) == (z1 == nullptr) && (z1 == nullptr) == (el1 == nullptr) &&
                      (el1 == nullptr) == (aux1 == nullptr),
                  ADAQP_EINVAL, "adaqp_gat_bwd_f32: halo g1, z1, el1 and aux1 must be given together");
    cudaStream_t s = (cudaStream_t)stream;
    int dev = 0;
    ADAQP_CUDA(cudaGetDevice(&dev));
    unsigned long long *counter = adaqp_frontier_counter(dev, s);
    ADAQP_REQUIRE(counter != nullptr, ADAQP_EINVAL, "adaqp_gat_bwd_f32: row counter allocation failed");
    const int64_t grid = frontier_grid(row_end - row_begin);
#define CALL_BWD(C)                                                                                                \
    gat_bwd_kernel<C><<<(unsigned)grid, kThreads, 0, s>>>(indptr, indices, n_split, g0, ldg0, g1, ldg1, z0, ldz0, z1, \
                                                          ldz1, el0, el1, aux0, aux1, a_l, a_r, H, F, mode, D, cpg,  \
                                                          row_begin, row_end, dz, lddz, del, der, counter)
    if (chunks == 1) CALL_BWD(1);
    else if (chunks == 2) CALL_BWD(2);
    else if (chunks == 4) CALL_BWD(4);
    else CALL_BWD(8);
#undef CALL_BWD
    return adaqp_check_launch("gat_bwd_kernel");
}

}  // extern "C"

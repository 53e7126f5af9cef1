// Row kernels of Correct & Smooth (DESIGN §16): the set-up before the correct steps and the combine between the
// correct and the smooth steps.  The propagation steps themselves are cs_prop_kernel (spmm.cu).
//
// One warp per row, the row's C <= 1024 columns strided over the lanes (column c on lane c % 32).  Rows are mapped
// statically to warps (CTA b, warp w takes rows (b + k * gridDim.x) * 8 + w), and every sum is a fixed-order loop
// per lane followed by a butterfly shuffle reduction, so the results and the per-CTA partials of the set-up depend
// only on the input and the grid, never on scheduling.  No float atomics.
#include "common.cuh"

namespace {

constexpr int kWarps = 8;
constexpr int kThreads = kWarps * 32;

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) v = fmaxf(v, __shfl_xor_sync(ADAQP_FULL_MASK, v, m));
    return v;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(ADAQP_FULL_MASK, v, m);
    return v;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int m = 16; m > 0; m >>= 1) v += __shfl_xor_sync(ADAQP_FULL_MASK, v, m);
    return v;
}

// yhat = softmax(z) per row (the row maximum subtracted); e0 = onehot(y) - yhat on rows with y >= 0, 0 elsewhere;
// partials[blockIdx.x] = sum over the CTA's rows of |e0|_1, in float64 (warps summed in warp order).
__global__ void __launch_bounds__(kThreads)
cs_init_kernel(const float *__restrict__ z, int64_t ldz, const int32_t *__restrict__ y, int64_t rows, int C,
               float *__restrict__ yhat, int64_t ldy, float *__restrict__ e0, int64_t lde,
               double *__restrict__ partials) {
    __shared__ double warp_l1[kWarps];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    double l1 = 0.0;                                   // this lane's share of the warp's rows
    for (int64_t r = ((int64_t)blockIdx.x) * kWarps + wib; r < rows; r += (int64_t)gridDim.x * kWarps) {
        const float *zr = z + r * ldz;
        float m = -INFINITY;
        for (int c = lane; c < C; c += 32) m = fmaxf(m, __ldg(zr + c));
        m = warp_max(m);
        float s = 0.f;
        for (int c = lane; c < C; c += 32) s += expf(__ldg(zr + c) - m);
        s = warp_sum(s);
        const int label = __ldg(y + r);
        for (int c = lane; c < C; c += 32) {
            const float p = __fdiv_rn(expf(__ldg(zr + c) - m), s);
            yhat[r * ldy + c] = p;
            float e = 0.f;
            if (label >= 0) e = (c == label ? 1.f : 0.f) - p;
            e0[r * lde + c] = e;
            l1 += (double)fabsf(e);
        }
    }
    l1 = warp_sum(l1);
    if (lane == 0) warp_l1[wib] = l1;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < kWarps; ++w) t += warp_l1[w];
        partials[blockIdx.x] = t;
    }
}

// g0[v] = onehot(y[v]) on rows with y >= 0; elsewhere g0[v] = yhat[v] + s[v] e[v] with
//   autoscale: s[v] = sigma / |e[v]|_1, and s[v] = 1 where |e[v]|_1 = 0 or s[v] > 1000 (in float64),
//   fixed    : s[v] = value.
__global__ void __launch_bounds__(kThreads)
cs_combine_kernel(const float *__restrict__ yhat, int64_t ldy, const float *__restrict__ e, int64_t lde,
                  const int32_t *__restrict__ y, int64_t rows, int C, int autoscale, double value,
                  float *__restrict__ g0, int64_t ldg) {
    const int lane = threadIdx.x & 31;
    const int64_t nwarps = (int64_t)gridDim.x * kWarps;
    for (int64_t r = (int64_t)blockIdx.x * kWarps + (threadIdx.x >> 5); r < rows; r += nwarps) {
        const int label = __ldg(y + r);
        float *gr = g0 + r * ldg;
        if (label >= 0) {
            for (int c = lane; c < C; c += 32) gr[c] = c == label ? 1.f : 0.f;
            continue;
        }
        const float *er = e + r * lde;
        float s = (float)value;
        if (autoscale) {
            double l1 = 0.0;
            for (int c = lane; c < C; c += 32) l1 += (double)fabsf(__ldg(er + c));
            l1 = warp_sum(l1);
            const double sd = l1 > 0.0 ? value / l1 : 1.0;
            s = sd > 1000.0 ? 1.f : (float)sd;
        }
        const float *yr = yhat + r * ldy;
        for (int c = lane; c < C; c += 32) gr[c] = __fmaf_rn(s, __ldg(er + c), __ldg(yr + c));
    }
}

}  // namespace

extern "C" {

int adaqp_cs_init_f32(const float *z, int64_t ldz, const int32_t *y, int64_t rows, int32_t C, float *yhat,
                      int64_t ldy, float *e0, int64_t lde, double *partials, int32_t n_partials, void *stream) {
    ADAQP_REQUIRE(C > 0 && C <= 1024, ADAQP_EINVAL, "adaqp_cs_init_f32: C=%d outside [1, 1024]", C);
    ADAQP_REQUIRE(rows >= 0 && ldz >= C && ldy >= C && lde >= C, ADAQP_EINVAL,
                  "adaqp_cs_init_f32: bad shape rows=%lld C=%d", (long long)rows, C);
    ADAQP_REQUIRE(n_partials > 0, ADAQP_EINVAL, "adaqp_cs_init_f32: n_partials=%d", n_partials);
    ADAQP_REQUIRE(z && y && yhat && e0 && partials, ADAQP_EINVAL, "adaqp_cs_init_f32: null pointer");
    cs_init_kernel<<<(unsigned)n_partials, kThreads, 0, (cudaStream_t)stream>>>(z, ldz, y, rows, C, yhat, ldy, e0, lde,
                                                                                partials);
    return adaqp_check_launch("cs_init_kernel");
}

int adaqp_cs_combine_f32(const float *yhat, int64_t ldy, const float *e, int64_t lde, const int32_t *y, int64_t rows,
                         int32_t C, int32_t autoscale, double value, float *g0, int64_t ldg, void *stream) {
    ADAQP_REQUIRE(C > 0 && C <= 1024, ADAQP_EINVAL, "adaqp_cs_combine_f32: C=%d outside [1, 1024]", C);
    ADAQP_REQUIRE(rows >= 0 && ldy >= C && lde >= C && ldg >= C, ADAQP_EINVAL,
                  "adaqp_cs_combine_f32: bad shape rows=%lld C=%d", (long long)rows, C);
    ADAQP_REQUIRE(autoscale ? (value >= 0.0 && value < INFINITY) : (value > 0.0 && value < INFINITY), ADAQP_EINVAL,
                  "adaqp_cs_combine_f32: bad %s %g", autoscale ? "sigma" : "scale", value);
    if (rows == 0) return 0;
    ADAQP_REQUIRE(yhat && e && y && g0, ADAQP_EINVAL, "adaqp_cs_combine_f32: null pointer");
    int64_t grid = (rows + kWarps - 1) / kWarps;
    const int sms = adaqp_sm_count() > 0 ? adaqp_sm_count() : 132;
    if (grid > (int64_t)sms * 8) grid = (int64_t)sms * 8;
    cs_combine_kernel<<<(unsigned)grid, kThreads, 0, (cudaStream_t)stream>>>(yhat, ldy, e, lde, y, rows, C,
                                                                             autoscale ? 1 : 0, value, g0, ldg);
    return adaqp_check_launch("cs_combine_kernel");
}

}  // extern "C"

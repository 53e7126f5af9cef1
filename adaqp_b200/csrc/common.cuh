// Shared device helpers for libadaqp_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/adaqp_b200.h"

#define ADAQP_FULL_MASK 0xffffffffu

// ---------------------------------------------------------------- errors
void adaqp_set_error(const char *fmt, ...);
int adaqp_check_launch(const char *what);

// Tunables set through adaqp_set_option() (runtime.cu); no environment reads in the library.
struct AdaqpOptions {
    int spmm_impl;            // 1 register gather (default), 2 cp.async ring, 3 TMA gather4 ring, 4 TMA bulk ring
    int spmm_rows_per_grab;   // 0 = per-kernel default
    int spmm_ctas_per_sm;     // frontier kernel grid cap per SM
    int spmm_hints;           // bit 0: streaming output stores, bit 1: streaming index loads
    int exch_send_ctas;       // 0 = one resident wave; > 0 = total CTA cap of the send kernels
    int exch_recv_ctas;       // same for the receive kernel
    int gemm_block_k;         // K block of gemm_tf32x3_kernel: 32 (SWIZZLE_128B, 2 stages) or 16 (SWIZZLE_64B, 4 stages)
    int spmm_slice_cols;      // column-slice width of the default aggregation: 0 = automatic, >= F = unsliced
};
AdaqpOptions &adaqp_options();

#define ADAQP_REQUIRE(cond, code, ...)            \
    do {                                          \
        if (!(cond)) {                            \
            adaqp_set_error(__VA_ARGS__);         \
            return (code);                        \
        }                                         \
    } while (0)

#define ADAQP_CUDA(call)                                                     \
    do {                                                                     \
        cudaError_t _e = (call);                                             \
        if (_e != cudaSuccess) {                                             \
            adaqp_set_error("%s failed: %s", #call, cudaGetErrorString(_e)); \
            return (int)_e;                                                  \
        }                                                                    \
    } while (0)

// ---------------------------------------------------------------- frontier row scheduler
// Row counter of the frontier scheduler: {next_row, finished CTAs}.  The last CTA to finish puts both
// words back to zero, so a launch needs no memset node and one counter pair per (device, stream)
// can never be shared by two launches that are in flight together.
__device__ __forceinline__ void frontier_release(unsigned long long *counter) {
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned long long prev = atomicAdd(counter + 1, 1ull);
        if (prev == (unsigned long long)gridDim.x - 1ull) {
            counter[0] = 0ull;
            counter[1] = 0ull;
            __threadfence();
        }
    }
}
// The counter pair of (device, stream), allocated zeroed on first use (spmm.cu).
unsigned long long *adaqp_frontier_counter(int dev, cudaStream_t s);
// Grid of a one-warp-per-row frontier kernel: enough CTAs for every row, at most 8 per SM.
inline int64_t adaqp_frontier_grid(int64_t rows, int warps_per_cta) {
    const int sms = adaqp_sm_count() > 0 ? adaqp_sm_count() : 132;
    int64_t grid = (rows + warps_per_cta - 1) / warps_per_cta;
    if (grid > (int64_t)sms * 8) grid = (int64_t)sms * 8;
    return grid;
}

// ---------------------------------------------------------------- Philox
// Philox4x32-10 exactly as curand's curand_Philox4x32_10 (curand_philox4x32_x.h):
// counter (x,y) = Philox offset / 4, (z,w) = subsequence, key = seed.
#define PHILOX_W0 0x9E3779B9u
#define PHILOX_W1 0xBB67AE85u
#define PHILOX_M0 0xD2511F53u
#define PHILOX_M1 0xCD9E8D57u

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint64_t p0 = (uint64_t)PHILOX_M0 * c.x;
        const uint64_t p1 = (uint64_t)PHILOX_M1 * c.z;
        const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
        const uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += PHILOX_W0;  // the bump after round 10 is dead code and is removed
        k.y += PHILOX_W1;
    }
    return c;
}

// _curand_uniform: x * 2^-32 + 2^-33 in fp32 (one rounding either way).
__device__ __forceinline__ float uniform_from_u32(uint32_t x) {
    return __fmaf_rn(__uint2float_rn(x), 2.3283064365386963e-10f, 1.1641532182693481e-10f);
}

// Round keys precomputed on the host and passed as a __grid_constant__ kernel parameter:
// the 20 key-schedule adds per block disappear and LOP3 reads the keys straight from the
// constant bank.
struct PhiloxKeys {
    uint32_t kx[10];
    uint32_t ky[10];
};

static inline PhiloxKeys make_philox_keys(uint64_t seed) {
    PhiloxKeys K;
    uint32_t x = (uint32_t)seed, y = (uint32_t)(seed >> 32);
    for (int r = 0; r < 10; ++r) {
        K.kx[r] = x;
        K.ky[r] = y;
        x += PHILOX_W0;
        y += PHILOX_W1;
    }
    return K;
}

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, const PhiloxKeys &K) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint64_t p0 = (uint64_t)PHILOX_M0 * c.x;
        const uint64_t p1 = (uint64_t)PHILOX_M1 * c.z;
        c = make_uint4((uint32_t)(p1 >> 32) ^ c.y ^ K.kx[r], (uint32_t)p1, (uint32_t)(p0 >> 32) ^ c.w ^ K.ky[r], (uint32_t)p0);
    }
    return c;
}

// N independent Philox blocks advanced round by round: the 10-round dependency chain of one
// block (IMAD.WIDE -> LOP3 -> ...) leaves the issue slots idle, N interleaved chains fill them.
template <int N>
__device__ __forceinline__ void philox4x32_10_xN(uint4 (&c)[N], const PhiloxKeys &K) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
#pragma unroll
        for (int j = 0; j < N; ++j) {
            const uint64_t p0 = (uint64_t)PHILOX_M0 * c[j].x;
            const uint64_t p1 = (uint64_t)PHILOX_M1 * c[j].z;
            c[j] = make_uint4((uint32_t)(p1 >> 32) ^ c[j].y ^ K.kx[r], (uint32_t)p1,
                              (uint32_t)(p0 >> 32) ^ c[j].w ^ K.ky[r], (uint32_t)p0);
        }
    }
}

// Fast-path noise for torch-style offsets (offset % 4 == 0) and WPT <= 4: one block per byte.
template <int WPT>
__device__ __forceinline__ void byte_noise_fast(const PhiloxKeys &K, uint32_t blk_lo, uint32_t blk_hi,
                                                uint32_t k_lo, uint32_t k_hi, float (&u)[WPT]) {
    const uint4 a = philox4x32_10(make_uint4(blk_lo, blk_hi, k_lo, k_hi), K);
    u[0] = uniform_from_u32(a.x);
    if (WPT > 1) u[1 % WPT] = uniform_from_u32(a.y);
    if (WPT > 2) { u[2 % WPT] = uniform_from_u32(a.z); u[3 % WPT] = uniform_from_u32(a.w); }
}

// The uniforms the reference draws for packed byte `k` of a pack call whose generator
// inputs are (seed, offset): curand_init(seed, subsequence = k, offset) followed by
// WPT = 8/bits curand_uniform draws.  Draw i is word (offset%4 + i)%4 of the Philox
// block at counter (offset/4 + (offset%4 + i)/4, k).  torch's Philox offsets are
// always multiples of 4, so one block serves all draws for bits >= 2 (fast path).
__device__ __forceinline__ uint4 philox_block(uint64_t blk, uint64_t k, uint2 key) {
    // carry from (x,y) into (z,w) needs offset >= 2^66: unreachable
    return philox4x32_10(make_uint4((uint32_t)blk, (uint32_t)(blk >> 32), (uint32_t)k, (uint32_t)(k >> 32)), key);
}

template <int WPT>
__device__ __forceinline__ void byte_noise(uint64_t seed, uint64_t k, uint64_t offset, float (&u)[WPT]) {
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    const uint64_t blk = offset >> 2;
    const uint32_t phase = (uint32_t)(offset & 3);
    if (phase == 0) {
        const uint4 a = philox_block(blk, k, key);
        u[0] = uniform_from_u32(a.x);
        if (WPT > 1) u[1 % WPT] = uniform_from_u32(a.y);
        if (WPT > 2) { u[2 % WPT] = uniform_from_u32(a.z); u[3 % WPT] = uniform_from_u32(a.w); }
        if (WPT > 4) {
            const uint4 b = philox_block(blk + 1, k, key);
            u[4 % WPT] = uniform_from_u32(b.x); u[5 % WPT] = uniform_from_u32(b.y);
            u[6 % WPT] = uniform_from_u32(b.z); u[7 % WPT] = uniform_from_u32(b.w);
        }
    } else {  // never taken with torch generators; kept for exactness of the contract
        uint32_t w[12];
#pragma unroll
        for (int b = 0; b < 3; ++b) {
            if ((uint32_t)(b * 4) < phase + WPT) {
                const uint4 o = philox_block(blk + b, k, key);
                w[4 * b] = o.x; w[4 * b + 1] = o.y; w[4 * b + 2] = o.z; w[4 * b + 3] = o.w;
            }
        }
#pragma unroll
        for (int i = 0; i < WPT; ++i) u[i] = uniform_from_u32(w[phase + i]);
    }
}

// One stochastic quantization step, bit-identical to the reference's
//   __float2int_rn(fmax((x - min) * scale + noise - 0.5, 0.0f))
// whose SASS is FADD, FFMA (contracted), F2F.F64, DADD -0.5, DMNMX 0, F2F.F32, F2I.RNI.
// For t >= 0.5 the double subtraction is exact whenever fp32 (t - 0.5) could round
// differently, so RN_f32(RN_f64(t - 0.5)) == RN_f32(t - 0.5) == __fsub_rn(t, 0.5f);
// for t < 0.5 (and NaN) the max() returns 0 on both paths (DESIGN.md, "quantize in fp32").
__device__ __forceinline__ int quantize_one(float x, float mn, float scale, float noise) {
    float t = __fsub_rn(x, mn);
    t = __fmaf_rn(t, scale, noise);
    float f = __fsub_rn(t, 0.5f);
    f = fmaxf(f, 0.0f);  // NaN -> 0 like fmax(double NaN, 0.0)
    return __float2int_rn(f);
}

// val / scale for a small non-negative integer val, bit-identical to the reference's IEEE
// division.  A zero numerator (every row minimum quantises to 0; relu'd rows are mostly 0)
// sends nvcc's division sequence (FCHK) to its slow-path subroutine, so the quotient for 0 is
// computed once per row (q_zero = __fdiv_rn(0.f, scale): +0, or NaN for scale 0 / NaN) and
// selected here; non-zero numerators with normal scales stay on the fast path.
__device__ __forceinline__ float dequant_div(uint32_t ival, float scale, float q_zero) {
    return ival == 0u ? q_zero : __fdiv_rn((float)ival, scale);
}

// fp32 -> bf16 bits with c10::BFloat16 semantics (RNE, NaN -> 0x7FC0).
__device__ __forceinline__ uint16_t f32_to_bf16_bits(float f) {
    if (f != f) return (uint16_t)0x7FC0;
    const uint32_t u = __float_as_uint(f);
    const uint32_t bias = ((u >> 16) & 1u) + 0x7FFFu;
    return (uint16_t)((u + bias) >> 16);
}

__device__ __forceinline__ float bf16_bits_to_f32(uint16_t h) {
    return __uint_as_float(((uint32_t)h) << 16);
}

// ---------------------------------------------------------------- memory ops
__device__ __forceinline__ uint64_t globaltimer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// streaming loads that do not pollute L1 (each boundary row is read once)
__device__ __forceinline__ float4 ldg_stream_f4(const float *p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
    return v;
}
__device__ __forceinline__ float2 ldg_stream_f2(const float *p) {
    float2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0,%1}, [%2];"
                 : "=f"(v.x), "=f"(v.y) : "l"(p));
    return v;
}
__device__ __forceinline__ float ldg_stream_f1(const float *p) {
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}

// Spin until *flag >= seq (sequence numbers are monotone per key; wrap-safe compare).
// Returns false on timeout.
__device__ __forceinline__ bool spin_wait_ge(const uint32_t *flag, uint32_t seq, uint64_t timeout_ns) {
    if ((int32_t)(ld_acquire_sys(flag) - seq) >= 0) return true;
    const uint64_t t0 = globaltimer_ns();
    unsigned backoff = 32;
    while (true) {
        if ((int32_t)(ld_acquire_sys(flag) - seq) >= 0) return true;
        __nanosleep(backoff);
        if (backoff < 1024) backoff <<= 1;
        if (globaltimer_ns() - t0 > timeout_ns) return false;
    }
}

__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(ADAQP_FULL_MASK, v, o));
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(ADAQP_FULL_MASK, v, o));
    return v;
}

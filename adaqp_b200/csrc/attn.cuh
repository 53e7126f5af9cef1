// Per-head column layout shared by the attention kernels (gat.cu, gatv2.cu).
//
// Rows are F = H * D floats (H heads of width D, F <= 256).  One warp per row; lane l owns columns c * 32 + l
// (c < CHUNKS), so a row gather is CHUNKS coalesced 128-byte loads.  Per-head dot products are reductions over the
// lanes / chunks of one head (head_reduce): the xor butterfly leaves the bit-identical sum on every lane of the
// head, so all lanes agree on every attention weight.
#pragma once

#include "common.cuh"

namespace {

// How the columns of one head map onto (chunk, lane): H == 1 -> the whole row; D % 32 == 0 -> `cpg` = D / 32
// consecutive whole chunks; 32 % D == 0 -> aligned groups of D lanes inside each chunk.
enum HeadMode { kHeadRow = 0, kHeadChunks = 1, kHeadLanes = 2 };

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(ADAQP_FULL_MASK, v, o);
    return v;
}

// v[c] <- sum of v over all columns of the head of column c * 32 + lane; every lane must call it
// (columns past F carry 0).
template <int CHUNKS>
__device__ __forceinline__ void head_reduce(float (&v)[CHUNKS], int mode, int D, int cpg) {
    if (mode == kHeadRow) {
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) s += v[c];
        s = warp_sum(s);
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) v[c] = s;
    } else if (mode == kHeadChunks) {
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            if (c % cpg == 0) {          // warp-uniform: first chunk of a head
                float s = 0.f;
#pragma unroll
                for (int k = 0; k < CHUNKS; ++k)
                    if (k >= c && k < c + cpg) s += v[k];
                s = warp_sum(s);
#pragma unroll
                for (int k = 0; k < CHUNKS; ++k)
                    if (k >= c && k < c + cpg) v[k] = s;
            }
        }
    } else {
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c)
            for (int o = D >> 1; o > 0; o >>= 1) v[c] += __shfl_xor_sync(ADAQP_FULL_MASK, v[c], o);
    }
}

template <int CHUNKS>
struct Cols {
    int hid[CHUNKS];     // head of column c * 32 + lane
    bool ok[CHUNKS];     // column < F
    bool lead[CHUNKS];   // first column of its head: writes the per-head scalars
    __device__ __forceinline__ Cols(int lane, int F, int D) {
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            const int col = c * 32 + lane;
            ok[c] = col < F;
            hid[c] = ok[c] ? col / D : 0;
            lead[c] = ok[c] && (col % D) == 0;
        }
    }
};

// Shape check shared by the attention entry points: sets (mode, D, cpg, chunks).
inline int head_layout(const char *what, int32_t H, int32_t F, int *mode, int *D, int *cpg, int *chunks) {
    ADAQP_REQUIRE(F > 0 && F <= 256, ADAQP_ELIMIT, "%s: F=%d outside (0,256]", what, F);
    ADAQP_REQUIRE(H > 0 && F % H == 0, ADAQP_EINVAL, "%s: H=%d does not divide F=%d", what, H, F);
    *D = F / H;
    *cpg = 1;
    if (H == 1) *mode = kHeadRow;
    else if (*D % 32 == 0) { *mode = kHeadChunks; *cpg = *D / 32; }
    else if (32 % *D == 0) *mode = kHeadLanes;
    else {
        adaqp_set_error("%s: head width D=%d (F=%d, H=%d) must be a multiple or a divisor of 32 when H > 1", what,
                        *D, F, H);
        return ADAQP_ELIMIT;
    }
    const int c = (F + 31) / 32;
    *chunks = c <= 1 ? 1 : c <= 2 ? 2 : c <= 4 ? 4 : 8;
    return 0;
}

}  // namespace

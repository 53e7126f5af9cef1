// Multilevel label-propagation graph partitioning (coarsen / refine / rebalance kernels).
// Replaces dgl.distributed.partition_graph(..., num_hops=1, balance_edges=False), i.e. METIS,
// called at AdaQP/helper/partition.py:71-72.  The level driver and the host initial partition
// live in adaqp_b200/partition.py; torch sorts the proposals and holds every buffer.
//
// Move rule of one sub-round (r, s) (DESIGN.md, "Graph partitioning"): a vertex v is active iff
// h(seed, r, v) & 1 == s.  It rates every neighbouring label c by rho(c) = sum of the weights of
// its edges to neighbours labelled c and proposes the label b != a = label[v] with the largest
// rho among the labels with room for it (lw[b] + vw[v] <= cap), ties to the smallest
// h(seed, r, c), then the smallest c, and only if rho(b) - rho(a) > 0.  Every quantity is an
// integer, so the atomics below are order-free and the result is identical on every run.
#include <assert.h>

#include "common.cuh"

namespace {

constexpr int RATE_WARPS = 4;                  // warps per CTA of the rating kernels
constexpr int HASH_SLOTS = 2 * ADAQP_LP_HUB_DEGREE;  // per-warp table, load factor <= 1/2
constexpr int32_t EMPTY_KEY = -1;

__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// h(seed, r, x): the one mixing function of the move rule (mirrored by oracle/partition_oracle.py)
__device__ __forceinline__ uint64_t lp_hash(uint64_t seed_mix, uint32_t round, uint64_t x) {
    return splitmix64(splitmix64(seed_mix ^ (uint64_t)round) ^ x);
}

// Better candidate: larger rho, then smaller h(c), then smaller c.
struct Cand {
    int64_t rho;
    uint64_t h;
    int32_t c;  // -1 = none
};

__device__ __forceinline__ bool better(const Cand &x, const Cand &y) {
    if (x.c < 0) return false;
    if (y.c < 0) return true;
    if (x.rho != y.rho) return x.rho > y.rho;
    if (x.h != y.h) return x.h < y.h;
    return x.c < y.c;
}

__device__ __forceinline__ Cand shfl_cand(const Cand &x, int src_lane_xor) {
    Cand o;
    o.rho = __shfl_xor_sync(ADAQP_FULL_MASK, x.rho, src_lane_xor);
    o.h = __shfl_xor_sync(ADAQP_FULL_MASK, x.h, src_lane_xor);
    o.c = __shfl_xor_sync(ADAQP_FULL_MASK, x.c, src_lane_xor);
    return o;
}

__device__ __forceinline__ Cand warp_best(Cand x) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const Cand y = shfl_cand(x, o);
        if (better(y, x)) x = y;
    }
    return x;
}

__device__ __forceinline__ int64_t warp_sum64(int64_t v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(ADAQP_FULL_MASK, v, o);
    return v;
}

__device__ __forceinline__ int64_t warp_max64(int64_t v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const int64_t y = __shfl_xor_sync(ADAQP_FULL_MASK, v, o);
        v = y > v ? y : v;
    }
    return v;
}

__device__ __forceinline__ uint32_t slot_of(int32_t key, uint32_t mask) {
    return (uint32_t)splitmix64((uint64_t)(uint32_t)key) & mask;
}

// Open-addressing insert of (key, w) into a per-warp shared-memory table of (mask + 1) slots.  32-bit keys and sums
// use the native atomics (64-bit shared-memory atomics are a compare-and-swap retry loop); a sum is at most the
// vertex's total edge weight, which int32 edge weights and ids bound.  The table holds twice as many slots as the
// vertex has edges, so a probe always ends within mask + 1 steps.
__device__ __forceinline__ void table_add(int32_t *keys, uint32_t *vals, uint32_t mask, int32_t key, uint32_t w) {
    uint32_t s = slot_of(key, mask);
    for (uint32_t probe = 0;; ++probe) {
        assert(probe <= mask);
        int32_t k = keys[s];
        if (k == EMPTY_KEY) {
            k = atomicCAS(&keys[s], EMPTY_KEY, key);
            if (k == EMPTY_KEY) k = key;
        }
        if (k == key) {
            atomicAdd(&vals[s], w);
            return;
        }
        s = (s + 1) & mask;
    }
}

__device__ __forceinline__ void write_proposal(int64_t v, const Cand &best, int64_t rho_a, int require_gain, int32_t *tgt,
                                               int64_t *gain) {
    const int64_t g = best.rho - rho_a;
    const bool ok = best.c >= 0 && (!require_gain || g > 0);
    tgt[v] = ok ? best.c : -1;
    gain[v] = ok ? g : 0;
}

// Clustering rating, one warp per vertex of degree <= ADAQP_LP_HUB_DEGREE (per-warp shared hash table).
__global__ void __launch_bounds__(RATE_WARPS * 32) lp_rate_clusters_kernel(
    const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices, const int32_t *__restrict__ ew,
    const int32_t *__restrict__ vw, int64_t n, const int32_t *__restrict__ label, const int64_t *__restrict__ lw,
    int64_t cap, uint64_t seed_mix, uint32_t round, int sub, int32_t *__restrict__ tgt, int64_t *__restrict__ gain,
    int64_t *__restrict__ hkey) {
    __shared__ int32_t s_keys[RATE_WARPS][HASH_SLOTS];
    __shared__ uint32_t s_vals[RATE_WARPS][HASH_SLOTS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    int32_t *keys = s_keys[warp];
    uint32_t *vals = s_vals[warp];
    const int64_t stride = (int64_t)gridDim.x * RATE_WARPS;
    for (int64_t v = (int64_t)blockIdx.x * RATE_WARPS + warp; v < n; v += stride) {
        const int64_t beg = indptr[v], end = indptr[v + 1];
        if (end - beg > ADAQP_LP_HUB_DEGREE) continue;  // lp_rate_hubs_kernel
        const uint64_t hv = lp_hash(seed_mix, round, (uint64_t)v);
        if (lane == 0) hkey[v] = (int64_t)(hv >> 1);
        if ((int)(hv & 1) != sub) {
            if (lane == 0) { tgt[v] = -1; gain[v] = 0; }
            continue;
        }
        for (int s = lane; s < HASH_SLOTS; s += 32) { keys[s] = EMPTY_KEY; vals[s] = 0; }
        __syncwarp();
        for (int64_t e = beg + lane; e < end; e += 32) table_add(keys, vals, HASH_SLOTS - 1, label[indices[e]], (uint32_t)ew[e]);
        __syncwarp();
        const int32_t a = label[v];
        const int64_t w = vw[v];
        Cand best{0, 0, -1};
        int64_t rho_a = 0;
        for (int s = lane; s < HASH_SLOTS; s += 32) {
            const int32_t c = keys[s];
            if (c == EMPTY_KEY) continue;
            if (c == a) { rho_a = vals[s]; continue; }
            if (lw[c] + w > cap) continue;
            const Cand x{(int64_t)vals[s], lp_hash(seed_mix, round, (uint64_t)c), c};
            if (better(x, best)) best = x;
        }
        best = warp_best(best);
        rho_a = warp_sum64(rho_a);
        if (lane == 0) write_proposal(v, best, rho_a, 1, tgt, gain);
        __syncwarp();
    }
}

// Clustering rating of the hub vertices (degree > ADAQP_LP_HUB_DEGREE): CTA b rates hubs b, b + gridDim.x, ...
// with a dense counter row scratch[b * n_labels ..] indexed by label (zero on entry; walking the same edges
// again puts it back to zero).  No hashing, so exact for any degree.  The counters are read with L2 loads:
// the block's own atomics bypass L1.
__global__ void __launch_bounds__(256) lp_rate_hubs_kernel(
    const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices, const int32_t *__restrict__ ew,
    const int32_t *__restrict__ vw, const int32_t *__restrict__ label, const int64_t *__restrict__ lw, int64_t cap,
    const int32_t *__restrict__ hubs, int64_t n_hubs, uint32_t *__restrict__ scratch, int64_t n_labels,
    uint64_t seed_mix, uint32_t round, int sub, int32_t *__restrict__ tgt, int64_t *__restrict__ gain,
    int64_t *__restrict__ hkey) {
    __shared__ Cand s_best[8];
    __shared__ int64_t s_rho[8];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t *cnt = scratch + (int64_t)blockIdx.x * n_labels;
    for (int64_t i = blockIdx.x; i < n_hubs; i += gridDim.x) {
        const int64_t v = hubs[i];
        const uint64_t hv = lp_hash(seed_mix, round, (uint64_t)v);
        if ((int)(hv & 1) != sub) {
            if (threadIdx.x == 0) { hkey[v] = (int64_t)(hv >> 1); tgt[v] = -1; gain[v] = 0; }
            continue;
        }
        const int64_t beg = indptr[v], end = indptr[v + 1];
        for (int64_t e = beg + threadIdx.x; e < end; e += blockDim.x) atomicAdd(&cnt[label[indices[e]]], (uint32_t)ew[e]);
        __syncthreads();
        const int32_t a = label[v];
        const int64_t w = vw[v];
        Cand best{0, 0, -1};
        int64_t rho_a = 0;
        for (int64_t e = beg + threadIdx.x; e < end; e += blockDim.x) {
            const int32_t c = label[indices[e]];
            const int64_t rho = __ldcg(&cnt[c]);
            if (c == a) { rho_a = rho; continue; }
            if (lw[c] + w > cap) continue;
            const Cand x{rho, lp_hash(seed_mix, round, (uint64_t)c), c};
            if (better(x, best)) best = x;
        }
        best = warp_best(best);
        rho_a = warp_max64(rho_a);
        if (lane == 0) { s_best[warp] = best; s_rho[warp] = rho_a; }
        __syncthreads();
        for (int64_t e = beg + threadIdx.x; e < end; e += blockDim.x) cnt[label[indices[e]]] = 0u;
        if (warp == 0) {
            const int nw = blockDim.x >> 5;
            best = lane < nw ? s_best[lane] : Cand{0, 0, -1};
            rho_a = lane < nw ? s_rho[lane] : 0;
            best = warp_best(best);
            rho_a = warp_max64(rho_a);
            if (lane == 0) { hkey[v] = (int64_t)(hv >> 1); write_proposal(v, best, rho_a, 1, tgt, gain); }
        }
        __syncthreads();
    }
}

// k-way rating (k <= 64): one warp per vertex, k counters per warp.  mode 0 = refinement (active by
// parity, gain > 0 required); mode 1 = rebalancing (active iff its block is over cap, every block with
// room is a candidate, any gain).
__global__ void __launch_bounds__(RATE_WARPS * 32) lp_rate_blocks_kernel(
    const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices, const int32_t *__restrict__ ew,
    const int32_t *__restrict__ vw, int64_t n, const int32_t *__restrict__ part, const int64_t *__restrict__ bw,
    int k, int64_t cap, uint64_t seed_mix, uint32_t round, int sub, int mode, int32_t *__restrict__ tgt,
    int64_t *__restrict__ gain, int64_t *__restrict__ hkey) {
    __shared__ uint32_t s_rho[RATE_WARPS][64];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint32_t *rho = s_rho[warp];
    const int64_t stride = (int64_t)gridDim.x * RATE_WARPS;
    for (int64_t v = (int64_t)blockIdx.x * RATE_WARPS + warp; v < n; v += stride) {
        const uint64_t hv = lp_hash(seed_mix, round, (uint64_t)v);
        const int32_t a = part[v];
        const bool active = mode == 0 ? (int)(hv & 1) == sub : bw[a] > cap;
        if (lane == 0) hkey[v] = (int64_t)(hv >> 1);
        if (!active) {
            if (lane == 0) { tgt[v] = -1; gain[v] = 0; }
            continue;
        }
        rho[lane] = 0;
        rho[lane + 32] = 0;
        __syncwarp();
        const int64_t beg = indptr[v], end = indptr[v + 1];
        for (int64_t e = beg + lane; e < end; e += 32) atomicAdd(&rho[part[indices[e]]], (uint32_t)ew[e]);
        __syncwarp();
        const int64_t w = vw[v];
        Cand best{0, 0, -1};
        for (int c = lane; c < k; c += 32) {
            if (c == a || bw[c] + w > cap) continue;
            const Cand x{(int64_t)rho[c], lp_hash(seed_mix, round, (uint64_t)c), c};
            if (better(x, best)) best = x;
        }
        best = warp_best(best);
        if (lane == 0) write_proposal(v, best, (int64_t)rho[a], mode == 0, tgt, gain);
        __syncwarp();
    }
}

// First position j <= i of the run of `i` in a sequence sorted by key[order[.]].
__device__ __forceinline__ int64_t run_start(const int32_t *order, const int32_t *key, int64_t i) {
    const int32_t b = key[order[i]];
    int64_t lo = 0, hi = i;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (key[order[mid]] < b) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// Accept, per target label, the longest prefix of its proposals that fits under cap (label weights as
// they were at the start of the sub-round), move the accepted vertices, accumulate the weight change.
__global__ void lp_apply_kernel(const int32_t *__restrict__ order, int64_t n_prop, const int64_t *__restrict__ csum,
                                const int32_t *__restrict__ tgt, const int32_t *__restrict__ vw,
                                int32_t *__restrict__ label, const int64_t *__restrict__ lw, int64_t cap,
                                int64_t *__restrict__ dlw) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_prop; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t v = order[i];
        const int32_t b = tgt[v];
        const int64_t j = run_start(order, tgt, i);
        const int64_t prefix = csum[i] - (j > 0 ? csum[j - 1] : 0);
        if (lw[b] + prefix > cap) continue;
        const int32_t a = label[v];
        const int64_t w = vw[v];
        label[v] = b;
        atomicAdd((unsigned long long *)&dlw[b], (unsigned long long)w);
        atomicAdd((unsigned long long *)&dlw[a], (unsigned long long)(-w));
    }
}

// Rebalancing, source side: of the proposals leaving each over-full block (sorted by source block, gain
// descending, h ascending), keep the shortest prefix whose weight covers the block's excess.
__global__ void lp_rebalance_select_kernel(const int32_t *__restrict__ order, int64_t n_prop,
                                           const int64_t *__restrict__ csum, const int32_t *__restrict__ part,
                                           const int32_t *__restrict__ vw, const int64_t *__restrict__ bw, int64_t cap,
                                           int32_t *__restrict__ tgt) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_prop; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t v = order[i];
        const int64_t j = run_start(order, part, i);
        const int64_t before = csum[i] - vw[v] - (j > 0 ? csum[j - 1] : 0);
        if (before >= bw[part[v]] - cap) tgt[v] = -1;
    }
}

// Contraction: edge (v -> u) becomes key (cid[v] << 32 | cid[u]), or INT64_MAX if both ends share a cluster.
__global__ void contract_edges_kernel(const int64_t *__restrict__ indptr, const int32_t *__restrict__ indices,
                                      int64_t n, const int32_t *__restrict__ cid, int64_t *__restrict__ key) {
    const int lane = threadIdx.x & 31;
    const int64_t stride = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t v = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); v < n; v += stride) {
        const int64_t cv = cid[v];
        for (int64_t e = indptr[v] + lane; e < indptr[v + 1]; e += 32) {
            const int64_t cu = cid[indices[e]];
            key[e] = cu == cv ? INT64_MAX : (cv << 32) | cu;
        }
    }
}

int grid_for(int64_t items, int per_block) {
    const int64_t g = (items + per_block - 1) / per_block;
    const int64_t lim = (int64_t)148 * 32;  // grid-stride loops: a few waves are enough
    return (int)(g < 1 ? 1 : (g > lim ? lim : g));
}

}  // namespace

extern "C" {

int adaqp_lp_rate_clusters(const int64_t *indptr, const int32_t *indices, const int32_t *ew, const int32_t *vw,
                           int64_t n, const int32_t *label, const int64_t *lw, int64_t cap, const int32_t *hubs,
                           int64_t n_hubs, uint32_t *hub_scratch, int32_t hub_ctas, uint64_t seed, uint32_t round, int sub,
                           int32_t *tgt, int64_t *gain, int64_t *hkey, void *stream) {
    ADAQP_REQUIRE(n >= 0 && n <= INT32_MAX && n_hubs >= 0 && n_hubs <= n && cap >= 0 && (sub == 0 || sub == 1),
                  ADAQP_EINVAL, "adaqp_lp_rate_clusters: bad sizes (n=%lld n_hubs=%lld cap=%lld sub=%d)",
                  (long long)n, (long long)n_hubs, (long long)cap, sub);
    ADAQP_REQUIRE(n == 0 || (indptr && indices && ew && vw && label && lw && tgt && gain && hkey), ADAQP_EINVAL,
                  "adaqp_lp_rate_clusters: null pointer");
    ADAQP_REQUIRE(n_hubs == 0 || (hubs && hub_scratch && hub_ctas >= 1), ADAQP_EINVAL,
                  "adaqp_lp_rate_clusters: hubs need hub_scratch and hub_ctas >= 1");
    if (n == 0) return 0;
    cudaStream_t s = (cudaStream_t)stream;
    const uint64_t sm = splitmix64(seed);
    lp_rate_clusters_kernel<<<grid_for(n, RATE_WARPS), RATE_WARPS * 32, 0, s>>>(
        indptr, indices, ew, vw, n, label, lw, cap, sm, round, sub, tgt, gain, hkey);
    if (int rc = adaqp_check_launch("lp_rate_clusters_kernel")) return rc;
    if (n_hubs > 0) {
        const unsigned grid = (unsigned)(n_hubs < hub_ctas ? n_hubs : hub_ctas);
        lp_rate_hubs_kernel<<<grid, 256, 0, s>>>(indptr, indices, ew, vw, label, lw, cap, hubs, n_hubs, hub_scratch, n,
                                                 sm, round, sub, tgt, gain, hkey);
        if (int rc = adaqp_check_launch("lp_rate_hubs_kernel")) return rc;
    }
    return 0;
}

int adaqp_lp_rate_blocks(const int64_t *indptr, const int32_t *indices, const int32_t *ew, const int32_t *vw, int64_t n,
                         const int32_t *part, const int64_t *bw, int32_t k, int64_t cap, uint64_t seed, uint32_t round,
                         int sub, int mode, int32_t *tgt, int64_t *gain, int64_t *hkey, void *stream) {
    ADAQP_REQUIRE(k >= 1 && k <= ADAQP_MAX_PARTS, ADAQP_EINVAL, "adaqp_lp_rate_blocks: k=%d outside [1, %d]", (int)k,
                  ADAQP_MAX_PARTS);
    ADAQP_REQUIRE(n >= 0 && n <= INT32_MAX && cap >= 0 && (sub == 0 || sub == 1) && (mode == 0 || mode == 1),
                  ADAQP_EINVAL, "adaqp_lp_rate_blocks: bad sizes (n=%lld cap=%lld sub=%d mode=%d)", (long long)n,
                  (long long)cap, sub, mode);
    ADAQP_REQUIRE(n == 0 || (indptr && indices && ew && vw && part && bw && tgt && gain && hkey), ADAQP_EINVAL,
                  "adaqp_lp_rate_blocks: null pointer");
    if (n == 0) return 0;
    lp_rate_blocks_kernel<<<grid_for(n, RATE_WARPS), RATE_WARPS * 32, 0, (cudaStream_t)stream>>>(
        indptr, indices, ew, vw, n, part, bw, k, cap, splitmix64(seed), round, sub, mode, tgt, gain, hkey);
    return adaqp_check_launch("lp_rate_blocks_kernel");
}

int adaqp_lp_apply(const int32_t *order, int64_t n_prop, const int64_t *csum, const int32_t *tgt, const int32_t *vw,
                   int32_t *label, const int64_t *lw, int64_t cap, int64_t *dlw, void *stream) {
    ADAQP_REQUIRE(n_prop >= 0 && n_prop <= INT32_MAX && cap >= 0, ADAQP_EINVAL,
                  "adaqp_lp_apply: bad sizes (n_prop=%lld cap=%lld)", (long long)n_prop, (long long)cap);
    ADAQP_REQUIRE(n_prop == 0 || (order && csum && tgt && vw && label && lw && dlw), ADAQP_EINVAL,
                  "adaqp_lp_apply: null pointer");
    if (n_prop == 0) return 0;
    lp_apply_kernel<<<grid_for(n_prop, 256), 256, 0, (cudaStream_t)stream>>>(order, n_prop, csum, tgt, vw, label, lw,
                                                                              cap, dlw);
    return adaqp_check_launch("lp_apply_kernel");
}

int adaqp_lp_rebalance_select(const int32_t *order, int64_t n_prop, const int64_t *csum, const int32_t *part,
                              const int32_t *vw, const int64_t *bw, int64_t cap, int32_t *tgt, void *stream) {
    ADAQP_REQUIRE(n_prop >= 0 && n_prop <= INT32_MAX && cap >= 0, ADAQP_EINVAL,
                  "adaqp_lp_rebalance_select: bad sizes (n_prop=%lld cap=%lld)", (long long)n_prop, (long long)cap);
    ADAQP_REQUIRE(n_prop == 0 || (order && csum && part && vw && bw && tgt), ADAQP_EINVAL,
                  "adaqp_lp_rebalance_select: null pointer");
    if (n_prop == 0) return 0;
    lp_rebalance_select_kernel<<<grid_for(n_prop, 256), 256, 0, (cudaStream_t)stream>>>(order, n_prop, csum, part, vw,
                                                                                          bw, cap, tgt);
    return adaqp_check_launch("lp_rebalance_select_kernel");
}

int adaqp_contract_edges(const int64_t *indptr, const int32_t *indices, int64_t n, const int32_t *cid, int64_t *key,
                         void *stream) {
    ADAQP_REQUIRE(n >= 0 && n <= INT32_MAX, ADAQP_EINVAL, "adaqp_contract_edges: bad size n=%lld", (long long)n);
    ADAQP_REQUIRE(n == 0 || (indptr && indices && cid && key), ADAQP_EINVAL, "adaqp_contract_edges: null pointer");
    if (n == 0) return 0;
    contract_edges_kernel<<<grid_for(n, 8), 256, 0, (cudaStream_t)stream>>>(indptr, indices, n, cid, key);
    return adaqp_check_launch("contract_edges_kernel");
}

}  // extern "C"

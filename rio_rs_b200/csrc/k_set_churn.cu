// k_set_churn.cu -- the erase half of object churn in a resident set (DESIGN.md 3.18): the erase-key hash set, the mark pass, the
// hole/mover pairing and the row moves.  In a translation unit of its own, so that no existing kernel's code depends on it.
#include "kernels.cuh"
#include "k_set_churn.cuh"
#include "k_key_probe.cuh"
#include "k_rank_common.cuh"

namespace rio {

namespace {

constexpr int kScanThreads = 1024;

// one thread per erase key; duplicates find their own key and stop
__global__ void __launch_bounds__(256)
k_churn_build(const uint64_t *__restrict__ keys, uint64_t m, unsigned long long *__restrict__ table, uint32_t lg, uint32_t *__restrict__ has_empty) {
    const uint64_t mask = (1ull << lg) - 1, stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += stride) {
        const unsigned long long k = __ldg(keys + t);
        if (k == kEmptyKey) { *has_empty = 1; continue; }
        for (uint64_t s = churn_slot(k, lg);; s = (s + 1) & mask) {
            const unsigned long long old = atomicCAS(table + s, kEmptyKey, k);
            if (old == kEmptyKey || old == k) break;
        }
    }
}

// One block per kChurnRows rows, one thread per row: 8 B of key and a probe of the (L2-resident) table per row, a flag byte written,
// 4 B of idx read for an erased row of an assigned set.  The counter updates of a warp are merged per node.
__global__ void __launch_bounds__(kChurnRows)
k_churn_mark(const uint64_t *__restrict__ keys, const uint32_t *__restrict__ idx, uint64_t n, const unsigned long long *__restrict__ table, uint32_t lg,
             const uint32_t *__restrict__ has_empty, uint32_t *__restrict__ counters, uint32_t n_total, uint8_t *__restrict__ flag,
             uint32_t *__restrict__ block_cnt, unsigned long long *__restrict__ erased) {
    const uint64_t i = (uint64_t)blockIdx.x * kChurnRows + threadIdx.x, mask = (1ull << lg) - 1;
    bool hit = false;
    if (i < n) {
        const unsigned long long k = __ldg(keys + i);
        if (k == kEmptyKey) {
            hit = __ldg(has_empty) != 0;
        } else {
            for (uint64_t s = churn_slot(k, lg);; s = (s + 1) & mask) {
                const unsigned long long t = __ldg(table + s);
                if (t == k) { hit = true; break; }
                if (t == kEmptyKey) break;
            }
        }
        flag[i] = hit ? 1 : 0;
    }
    uint32_t node = kNone;
    if (hit && counters) {
        node = __ldg(idx + i);
        if (node >= n_total) node = kNone;
    }
    warp_count_add(counters, node, 0xFFFFFFFFu);
    const uint32_t c = (uint32_t)__syncthreads_count(hit);
    if (threadIdx.x == 0) {
        block_cnt[blockIdx.x] = c;
        if (c) atomicAdd(erased, (unsigned long long)c);
    }
}

// holes and movers of block b, given its flagged count and the holes of the block that holds row n_new
__device__ __forceinline__ void block_split(uint64_t b, uint64_t n, uint64_t n_new, uint32_t cnt, uint32_t straddle_holes, uint32_t &holes,
                                            uint32_t &movers) {
    const uint64_t lo = b * kChurnRows, hi = lo + kChurnRows < n ? lo + kChurnRows : n;
    if (hi <= n_new) { holes = cnt; movers = 0; }
    else if (lo >= n_new) { holes = 0; movers = (uint32_t)(hi - lo) - cnt; }
    else { holes = straddle_holes; movers = (uint32_t)(hi - n_new) - (cnt - straddle_holes); }
}

// inclusive sum over the block of (a, b); every thread gets the block totals too
__device__ __forceinline__ void block_scan2(uint32_t &a, uint32_t &b, uint32_t &tot_a, uint32_t &tot_b) {
    __shared__ uint32_t wa[kScanThreads / 32], wb[kScanThreads / 32];
    const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t ta = __shfl_up_sync(0xFFFFFFFFu, a, o), tb = __shfl_up_sync(0xFFFFFFFFu, b, o);
        if (lane >= (unsigned)o) { a += ta; b += tb; }
    }
    if (lane == 31) { wa[w] = a; wb[w] = b; }
    __syncthreads();
    if (w == 0) {
        uint32_t x = wa[lane], y = wb[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t tx = __shfl_up_sync(0xFFFFFFFFu, x, o), ty = __shfl_up_sync(0xFFFFFFFFu, y, o);
            if (lane >= (unsigned)o) { x += tx; y += ty; }
        }
        wa[lane] = x; wb[lane] = y;
    }
    __syncthreads();
    if (w) { a += wa[w - 1]; b += wb[w - 1]; }
    tot_a = wa[kScanThreads / 32 - 1];
    tot_b = wb[kScanThreads / 32 - 1];
    __syncthreads();
}

// One block: the exclusive offsets of every block's holes and movers.  Thread t takes a contiguous run of blocks, so the block counts
// are read twice (8 B per kChurnRows rows).
__global__ void __launch_bounds__(kScanThreads)
k_churn_scan(const uint8_t *__restrict__ flag, uint64_t n, uint64_t n_new, const uint32_t *__restrict__ block_cnt, uint32_t *__restrict__ hole_off,
             uint32_t *__restrict__ mover_off, unsigned long long *__restrict__ pairs) {
    const uint64_t nb = (n + kChurnRows - 1) / kChurnRows, sb = n_new / kChurnRows;
    uint32_t mine = 0;
    if (threadIdx.x < kChurnRows) {
        const uint64_t i = sb * kChurnRows + threadIdx.x;
        mine = i < n_new && flag[i];
    }
    const uint32_t straddle = (uint32_t)__syncthreads_count(mine);
    const uint64_t per = (nb + kScanThreads - 1) / kScanThreads, b0 = threadIdx.x * per, b1 = b0 + per < nb ? b0 + per : nb;
    uint32_t h = 0, m = 0;
    for (uint64_t b = b0; b < b1; b++) {
        uint32_t bh, bm;
        block_split(b, n, n_new, __ldg(block_cnt + b), straddle, bh, bm);
        h += bh; m += bm;
    }
    uint32_t ih = h, im = m, tot_h, tot_m;
    block_scan2(ih, im, tot_h, tot_m);
    h = ih - h; m = im - m;   // exclusive
    for (uint64_t b = b0; b < b1; b++) {
        uint32_t bh, bm;
        block_split(b, n, n_new, __ldg(block_cnt + b), straddle, bh, bm);
        hole_off[b] = h; mover_off[b] = m;
        h += bh; m += bm;
    }
    if (threadIdx.x == 0) *pairs = tot_h;
}

// One block per kChurnRows rows: each hole and mover written at its block's offset plus its rank in the block.  A block with no hole
// and no mover reads only its count.
__global__ void __launch_bounds__(kChurnRows)
k_churn_list(const uint8_t *__restrict__ flag, uint64_t n, uint64_t n_new, const uint32_t *__restrict__ block_cnt, const uint32_t *__restrict__ hole_off,
             const uint32_t *__restrict__ mover_off, uint32_t *__restrict__ holes, uint32_t *__restrict__ movers) {
    __shared__ uint32_t wh[kChurnRows / 32], wm[kChurnRows / 32];
    const uint64_t b = blockIdx.x, lo = b * kChurnRows, hi = lo + kChurnRows < n ? lo + kChurnRows : n;
    const uint32_t cnt = __ldg(block_cnt + b);
    if (hi <= n_new && cnt == 0) return;              // no hole
    if (lo >= n_new && cnt == hi - lo) return;        // no mover
    const uint64_t i = lo + threadIdx.x;
    const bool f = i < hi && flag[i] != 0;
    const bool hole = f && i < n_new, mover = i < hi && !f && i >= n_new;
    const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5, below = (1u << lane) - 1u;
    const unsigned bh = __ballot_sync(0xFFFFFFFFu, hole), bm = __ballot_sync(0xFFFFFFFFu, mover);
    if (lane == 0) { wh[w] = __popc(bh); wm[w] = __popc(bm); }
    __syncthreads();
    uint32_t ph = 0, pm = 0;
    for (unsigned q = 0; q < w; q++) { ph += wh[q]; pm += wm[q]; }
    if (hole) holes[__ldg(hole_off + b) + ph + __popc(bh & below)] = (uint32_t)i;
    if (mover) movers[__ldg(mover_off + b) + pm + __popc(bm & below)] = (uint32_t)i;
}

// One warp per pair: lane 0 moves the key and idx, the lanes below ranks the list row, the lanes the feature row in 32-float strides.
// Holes lie below n_new and movers at or above it, so no pair reads a row another pair writes.
__global__ void __launch_bounds__(256)
k_churn_move(const uint32_t *__restrict__ holes, const uint32_t *__restrict__ movers, const unsigned long long *__restrict__ pairs,
             uint64_t *__restrict__ keys, uint32_t *__restrict__ idx, uint32_t *__restrict__ lists, uint32_t R, float *__restrict__ feats, uint32_t K) {
    const uint64_t P = __ldg(pairs), wstride = (uint64_t)gridDim.x * (blockDim.x / 32);
    const uint32_t lane = threadIdx.x & 31;
    for (uint64_t j = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) / 32; j < P; j += wstride) {
        const uint64_t h = __ldg(holes + j), s = __ldg(movers + j);
        if (lane == 0) { keys[h] = keys[s]; idx[h] = idx[s]; }
        if (lists && lane < R) lists[h * R + lane] = lists[s * R + lane];
        if (feats)
            for (uint32_t k = lane; k < K; k += 32) feats[h * K + k] = feats[s * K + k];
    }
}

int capped_grid(uint64_t blocks, const Launch &L, int per_sm) {
    const uint64_t cap = (uint64_t)L.sm_count * per_sm;
    if (blocks < 1) blocks = 1;
    return (int)(blocks < cap ? blocks : cap);
}

}  // namespace

void launch_churn_build(const Launch &L, const uint64_t *d_keys, uint64_t m, unsigned long long *d_table, uint32_t lg, uint32_t *d_has_empty) {
    if (!m) return;
    k_churn_build<<<capped_grid((m + 255) / 256, L, 8), 256, 0, L.stream>>>(d_keys, m, d_table, lg, d_has_empty);
    RIO_COUNT_LAUNCH(L);
}

void launch_churn_mark(const Launch &L, const uint64_t *d_keys, const uint32_t *d_idx, uint64_t n, const unsigned long long *d_table, uint32_t lg,
                       const uint32_t *d_has_empty, uint32_t *d_counters, uint32_t n_total, uint8_t *d_flag, uint32_t *d_block_cnt,
                       unsigned long long *d_erased) {
    if (!n) return;
    k_churn_mark<<<(unsigned)((n + kChurnRows - 1) / kChurnRows), kChurnRows, 0, L.stream>>>(d_keys, d_idx, n, d_table, lg, d_has_empty, d_counters, n_total,
                                                                                           d_flag, d_block_cnt, d_erased);
    RIO_COUNT_LAUNCH(L);
}

void launch_churn_pairs(const Launch &L, const uint8_t *d_flag, uint64_t n, uint64_t n_new, const uint32_t *d_block_cnt, uint32_t *d_hole_off,
                        uint32_t *d_mover_off, uint32_t *d_holes, uint32_t *d_movers, unsigned long long *d_pairs) {
    if (!n) return;
    k_churn_scan<<<1, kScanThreads, 0, L.stream>>>(d_flag, n, n_new, d_block_cnt, d_hole_off, d_mover_off, d_pairs);
    RIO_COUNT_LAUNCH(L);
    k_churn_list<<<(unsigned)((n + kChurnRows - 1) / kChurnRows), kChurnRows, 0, L.stream>>>(d_flag, n, n_new, d_block_cnt, d_hole_off, d_mover_off, d_holes,
                                                                                           d_movers);
    RIO_COUNT_LAUNCH(L);
}

void launch_churn_move(const Launch &L, const uint32_t *d_holes, const uint32_t *d_movers, uint64_t max_pairs, const unsigned long long *d_pairs,
                       uint64_t *d_keys, uint32_t *d_idx, uint32_t *d_lists, uint32_t ranks, float *d_feats, uint32_t K) {
    if (!max_pairs) return;
    k_churn_move<<<capped_grid((max_pairs + 7) / 8, L, 16), 256, 0, L.stream>>>(d_holes, d_movers, d_pairs, d_keys, d_idx, d_lists, ranks, d_feats, K);
    RIO_COUNT_LAUNCH(L);
}

}  // namespace rio

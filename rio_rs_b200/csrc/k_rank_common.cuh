// k_rank_common.cuh -- launch shape, shared-memory staging, the exact HRW2 contest, the compare-mode epilogue, the warp-aggregated
// list append and the rank dispatch of the ranked walks (k_ranked.cu, k_spread.cu) and the change-set passes (k_directory.cu,
// k_affinity_set.cu, k_set_bounded_affinity.cu, k_set_churn.cu).
// Included by .cu files only: everything is internal to the including translation unit.
#pragma once
#include "kernels.cuh"
#include "spec.cuh"

#include <type_traits>

namespace rio {

namespace {

constexpr int kRankThreads = 256;
constexpr uint32_t kRankLevels = 16;

// per-level contest constants (pseudo-node seeds c_l, DESIGN.md 3.8), passed by value: spec constants, the same for every handle
struct LevelConsts { uint32_t s0[kRankLevels], m2[kRankLevels], h2[kRankLevels]; };

LevelConsts level_consts() {
    LevelConsts c{};
    for (uint32_t l = 0; l < kRankLevels; l++) {
        const ContestRec r = contest_rec(level_seed(l));
        c.s0[l] = r.s0; c.m2[l] = r.m2; c.h2[l] = r.h2;
    }
    return c;
}

// 16-byte cooperative copy into shared memory (bytes is a multiple of 16)
__device__ __forceinline__ void stage16(unsigned char *dst, const void *src, uint32_t bytes) {
    const uint4 *s = reinterpret_cast<const uint4 *>(src);
    uint4 *d = reinterpret_cast<uint4 *>(dst);
    for (uint32_t i = threadIdx.x; i < bytes / 16; i += blockDim.x) d[i] = __ldg(s + i);
}

// v < floor(2^31 wl / (wl + wr))  <=>  (v + 1)(wl + wr) <= 2^31 wl, exactly; wl = 0 never takes LEFT, wr = 0 always does
__device__ __forceinline__ bool contest_left_exact(uint32_t v, unsigned long long wl, unsigned long long wr) {
    const unsigned long long a = (unsigned long long)v + 1ull, s = wl + wr;
    const unsigned long long plo = a * s, phi = __umul64hi(a, s);
    const unsigned long long qlo = wl << 31, qhi = wl >> 33;
    return phi < qhi || (phi == qhi && plo <= qlo);
}

// Domain-aware insert of a failure-domain list (DESIGN.md 3.12), best first under the order (E(u)*r, ~u, j) of cand_better, for a
// candidate the caller has already found better than the last entry.  A listed entry of the same domain that is better drops the
// candidate; otherwise the shift stops at the same-domain entry it replaces, if there is one.  Dense domain ids: no live node has kNone.
template <int R>
__device__ __forceinline__ void spread_insert(uint64_t (&gs)[R], uint32_t (&gu)[R], uint32_t (&gj)[R], uint32_t (&gd)[R], uint64_t s, uint32_t u,
                                              uint32_t j, uint32_t d) {
    bool keep = true;
#pragma unroll
    for (int y = 0; y < R; y++) keep &= !(gd[y] == d && cand_better(gs[y], gu[y], gj[y], s, u, j));
    if (!keep) return;
    const uint32_t dc = d;
    bool go = true;
#pragma unroll
    for (int y = 0; y < R; y++) {
        const bool sw = go && cand_better(s, u, j, gs[y], gu[y], gj[y]);
        const uint64_t ts = gs[y]; const uint32_t tu = gu[y], tj = gj[y], td = gd[y];
        gs[y] = sw ? s : ts; gu[y] = sw ? u : tu; gj[y] = sw ? j : tj; gd[y] = sw ? d : td;
        s = sw ? ts : s; u = sw ? tu : u; j = sw ? tj : j; d = sw ? td : d;
        go = go && !(sw && td == dc);
    }
}

// Every lane of the warp calls this with its number of items; returns the position of the lane's first item in a list whose
// length is *n (one atomic per warp).
__device__ __forceinline__ unsigned long long warp_reserve(unsigned long long *n, uint32_t mine) {
    const unsigned lane = threadIdx.x & 31;
    uint32_t pre = mine;   // inclusive warp prefix sum
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, pre, o); if (lane >= (unsigned)o) pre += t; }
    const uint32_t total = __shfl_sync(0xFFFFFFFFu, pre, 31);
    unsigned long long b = 0;
    if (lane == 0 && total) b = atomicAdd(n, (unsigned long long)total);
    return __shfl_sync(0xFFFFFFFFu, b, 0) + (pre - mine);
}

// counters[j] += delta for every lane's j (kNone: none), one atomic per distinct node of the warp: a joined node that many objects of a
// warp prefer, a leaving node they all held, or an erased rack, costs one atomic.  Every lane of the warp calls this.
__device__ __forceinline__ void warp_count_add(uint32_t *counters, uint32_t j, uint32_t delta) {
    if (__ballot_sync(0xFFFFFFFFu, j != kNone) == 0) return;
    const unsigned peers = __match_any_sync(0xFFFFFFFFu, j);
    if (j != kNone && (threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) atomicAdd(&counters[j], delta * (uint32_t)__popc(peers));
}

// loads[j] += w for every lane's (j, w) (kNone: none), one atomic per distinct node of the warp carrying the sum of its lanes' weights
// (DESIGN.md 3.19).  Every lane of the warp calls this.
__device__ __forceinline__ void warp_load_add(uint32_t *loads, uint32_t j, uint32_t w) {
    if (__ballot_sync(0xFFFFFFFFu, j != kNone) == 0) return;
    const unsigned peers = __match_any_sync(0xFFFFFFFFu, j);
    const uint32_t sum = __reduce_add_sync(peers, w);
    if (j != kNone && sum && (threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) atomicAdd(&loads[j], sum);
}

// Compare mode of the HRW2 walks (DESIGN.md 3.11, 3.13): the output holds the stored lists of a resident set.  Each walk is compared
// with the stored row, only changed rows are written, and the set's primary index and counters follow column 0.
struct RankedCmp {
    uint32_t *idx, *counters;
    uint32_t n_total;
    unsigned long long *moved, *changed;
};

// Stores object i's finished row res at dst.  Compare mode counts a changed row in n_changed and a changed column 0 in n_moved.
template <int R, bool CMP>
__device__ __forceinline__ void ranked_store(uint32_t *dst, const uint32_t (&res)[R], uint64_t i, const RankedCmp &cmp, uint32_t &n_moved,
                                             uint32_t &n_changed) {
    if (CMP) {
        bool changed = false;
#pragma unroll
        for (int r = 0; r < R; r++) changed |= dst[r] != res[r];
        if (changed) {
            const uint32_t old0 = dst[0];
#pragma unroll
            for (int r = 0; r < R; r++) dst[r] = res[r];
            n_changed++;
            if (old0 != res[0]) {
                cmp.idx[i] = res[0];
                n_moved++;
                if (old0 < cmp.n_total) atomicSub(&cmp.counters[old0], 1u);
                if (res[0] < cmp.n_total) atomicAdd(&cmp.counters[res[0]], 1u);
            }
        }
    } else {
#pragma unroll
        for (int r = 0; r < R; r++) dst[r] = res[r];
    }
}

// The end of a compare-mode kernel: every thread of the block gets here; one atomic per warp and counter.
template <bool CMP>
__device__ __forceinline__ void ranked_flush(const RankedCmp &cmp, uint32_t n_moved, uint32_t n_changed) {
    if (CMP) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { n_moved += __shfl_xor_sync(0xFFFFFFFFu, n_moved, o); n_changed += __shfl_xor_sync(0xFFFFFFFFu, n_changed, o); }
        if ((threadIdx.x & 31) == 0) {
            if (n_moved) atomicAdd(cmp.moved, (unsigned long long)n_moved);
            if (n_changed) atomicAdd(cmp.changed, (unsigned long long)n_changed);
        }
    }
}

// smem_budget: the most dynamic shared memory the including file's launchers give the kernel.  attr_set: one flag per device for THIS
// kernel instantiation (the attribute call costs ~1 us of host time per launch otherwise)
template <class K>
int ranked_grid(const Launch &L, K kern, size_t smem, uint32_t smem_budget, uint64_t n, bool (&attr_set)[64]) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !attr_set[dev]) {
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_budget);
        if (dev >= 0 && dev < 64) attr_set[dev] = true;
    }
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kRankThreads, smem);
    const uint64_t blocks = (n + kRankThreads - 1) / kRankThreads, cap = (uint64_t)L.sm_count * (uint64_t)(per_sm > 0 ? per_sm : 1);
    return (int)(blocks < cap ? blocks : cap);
}

// Launches kernel K over n objects with kRankThreads threads and smem bytes of dynamic shared memory
template <auto K, class... A>
void launch_rank_kernel(const Launch &L, size_t smem, uint32_t smem_budget, uint64_t n, const A &...args) {
    static bool attr_set[64] = {};
    const int grid = ranked_grid(L, K, smem, smem_budget, n, attr_set);
    K<<<grid, kRankThreads, smem, L.stream>>>(args...);
}

// Calls f(std::integral_constant<int, R>{}) for ranks = R in 1..8 and returns true; any other ranks launches nothing and returns false
template <class F>
bool with_ranks(uint32_t ranks, F &&f) {
    switch (ranks) {
        case 1: f(std::integral_constant<int, 1>{}); return true;
        case 2: f(std::integral_constant<int, 2>{}); return true;
        case 3: f(std::integral_constant<int, 3>{}); return true;
        case 4: f(std::integral_constant<int, 4>{}); return true;
        case 5: f(std::integral_constant<int, 5>{}); return true;
        case 6: f(std::integral_constant<int, 6>{}); return true;
        case 7: f(std::integral_constant<int, 7>{}); return true;
        case 8: f(std::integral_constant<int, 8>{}); return true;
        default: return false;
    }
}

}  // namespace

}  // namespace rio

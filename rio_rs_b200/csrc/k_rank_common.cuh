// k_rank_common.cuh -- launch shape, shared-memory staging and the exact HRW2 contest of the ranked walks (k_ranked.cu, k_spread.cu).
// Included by .cu files only: everything is internal to the including translation unit.
#pragma once
#include "kernels.cuh"
#include "spec.cuh"

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

// Compare mode of the HRW2 walks (DESIGN.md 3.11, 3.13): the output holds the stored lists of a resident set.  Each walk is compared
// with the stored row, only changed rows are written, and the set's primary index and counters follow column 0.
struct RankedCmp {
    uint32_t *idx, *counters;
    uint32_t n_total;
    unsigned long long *moved, *changed;
};

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

}  // namespace

}  // namespace rio

#define RIO_RANK_CASES(F, ...) \
    switch (ranks) { case 1: F<1>(__VA_ARGS__); break; case 2: F<2>(__VA_ARGS__); break; case 3: F<3>(__VA_ARGS__); break; \
                     case 4: F<4>(__VA_ARGS__); break; case 5: F<5>(__VA_ARGS__); break; case 6: F<6>(__VA_ARGS__); break; \
                     case 7: F<7>(__VA_ARGS__); break; case 8: F<8>(__VA_ARGS__); break; default: return; }

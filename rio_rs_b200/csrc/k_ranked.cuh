// k_ranked.cuh -- launchers and the side table of the ranked placement lists (k_ranked.cu, DESIGN.md 3.9).
#pragma once
#include "kernels.cuh"

namespace rio {

// ---- side table of the ranked HRW2 walk, built on the first ranked call after a table change ---------------------------------
//   [0, 16 << bits)             u64 subtree weights in heap order (index 1 = root, buckets at [2^bits, 2^(bits+1)); [0] unused)
//   then n_total x uint2        per interned node: {bucket, weight}; weight 0 = not a member of the trie
// One allocation, node part padded to 16 bytes so both parts can be staged with 16-byte copies.
struct TrieRankDev {
    const unsigned long long *wsum;
    const uint2 *node;
    uint32_t n_total;
    uint32_t n_members;    // live members of the trie: rank r > n_members is RIO_NONE
    uint32_t bytes;        // whole side table, multiple of 16
};
constexpr uint32_t kMaxRanks = 8;   // RIO_MAX_RANKS

// d_out_idx is n x ranks row-major, ranks in [1, kMaxRanks]; RIO_NONE pads a list longer than the live set.
// Declared weak: the engine's host code (engine.cu) can be linked into a library or test harness without k_ranked.cu, and then
// the ranked entry points answer with an error instead of failing to load; librio_cuda.so always links the kernels.
__attribute__((weak)) void launch_assign_hrw_ranked(const Launch &L, const uint64_t *d_keys, uint64_t n, const NodeTabDev &tab, uint32_t ranks,
                                                    uint32_t *d_out_idx);
__attribute__((weak)) void launch_assign_trie_ranked(const Launch &L, const uint64_t *d_keys, uint64_t n, const TrieDev &t, const TrieRankDev &rk,
                                                     uint32_t ranks, uint32_t *d_out_idx);

}  // namespace rio

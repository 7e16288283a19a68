// k_spread.cuh -- launchers and the side table of the failure-domain ranked lists (k_spread.cu, DESIGN.md 3.12).
#pragma once
#include "kernels.cuh"

namespace rio {

// ---- side table of the spread walks, built on the first spread call after a table or label change -----------------------------
// One allocation; every part starts on a 16-byte boundary.  The HRW2 walk stages [0, o_ndom) -- the bytes of TrieRankDev -- and reads
// the domain parts through the read-only path; the flat kernel stages the last part beside its records:
//   [0, 16 << bits)      u64 subtree weights in heap order (as TrieRankDev)
//   o_node               n_total x uint2: per interned node {bucket, weight}; weight 0 = not live
//   o_ndom               n_total x u32: dense domain id of a live node, kNone otherwise
//   o_pre                (n_members + 1) x u64: running weight of the live members sorted by (domain, bucket, index)
//   o_mb                 n_members x u32: the bucket of each member in that order
//   o_dstart             (n_domains + 1) x u32: first member of each domain in that order
//   trie_bytes           n_members x u32: dense domain id per class-sorted position of NodeTabDev::recs (the flat kernel)
struct SpreadTabDev {
    const unsigned char *base;
    uint32_t o_node, o_ndom, o_pre, o_mb, o_dstart;
    uint32_t trie_bytes;   // bytes of the HRW2 part = offset of the flat part, multiple of 16
    uint32_t n_members;    // live nodes
    uint32_t n_domains;    // distinct domains among them: rank r > n_domains is RIO_NONE
};

// d_out_idx is n x ranks row-major, ranks in [1, kMaxRanks]; RIO_NONE pads a list past the live domain count.
// Declared weak like the launchers of k_ranked.cuh: a build without k_spread.cu answers the spread calls with an error.
__attribute__((weak)) void launch_assign_hrw_spread(const Launch &L, const uint64_t *d_keys, uint64_t n, const NodeTabDev &tab, const SpreadTabDev &sp,
                                                    uint32_t ranks, uint32_t *d_out_idx);
__attribute__((weak)) void launch_assign_trie_spread(const Launch &L, const uint64_t *d_keys, uint64_t n, const TrieDev &t, const SpreadTabDev &sp,
                                                     uint32_t ranks, uint32_t *d_out_idx);

}  // namespace rio

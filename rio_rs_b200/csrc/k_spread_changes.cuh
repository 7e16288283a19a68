// k_spread_changes.cuh -- launchers of the failure-domain resident sets (DESIGN.md 3.13): spread lists of a set brought up to date by
// one change-set pass (k_directory.cu for the flat policy, the compare mode of k_assign_trie_spread in k_spread.cu for HRW2).
#pragma once
#include "kernels.cuh"
#include "k_changes.cuh"
#include "k_spread.cuh"

namespace rio {

// Declared weak, as in k_ranked_changes.cuh: the engine's host code can be linked without these launchers (the spread-set calls then
// answer with an error); librio_cuda.so always links them.  d_lists, d_idx and d_counters as in k_ranked_changes.cuh.
//
// Flat policy, one pass over keys and lists, the rule of launch_rebalance_changes_ranked with the domain-aware insert: an S2 list (no
// member in REPLACE or past the table) becomes the first ranks domain representatives of itself u CANDIDATES under the order of 3.4,
// with the dense domain ids of sp at the current labels; an S1 object is appended to d_sel, its row left alone.  A relabelled live
// node is REPLACE | CANDIDATE in cs.  The S1 rows are then recomputed by launch_assign_hrw_spread and written by launch_scatter_ranked.
__attribute__((weak)) void launch_rebalance_changes_spread(const Launch &L, const uint64_t *d_keys, uint32_t *d_lists, uint32_t ranks, uint32_t *d_idx, uint64_t n,
                                                           const NodeTabDev &tab, const ChangeSetDev &cs, const SpreadTabDev &sp, uint32_t *d_counters,
                                                           uint32_t *d_sel, unsigned long long *d_nsel, unsigned long long *d_moved,
                                                           unsigned long long *d_changed);
// HRW2: every list walked again with the domain exclusions and compared with the stored row; only the rows that changed are written
__attribute__((weak)) void launch_reassign_trie_spread(const Launch &L, const uint64_t *d_keys, uint64_t n, const TrieDev &t, const SpreadTabDev &sp, uint32_t ranks,
                                                       uint32_t *d_lists, uint32_t *d_idx, uint32_t *d_counters, uint32_t n_total,
                                                       unsigned long long *d_moved, unsigned long long *d_changed);

}  // namespace rio

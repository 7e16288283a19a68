// k_ranked_changes.cuh -- launchers of the ranked resident sets (DESIGN.md 3.11): the lists of a set brought up to date by one
// change-set pass (k_directory.cu for the flat policy, the compare mode of k_assign_trie_ranked in k_ranked.cu for HRW2).
#pragma once
#include "kernels.cuh"
#include "k_changes.cuh"
#include "k_ranked.cuh"

namespace rio {

// Declared weak, as in k_ranked.cuh and k_changes.cuh: the engine's host code can be linked without these launchers (the ranked set
// calls then answer with an error); librio_cuda.so always links them.  d_lists is n x ranks row-major, ranks in [1, kMaxRanks];
// d_idx is column 0 of it and d_counters its histogram over tab.n_total nodes; both are kept exact by every launcher below.
//
// set_assign_ranked: d_idx = column 0 of fresh lists (the counters are then rebuilt from d_idx)
__attribute__((weak)) void launch_ranked_primary(const Launch &L, const uint32_t *d_lists, uint64_t n, uint32_t ranks, uint32_t *d_idx);
// Flat policy, one pass over keys and lists: an S2 list (no member in REPLACE or past the table) becomes the first ranks elements of
// itself u CANDIDATES under the order of 3.4, written only if it changed; an S1 object is appended to d_sel, its row left alone.
// d_moved counts rows whose column 0 changed, d_changed rows that changed at all.
__attribute__((weak)) void launch_rebalance_changes_ranked(const Launch &L, const uint64_t *d_keys, uint32_t *d_lists, uint32_t ranks, uint32_t *d_idx, uint64_t n,
                                                           const NodeTabDev &tab, const ChangeSetDev &cs, uint32_t *d_counters, uint32_t *d_sel,
                                                           unsigned long long *d_nsel, unsigned long long *d_moved, unsigned long long *d_changed);
// ... then, once d_fresh (n_sel x ranks) holds the fresh lists of the selected objects: write back the rows that changed
__attribute__((weak)) void launch_scatter_ranked(const Launch &L, const uint32_t *d_fresh, const uint32_t *d_sel, uint64_t n_sel, uint32_t ranks, uint32_t *d_lists,
                                                 uint32_t *d_idx, uint32_t *d_counters, uint32_t n_total, unsigned long long *d_moved,
                                                 unsigned long long *d_changed);
// HRW2: every list walked again and compared with the stored row; only the rows that changed are written
__attribute__((weak)) void launch_reassign_trie_ranked(const Launch &L, const uint64_t *d_keys, uint64_t n, const TrieDev &t, const TrieRankDev &rk, uint32_t ranks,
                                                       uint32_t *d_lists, uint32_t *d_idx, uint32_t *d_counters, uint32_t n_total,
                                                       unsigned long long *d_moved, unsigned long long *d_changed);

}  // namespace rio

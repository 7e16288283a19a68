// k_set_churn.cuh -- launchers of the erase half of object churn in a resident set (DESIGN.md 3.18): a device hash set of the erase
// keys, one pass over the set's keys that flags the erased rows and takes them off the counters, the deterministic pairing of holes
// (erased rows below the new size) with movers (surviving rows at or above it), and the row moves.  Inserting needs no kernel of its
// own: the new rows are placed by the existing launchers on staged copies.
#pragma once
#include "kernels.cuh"

namespace rio {

// rows per block of the mark and pairing passes: d_block_cnt has one entry per kChurnRows rows
constexpr uint32_t kChurnRows = 256;
// the erase hash set: 1 << lg slots, kEmptyKey in a free slot; a key's first slot is the top lg bits of key * kChurnHashMul
constexpr unsigned long long kChurnHashMul = 0x9E3779B97F4A7C15ull;

// Declared weak, as in k_affinity_set.cuh: the engine's host code can be linked without these launchers (insert and erase then answer
// with an error); librio_cuda.so always links them.
//
// Inserts the m keys into the table (1 << lg slots, every slot kEmptyKey on entry, 2m <= 1 << lg), linear probing from the first slot.
// A key equal to kEmptyKey is not stored: *d_has_empty becomes 1 instead.
__attribute__((weak)) void launch_churn_build(const Launch &L, const uint64_t *d_keys, uint64_t m, unsigned long long *d_table, uint32_t lg,
                                              uint32_t *d_has_empty);
// One pass over the set's n rows: d_flag[i] = 1 if keys[i] is in the table (kEmptyKey: if *d_has_empty), else 0.  With d_counters
// (nullable), every flagged row whose idx is below n_total takes 1 from that node's counter.  d_block_cnt[b] = the flagged rows of
// [b * kChurnRows, (b + 1) * kChurnRows) and *d_erased += all of them.
__attribute__((weak)) void launch_churn_mark(const Launch &L, const uint64_t *d_keys, const uint32_t *d_idx, uint64_t n, const unsigned long long *d_table,
                                             uint32_t lg, const uint32_t *d_has_empty, uint32_t *d_counters, uint32_t n_total, uint8_t *d_flag,
                                             uint32_t *d_block_cnt, unsigned long long *d_erased);
// From the flags and block counts of launch_churn_mark, with n_new = n - (flagged rows): d_holes[j] = the j-th flagged row below n_new
// and d_movers[j] = the j-th unflagged row at or above n_new, both in increasing row order; *d_pairs = the number of holes (= movers).
// d_hole_off and d_mover_off (one entry per block each) are scratch.
__attribute__((weak)) void launch_churn_pairs(const Launch &L, const uint8_t *d_flag, uint64_t n, uint64_t n_new, const uint32_t *d_block_cnt,
                                              uint32_t *d_hole_off, uint32_t *d_mover_off, uint32_t *d_holes, uint32_t *d_movers,
                                              unsigned long long *d_pairs);
// For each j < *d_pairs (at most max_pairs): row d_movers[j] is copied over row d_holes[j] in every column -- the key, idx, the list
// row (ranks entries, d_lists nullable) and the feature row (K floats, d_feats nullable).
__attribute__((weak)) void launch_churn_move(const Launch &L, const uint32_t *d_holes, const uint32_t *d_movers, uint64_t max_pairs,
                                             const unsigned long long *d_pairs, uint64_t *d_keys, uint32_t *d_idx, uint32_t *d_lists, uint32_t ranks,
                                             float *d_feats, uint32_t K);

}  // namespace rio

// k_affinity_set.cuh -- launchers of the affinity resident sets (DESIGN.md 3.15): ranked and failure-domain affinity lists of a set
// brought up to date by one change-set pass (k_affinity_set.cu).  The S1 rows are recomputed by the ranked or failure-domain affinity
// launchers of the path the set recorded and written back by launch_scatter_ranked.
#pragma once
#include "kernels.cuh"
#include "k_changes.cuh"
#include "k_affinity_ranked.cuh"

namespace rio {

// Declared weak, as in k_ranked_changes.cuh: the engine's host code can be linked without these launchers (the affinity-set calls then
// answer with an error); librio_cuda.so always links them.  d_lists, d_idx and d_counters as in k_ranked_changes.cuh.
//
// One pass over the lists, one thread per object.  cs is the affinity change set of 3.15 (REPLACE: not live, refeatured or, for
// failure-domain lists, relabelled; CANDIDATES: joined, refeatured or relabelled).  A list with a member in REPLACE or past the table,
// or with no member at all, is S1: the object is appended to d_sel and its row left alone.  Any other list becomes the first `ranks`
// entries of itself u CANDIDATES in (fp32 cost, node index) order, cost = -sum_k fmaf(F_obj[i,k], F_node[j,k]) for k = 0..K-1 from 0,
// or with d_ndom (dense domain id per interned index at the current labels) the first `ranks` domain representatives of that union.
// Only changed rows are written; d_moved counts rows whose column 0 changed, d_changed rows that changed at all.  d_fobj (n x K) is
// read only when cs.n_cand > 0, and then only for S2 rows.
__attribute__((weak)) void launch_rebalance_changes_affinity(const Launch &L, const float *d_fobj, uint32_t K, uint32_t *d_lists, uint32_t ranks, uint32_t *d_idx,
                                                             uint64_t n, const float *d_fnode, uint32_t n_total, const ChangeSetDev &cs,
                                                             const uint32_t *d_ndom /*nullable: ranked lists*/, uint32_t *d_counters, uint32_t *d_sel,
                                                             unsigned long long *d_nsel, unsigned long long *d_moved, unsigned long long *d_changed);
// d_out (n_sel x K) = the rows d_sel names of d_rows (n x K): the selected objects' features for the S1 recomputation
__attribute__((weak)) void launch_gather_rows(const Launch &L, const float *d_rows, uint32_t K, const uint32_t *d_sel, uint64_t n_sel, float *d_out);

}  // namespace rio

// k_set_bounded_affinity.cuh -- launchers of the change-set pass of a bounded-load affinity set (DESIGN.md 3.17): pass 0 works in place
// on the set's idx and counters; its S1 objects are then re-placed by the affinity launcher of the recorded path (launch_gather_rows,
// launch_scatter_idx) and the capacity rounds of 3.16 run from the counters it leaves.
#pragma once
#include "kernels.cuh"
#include "k_changes.cuh"

namespace rio {

// Declared weak, as in k_affinity_set.cuh: the engine's host code can be linked without these launchers (the call then answers with an
// error); librio_cuda.so always links them.
//
// One pass over idx (n), one thread per object; cs is the affinity change set of 3.15 (REPLACE: not live or refeatured; CANDIDATES:
// joined or refeatured).  d_prev[i] = the node object i held before the pass.  An object whose node y is NONE, past the table or in
// REPLACE is S1: appended to d_sel, its idx left alone and y's counter (if y is interned) decremented.  Any other object moves to the
// first node of {y} u CANDIDATES in (fp32 cost, node index) order, cost = -sum_k fmaf(F_obj[i,k], F_node[j,k]) for k = 0..K-1 from 0;
// a move rewrites idx[i] and takes 1 from y's counter and adds 1 to the new node's.  d_fobj (n x K) is read only when cs.n_cand > 0,
// and then only for S2 objects.
__attribute__((weak)) void launch_rebalance_changes_bounded_affinity(const Launch &L, const float *d_fobj, uint32_t K, uint32_t *d_idx, uint32_t *d_prev,
                                                                     uint64_t n, const float *d_fnode, uint32_t n_total, const ChangeSetDev &cs,
                                                                     uint32_t *d_counters, uint32_t *d_sel, unsigned long long *d_nsel);
// *d_count += the number of i < n with d_a[i] != d_b[i]
__attribute__((weak)) void launch_count_diff(const Launch &L, const uint32_t *d_a, const uint32_t *d_b, uint64_t n, unsigned long long *d_count);

}  // namespace rio

// k_bounded_weighted.cuh -- launchers of weighted bounded-load placement (DESIGN.md 3.19): the capacity rounds of 3.5 / 3.16 over
// per-object loads (a u32 weight per row) instead of object counts.  The exchange, the capacity check, the closed set and the spill
// hash are those of 3.5; what is new is how a load is summed, how a spill takes its weight off its node, and how a re-placed object
// puts it back.
#pragma once
#include "kernels.cuh"

namespace rio {

// Declared weak, as in k_set_churn.cuh: the engine's host code can be linked without these launchers (the weighted calls and set_loads
// then answer with an error, and erase refuses a set with a weight column); librio_cuda.so always links them.
//
// *d_sum += the sum of d_w[0..n) (u64).
__attribute__((weak)) void launch_weight_sum(const Launch &L, const uint32_t *d_w, uint64_t n, unsigned long long *d_sum);
// d_loads[idx[i]] += w[i] for every i < n with idx[i] < n_total; d_w == nullptr: every weight is 1.
__attribute__((weak)) void launch_load_histogram(const Launch &L, const uint32_t *d_idx, const uint32_t *d_w, uint64_t n, uint32_t *d_loads, uint32_t n_total);
// launch_select_spill with weights: object i spills iff idx[i] is over (d_over), w[i] > 0 and spill_hash(key, round) < thr[idx[i]]; a
// spilled object is appended to d_sel (*d_nsel counts them) and its weight taken off d_loads[idx[i]].  d_w == nullptr: every weight is 1.
__attribute__((weak)) void launch_select_spill_weighted(const Launch &L, const uint64_t *d_keys, const uint32_t *d_idx, const uint32_t *d_w, uint64_t n,
                                                        const uint32_t *d_thr, const uint8_t *d_over, uint32_t round, uint32_t *d_sel,
                                                        unsigned long long *d_nsel, uint32_t *d_loads);
// After a round's re-placement: d_loads[idx[sel[t]]] += w[sel[t]] for every t < n_sel whose new node is below n_total.
__attribute__((weak)) void launch_add_loads_sel(const Launch &L, const uint32_t *d_sel, uint64_t n_sel, const uint32_t *d_idx, const uint32_t *d_w,
                                                uint32_t *d_loads, uint32_t n_total);
// The weight column of set_erase: for each j < *d_pairs (at most max_pairs), d_w[d_holes[j]] = d_w[d_movers[j]], over the pairing
// launch_churn_pairs wrote.
__attribute__((weak)) void launch_churn_move_weights(const Launch &L, const uint32_t *d_holes, const uint32_t *d_movers, uint64_t max_pairs,
                                                     const unsigned long long *d_pairs, uint32_t *d_w);

}  // namespace rio

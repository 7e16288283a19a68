// bounded_weighted_launchers.cpp -- TEST INFRASTRUCTURE: host restatements of the launchers declared in csrc/k_bounded_weighted.cuh,
// linked beside launchers.cpp and the other doubles by tests/test_gpu_set_bounded_weighted.py so that the weighted bounded calls,
// set_loads and erase on a set with a weight column run without a GPU.
//
// Like launchers.cpp: each function does, sequentially and in the plainest way, what the launcher is SPECIFIED to do (DESIGN.md 3.19).
// Nothing here says anything about the kernels.
#include "../../../rio_rs_b200/csrc/k_bounded_weighted.cuh"
#include "../../../rio_rs_b200/csrc/spec.cuh"

namespace rio {

static uint32_t weight_of(const uint32_t *w, uint64_t i) { return w ? w[i] : 1u; }

void launch_weight_sum(const Launch &L, const uint32_t *w, uint64_t n, unsigned long long *sum) {
    if (!n) return;
    for (uint64_t i = 0; i < n; i++) *sum += w[i];
    if (L.launch_counter) ++*L.launch_counter;
}

void launch_load_histogram(const Launch &L, const uint32_t *idx, const uint32_t *w, uint64_t n, uint32_t *loads, uint32_t n_total) {
    if (!n) return;
    for (uint64_t i = 0; i < n; i++)
        if (idx[i] < n_total) loads[idx[i]] += weight_of(w, i);
    if (L.launch_counter) ++*L.launch_counter;
}

void launch_select_spill_weighted(const Launch &L, const uint64_t *keys, const uint32_t *idx, const uint32_t *w, uint64_t n, const uint32_t *thr,
                                  const uint8_t *over, uint32_t round, uint32_t *sel, unsigned long long *nsel, uint32_t *loads) {
    if (!n) return;
    for (uint64_t i = 0; i < n; i++) {
        const uint32_t j = idx[i];
        if (j == kNone || !over[j] || !weight_of(w, i) || spill_hash(keys[i], round) >= thr[j]) continue;
        sel[(*nsel)++] = (uint32_t)i;
        if (loads) loads[j] -= weight_of(w, i);
    }
    if (L.launch_counter) ++*L.launch_counter;
}

void launch_add_loads_sel(const Launch &L, const uint32_t *sel, uint64_t n_sel, const uint32_t *idx, const uint32_t *w, uint32_t *loads, uint32_t n_total) {
    if (!n_sel) return;
    for (uint64_t t = 0; t < n_sel; t++)
        if (idx[sel[t]] < n_total) loads[idx[sel[t]]] += weight_of(w, sel[t]);
    if (L.launch_counter) ++*L.launch_counter;
}

void launch_churn_move_weights(const Launch &L, const uint32_t *holes, const uint32_t *movers, uint64_t max_pairs, const unsigned long long *pairs,
                               uint32_t *w) {
    if (!max_pairs) return;
    for (uint64_t j = 0; j < *pairs; j++) w[holes[j]] = w[movers[j]];
    if (L.launch_counter) ++*L.launch_counter;
}

}  // namespace rio

// set_weighted_changes_launchers.cpp -- TEST INFRASTRUCTURE: host restatements of the launchers declared in
// csrc/k_set_weighted_changes.cuh, linked beside launchers.cpp and the other doubles by tests/test_gpu_set_bounded_weighted_changes.py so
// that rio_cuda_set_write_weights_by_key and rio_cuda_set_rebalance_changes_bounded_weighted run without a GPU.
//
// Like launchers.cpp: each function does, sequentially and in the plainest way, what the launcher is SPECIFIED to do (DESIGN.md 3.21):
// the table of k_set_weighted_changes.cuh, linear probing from the first slot k_set_churn.cuh defines.  Nothing here says anything about
// the kernels.
#include "../../../rio_rs_b200/csrc/k_set_weighted_changes.cuh"
#include "../../../rio_rs_b200/csrc/k_set_churn.cuh"
#include "../../../rio_rs_b200/csrc/spec.cuh"

namespace rio {

static uint64_t first_slot(uint64_t key, uint32_t lg) { return (key * kChurnHashMul) >> (64 - lg); }

void launch_weight_keys_build(const Launch &L, const uint64_t *keys, uint64_t m, unsigned long long *table, uint32_t *pos, uint32_t lg, uint32_t *empty_pos) {
    if (!m) return;
    const uint64_t mask = (1ull << lg) - 1;
    for (uint64_t j = 0; j < m; j++) {
        if (keys[j] == kEmptyKey) { *empty_pos = (uint32_t)j + 1; continue; }
        uint64_t s = first_slot(keys[j], lg);
        while (table[s] != kEmptyKey && table[s] != keys[j]) s = (s + 1) & mask;
        table[s] = keys[j];
        pos[s] = (uint32_t)j;
    }
    if (L.launch_counter) ++*L.launch_counter;
}

void launch_weight_keys_apply(const Launch &L, const uint64_t *keys, uint64_t n, const unsigned long long *table, const uint32_t *pos, uint32_t lg,
                              const uint32_t *empty_pos, const uint32_t *w, uint32_t *weights, unsigned long long *written) {
    if (!n) return;
    const uint64_t mask = (1ull << lg) - 1;
    for (uint64_t i = 0; i < n; i++) {
        if (keys[i] == kEmptyKey) {
            if (*empty_pos) { weights[i] = w[*empty_pos - 1]; ++*written; }
            continue;
        }
        for (uint64_t s = first_slot(keys[i], lg); table[s] != kEmptyKey; s = (s + 1) & mask)
            if (table[s] == keys[i]) { weights[i] = w[pos[s]]; ++*written; break; }
    }
    if (L.launch_counter) ++*L.launch_counter;
}

void launch_merge_walk_changes(const Launch &L, uint32_t *idx, const uint32_t *walk, uint64_t n, const uint8_t *flag, uint32_t n_total) {
    if (!n) return;
    for (uint64_t i = 0; i < n; i++) {
        const uint32_t y = idx[i], f = walk[i];
        const bool s1 = y >= n_total || (flag[y] & kChgReplace);
        if (s1 || (f < n_total && (flag[f] & kChgCandidate))) idx[i] = f;
    }
    if (L.launch_counter) ++*L.launch_counter;
}

}  // namespace rio

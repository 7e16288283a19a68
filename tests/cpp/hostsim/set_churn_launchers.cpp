// set_churn_launchers.cpp -- TEST INFRASTRUCTURE: host restatements of the launchers declared in csrc/k_set_churn.cuh, linked beside
// launchers.cpp and the other doubles by tests/test_gpu_set_churn.py so that rio_cuda_set_insert and rio_cuda_set_erase run without a
// GPU.
//
// Like launchers.cpp: each function does, sequentially and in the plainest way, what the launcher is SPECIFIED to do (DESIGN.md 3.18).
// Nothing here says anything about the kernels.
#include "../../../rio_rs_b200/csrc/k_set_churn.cuh"
#include "../../../rio_rs_b200/csrc/spec.cuh"

namespace rio {

static uint64_t first_slot(unsigned long long key, uint32_t lg) { return (key * kChurnHashMul) >> (64 - lg); }

static bool in_table(const unsigned long long *table, uint32_t lg, unsigned long long key) {
    const uint64_t mask = (1ull << lg) - 1;
    for (uint64_t s = first_slot(key, lg);; s = (s + 1) & mask) {
        if (table[s] == key) return true;
        if (table[s] == kEmptyKey) return false;
    }
}

void launch_churn_build(const Launch &L, const uint64_t *keys, uint64_t m, unsigned long long *table, uint32_t lg, uint32_t *has_empty) {
    if (!m) return;
    const uint64_t mask = (1ull << lg) - 1;
    for (uint64_t t = 0; t < m; t++) {
        if (keys[t] == kEmptyKey) { *has_empty = 1; continue; }
        uint64_t s = first_slot(keys[t], lg);
        while (table[s] != kEmptyKey && table[s] != keys[t]) s = (s + 1) & mask;
        table[s] = keys[t];
    }
    if (L.launch_counter) ++*L.launch_counter;
}

void launch_churn_mark(const Launch &L, const uint64_t *keys, const uint32_t *idx, uint64_t n, const unsigned long long *table, uint32_t lg,
                       const uint32_t *has_empty, uint32_t *counters, uint32_t n_total, uint8_t *flag, uint32_t *block_cnt, unsigned long long *erased) {
    if (!n) return;
    for (uint64_t b = 0; b * kChurnRows < n; b++) block_cnt[b] = 0;
    for (uint64_t i = 0; i < n; i++) {
        const bool hit = keys[i] == kEmptyKey ? *has_empty != 0 : in_table(table, lg, keys[i]);
        flag[i] = hit ? 1 : 0;
        if (!hit) continue;
        block_cnt[i / kChurnRows]++;
        ++*erased;
        if (counters && idx[i] < n_total) counters[idx[i]]--;
    }
    if (L.launch_counter) ++*L.launch_counter;
}

void launch_churn_pairs(const Launch &L, const uint8_t *flag, uint64_t n, uint64_t n_new, const uint32_t *, uint32_t *, uint32_t *, uint32_t *holes,
                        uint32_t *movers, unsigned long long *pairs) {
    if (!n) return;
    uint64_t nh = 0, nm = 0;
    for (uint64_t i = 0; i < n; i++) {
        if (i < n_new && flag[i]) holes[nh++] = (uint32_t)i;
        if (i >= n_new && !flag[i]) movers[nm++] = (uint32_t)i;
    }
    *pairs = nh;
    if (L.launch_counter) *L.launch_counter += 2;
}

void launch_churn_move(const Launch &L, const uint32_t *holes, const uint32_t *movers, uint64_t max_pairs, const unsigned long long *pairs, uint64_t *keys,
                       uint32_t *idx, uint32_t *lists, uint32_t ranks, float *feats, uint32_t K) {
    if (!max_pairs) return;
    for (uint64_t j = 0; j < *pairs; j++) {
        const uint64_t h = holes[j], s = movers[j];
        keys[h] = keys[s];
        idx[h] = idx[s];
        for (uint32_t r = 0; lists && r < ranks; r++) lists[h * ranks + r] = lists[s * ranks + r];
        for (uint32_t k = 0; feats && k < K; k++) feats[h * K + k] = feats[s * K + k];
    }
    if (L.launch_counter) ++*L.launch_counter;
}

}  // namespace rio

// set_bounded_affinity_launchers.cpp -- TEST INFRASTRUCTURE: host restatements of the launchers declared in
// csrc/k_set_bounded_affinity.cuh, linked beside launchers.cpp and the affinity-set and bounded-affinity doubles by
// tests/test_gpu_set_bounded_affinity.py so that rio_cuda_set_rebalance_changes_bounded_affinity runs without a GPU.
//
// Like launchers.cpp: each function does, sequentially and in the plainest way, what the kernel is SPECIFIED to do (DESIGN.md 3.17);
// the costs are summed with std::fmaf in k order, as the affinity doubles sum them.  Nothing here says anything about the kernels.
#include <cmath>

#include "../../../rio_rs_b200/csrc/k_set_bounded_affinity.cuh"
#include "../../../rio_rs_b200/csrc/spec.cuh"

namespace rio {

static float cost(const float *fo, const float *fn, uint32_t K) {
    float acc = 0.f;
    for (uint32_t k = 0; k < K; k++) acc = std::fmaf(fo[k], fn[k], acc);
    return -acc;
}

// S1 (node NONE, past the table or in REPLACE): selected, its node's counter decremented.  Otherwise the first of {y} u CANDIDATES in
// (cost, index) order; a move rewrites idx and both counters.
void launch_rebalance_changes_bounded_affinity(const Launch &L, const float *fobj, uint32_t K, uint32_t *idx, uint32_t *prev, uint64_t n,
                                               const float *fnode, uint32_t n_total, const ChangeSetDev &cs, uint32_t *counters, uint32_t *sel,
                                               unsigned long long *nsel) {
    if (!n) return;
    for (uint64_t i = 0; i < n; i++) {
        const uint32_t y = idx[i];
        prev[i] = y;
        if (y >= n_total || (cs.flag[y] & kChgReplace)) {
            if (y < n_total) counters[y]--;
            sel[(*nsel)++] = (uint32_t)i;
            continue;
        }
        float bc = cost(fobj + i * K, fnode + (size_t)y * K, K);
        uint32_t bj = y;
        for (uint32_t q = 0; q < cs.n_cand; q++) {
            const uint32_t j = cs.cand[q];
            const float c = cost(fobj + i * K, fnode + (size_t)j * K, K);
            if (c < bc || (c == bc && j < bj)) { bc = c; bj = j; }
        }
        if (bj != y) {
            counters[y]--;
            counters[bj]++;
            idx[i] = bj;
        }
    }
    if (L.launch_counter) ++*L.launch_counter;
}

void launch_count_diff(const Launch &L, const uint32_t *a, const uint32_t *b, uint64_t n, unsigned long long *count) {
    if (!n) return;
    for (uint64_t i = 0; i < n; i++) *count += a[i] != b[i];
    if (L.launch_counter) ++*L.launch_counter;
}

}  // namespace rio

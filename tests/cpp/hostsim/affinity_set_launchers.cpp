// affinity_set_launchers.cpp -- TEST INFRASTRUCTURE: host restatements of the affinity-set launchers declared in
// csrc/k_affinity_set.cuh, linked beside launchers.cpp and the ranked, ranked-set, spread, spread-set and affinity doubles by
// tests/test_gpu_set_affinity.py so that the affinity-set entry points of csrc/engine.cu run without a GPU.
//
// Like launchers.cpp: each function does, sequentially and in the plainest way, what the kernel is SPECIFIED to do (DESIGN.md 3.15);
// the costs are summed exactly as launchers.cpp's launch_assign_affinity sums them, so an S2 row is what the affinity doubles would
// list.  Nothing here says anything about the kernels, which are proven on the GPU against the fp64 oracle.
#include <algorithm>
#include <tuple>
#include <vector>

#include "../../../rio_rs_b200/csrc/k_affinity_set.cuh"
#include "../../../rio_rs_b200/csrc/spec.cuh"

namespace rio {

// S1 (a member in REPLACE or past the table, or no member): selected.  S2: L u CANDIDATES costed, sorted by (cost, node index), and the
// first `ranks` kept (with ndom: the first node of each domain, up to `ranks` of them); the row written only if it changed.
void launch_rebalance_changes_affinity(const Launch &L, const float *fobj, uint32_t K, uint32_t *lists, uint32_t ranks, uint32_t *idx, uint64_t n,
                                       const float *fnode, uint32_t n_total, const ChangeSetDev &cs, const uint32_t *ndom, uint32_t *counters,
                                       uint32_t *sel, unsigned long long *nsel, unsigned long long *moved, unsigned long long *changed) {
    if (!n) return;
    for (uint64_t i = 0; i < n; i++) {
        uint32_t *row = lists + i * ranks;
        bool s1 = row[0] == kNone;
        for (uint32_t x = 0; x < ranks; x++) s1 |= row[x] != kNone && (row[x] >= n_total || (cs.flag[row[x]] & kChgReplace));
        if (s1) { sel[(*nsel)++] = (uint32_t)i; continue; }
        if (!cs.n_cand) continue;
        std::vector<uint32_t> nodes;
        for (uint32_t x = 0; x < ranks; x++) if (row[x] != kNone) nodes.push_back(row[x]);
        for (uint32_t q = 0; q < cs.n_cand; q++) if (std::find(nodes.begin(), nodes.end(), cs.cand[q]) == nodes.end()) nodes.push_back(cs.cand[q]);
        std::vector<std::tuple<float, uint32_t>> c;
        for (uint32_t j : nodes) {
            float acc = 0.f;
            for (uint32_t k = 0; k < K; k++) acc += fobj[i * K + k] * fnode[(size_t)j * K + k];
            c.emplace_back(-acc, j);
        }
        std::sort(c.begin(), c.end());
        std::vector<uint32_t> fresh;
        for (const auto &e : c) {
            if (fresh.size() == ranks) break;
            const uint32_t j = std::get<1>(e);
            bool seen = false;
            if (ndom) for (uint32_t x : fresh) seen |= ndom[x] == ndom[j];
            if (!seen) fresh.push_back(j);
        }
        fresh.resize(ranks, kNone);
        if (std::equal(fresh.begin(), fresh.end(), row)) continue;
        ++*changed;
        if (fresh[0] != row[0]) {
            ++*moved;
            if (counters && row[0] < n_total) counters[row[0]]--;
            if (counters && fresh[0] < n_total) counters[fresh[0]]++;
            idx[i] = fresh[0];
        }
        std::copy(fresh.begin(), fresh.end(), row);
    }
    if (L.launch_counter) ++*L.launch_counter;
}

void launch_gather_rows(const Launch &L, const float *rows, uint32_t K, const uint32_t *sel, uint64_t n_sel, float *out) {
    if (!n_sel) return;
    for (uint64_t i = 0; i < n_sel; i++) std::copy(rows + (size_t)sel[i] * K, rows + ((size_t)sel[i] + 1) * K, out + i * K);
    if (L.launch_counter) ++*L.launch_counter;
}

}  // namespace rio

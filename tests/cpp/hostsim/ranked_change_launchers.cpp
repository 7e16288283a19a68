// ranked_change_launchers.cpp -- TEST INFRASTRUCTURE: host restatements of the ranked-set launchers declared in
// csrc/k_ranked_changes.cuh, linked beside launchers.cpp, ranked_launchers.cpp and change_launchers.cpp by
// tests/test_gpu_set_ranked.py so that the ranked-set entry points of csrc/engine.cu run without a GPU.
//
// Like launchers.cpp: each function does, sequentially and in the plainest way, what the kernel is SPECIFIED to do (DESIGN.md 3.11) on
// the tables the engine builds; it says nothing about the kernels, which are proven on the GPU against the oracle.  The HRW2 compare
// mode walks through the restated launch_assign_trie_ranked of ranked_launchers.cpp.
#include <algorithm>
#include <vector>

#include "../../../rio_rs_b200/csrc/k_ranked_changes.cuh"
#include "../../../rio_rs_b200/csrc/spec.cuh"

namespace rio {

namespace {

inline void count(const Launch &L) { if (L.launch_counter) ++*L.launch_counter; }

// write `fresh` over row o of the lists when it differs; the primary index and counters follow column 0
void write_row(uint64_t o, const uint32_t *fresh, uint32_t ranks, uint32_t *lists, uint32_t *idx, uint32_t *counters, uint32_t n_total,
               unsigned long long *moved, unsigned long long *changed) {
    uint32_t *row = lists + o * ranks;
    if (std::equal(fresh, fresh + ranks, row)) return;
    ++*changed;
    if (fresh[0] != row[0]) {
        ++*moved;
        if (counters && row[0] < n_total) counters[row[0]]--;
        if (counters && fresh[0] < n_total) counters[fresh[0]]++;
        idx[o] = fresh[0];
    }
    std::copy(fresh, fresh + ranks, row);
}

}  // namespace

void launch_ranked_primary(const Launch &L, const uint32_t *lists, uint64_t n, uint32_t ranks, uint32_t *idx) {
    if (!n) return;
    for (uint64_t i = 0; i < n; i++) idx[i] = lists[i * ranks];
    count(L);
}

// S1 (a member not live now or lost weight, or past the table): selected.  S2: the first `ranks` nodes of L u CANDIDATES, every one
// scored at the current weights and sorted under the order (E(u) r, ~u, j) of 3.4.
void launch_rebalance_changes_ranked(const Launch &L, const uint64_t *keys, uint32_t *lists, uint32_t ranks, uint32_t *idx, uint64_t n, const NodeTabDev &tab,
                                     const ChangeSetDev &cs, uint32_t *counters, uint32_t *sel, unsigned long long *nsel, unsigned long long *moved,
                                     unsigned long long *changed) {
    if (!n) return;
    struct Cand { uint64_t s; uint32_t u, j; };
    for (uint64_t i = 0; i < n; i++) {
        const uint32_t *row = lists + i * ranks;
        bool s1 = false;
        for (uint32_t x = 0; x < ranks; x++) s1 |= row[x] != kNone && (row[x] >= tab.n_total || (cs.flag[row[x]] & kChgReplace));
        if (s1) { sel[(*nsel)++] = (uint32_t)i; continue; }
        std::vector<uint32_t> nodes;
        for (uint32_t x = 0; x < ranks; x++) if (row[x] != kNone) nodes.push_back(row[x]);
        for (uint32_t q = 0; q < cs.n_cand; q++) if (std::find(nodes.begin(), nodes.end(), cs.cand[q]) == nodes.end()) nodes.push_back(cs.cand[q]);
        const ObjHash o = obj_hash(keys[i]);
        std::vector<Cand> c;
        for (uint32_t j : nodes) {
            const uint4 r = tab.by_idx[j];
            const uint32_t u = pair_hash(o, r.x, r.z, r.w);
            c.push_back(Cand{(uint64_t)elog(u) * r.y, u, j});
        }
        std::sort(c.begin(), c.end(), [](const Cand &a, const Cand &b) { return cand_better(a.s, a.u, a.j, b.s, b.u, b.j); });
        std::vector<uint32_t> fresh(ranks, kNone);
        for (uint32_t x = 0; x < ranks && x < c.size(); x++) fresh[x] = c[x].j;
        write_row(i, fresh.data(), ranks, lists, idx, counters, tab.n_total, moved, changed);
    }
    count(L);
}

void launch_scatter_ranked(const Launch &L, const uint32_t *fresh, const uint32_t *sel, uint64_t n_sel, uint32_t ranks, uint32_t *lists, uint32_t *idx,
                           uint32_t *counters, uint32_t n_total, unsigned long long *moved, unsigned long long *changed) {
    if (!n_sel) return;
    for (uint64_t i = 0; i < n_sel; i++) write_row(sel[i], fresh + i * ranks, ranks, lists, idx, counters, n_total, moved, changed);
    count(L);
}

void launch_reassign_trie_ranked(const Launch &L, const uint64_t *keys, uint64_t n, const TrieDev &t, const TrieRankDev &rk, uint32_t ranks, uint32_t *lists,
                                 uint32_t *idx, uint32_t *counters, uint32_t n_total, unsigned long long *moved, unsigned long long *changed) {
    if (!n) return;
    std::vector<uint32_t> fresh((size_t)n * ranks);
    Launch quiet = L;
    quiet.launch_counter = nullptr;
    launch_assign_trie_ranked(quiet, keys, n, t, rk, ranks, fresh.data());
    for (uint64_t i = 0; i < n; i++) write_row(i, fresh.data() + i * ranks, ranks, lists, idx, counters, n_total, moved, changed);
    count(L);
}

}  // namespace rio

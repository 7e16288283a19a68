// spread_change_launchers.cpp -- TEST INFRASTRUCTURE: host restatements of the spread-set launchers declared in
// csrc/k_spread_changes.cuh, linked beside launchers.cpp, ranked_launchers.cpp, change_launchers.cpp, ranked_change_launchers.cpp and
// spread_launchers.cpp by tests/test_gpu_set_spread.py so that the spread-set entry points of csrc/engine.cu run without a GPU.
//
// Like launchers.cpp: each function does, sequentially and in the plainest way, what the kernel is SPECIFIED to do (DESIGN.md 3.13) on
// the tables the engine builds; it says nothing about the kernels, which are proven on the GPU against the oracle.  The HRW2 compare
// mode walks through the restated launch_assign_trie_spread of spread_launchers.cpp.
#include <algorithm>
#include <vector>

#include "../../../rio_rs_b200/csrc/k_spread_changes.cuh"
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

// S1 (a member in REPLACE or past the table): selected.  S2: L u CANDIDATES scored at the current weights, sorted under the order
// (E(u) r, ~u, j) of 3.4, and the first node of each dense domain kept, up to `ranks` of them.
void launch_rebalance_changes_spread(const Launch &L, const uint64_t *keys, uint32_t *lists, uint32_t ranks, uint32_t *idx, uint64_t n, const NodeTabDev &tab,
                                     const ChangeSetDev &cs, const SpreadTabDev &sp, uint32_t *counters, uint32_t *sel, unsigned long long *nsel,
                                     unsigned long long *moved, unsigned long long *changed) {
    if (!n) return;
    const uint32_t *ndom = reinterpret_cast<const uint32_t *>(sp.base + sp.o_ndom);
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
        std::vector<uint32_t> fresh, doms;
        for (const Cand &e : c) {
            if (fresh.size() == ranks) break;
            if (std::find(doms.begin(), doms.end(), ndom[e.j]) != doms.end()) continue;
            fresh.push_back(e.j);
            doms.push_back(ndom[e.j]);
        }
        fresh.resize(ranks, kNone);
        write_row(i, fresh.data(), ranks, lists, idx, counters, tab.n_total, moved, changed);
    }
    count(L);
}

void launch_reassign_trie_spread(const Launch &L, const uint64_t *keys, uint64_t n, const TrieDev &t, const SpreadTabDev &sp, uint32_t ranks, uint32_t *lists,
                                 uint32_t *idx, uint32_t *counters, uint32_t n_total, unsigned long long *moved, unsigned long long *changed) {
    if (!n) return;
    std::vector<uint32_t> fresh((size_t)n * ranks);
    Launch quiet = L;
    quiet.launch_counter = nullptr;
    launch_assign_trie_spread(quiet, keys, n, t, sp, ranks, fresh.data());
    for (uint64_t i = 0; i < n; i++) write_row(i, fresh.data() + i * ranks, ranks, lists, idx, counters, n_total, moved, changed);
    count(L);
}

}  // namespace rio

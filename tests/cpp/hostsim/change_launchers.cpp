// change_launchers.cpp -- TEST INFRASTRUCTURE: host restatements of the change-set launchers declared in csrc/k_changes.cuh, linked
// beside launchers.cpp by tests/test_gpu_rebalance_changes.py so that the change-set entry points of csrc/engine.cu run without a GPU.
//
// Like launchers.cpp: each function does, sequentially and in the plainest way, what the kernel is SPECIFIED to do (DESIGN.md 3.10) on
// the tables the engine builds; it says nothing about the kernels, which are proven on the GPU against the oracle.
#include "../../../rio_rs_b200/csrc/k_changes.cuh"
#include "../../../rio_rs_b200/csrc/spec.cuh"

namespace rio {

namespace {

inline void count(const Launch &L) { if (L.launch_counter) ++*L.launch_counter; }

uint32_t node_of(const DirSlot &s) { return (uint32_t)s.val; }

// the best node of {cur} u CANDIDATES under the order (E(u) r, ~u, j) of 3.4
uint32_t best_of(uint64_t key, uint32_t cur, const NodeTabDev &tab, const ChangeSetDev &cs) {
    const ObjHash o = obj_hash(key);
    auto score = [&](uint32_t j, uint32_t *u) { const uint4 r = tab.by_idx[j]; *u = pair_hash(o, r.x, r.z, r.w); return (uint64_t)elog(*u) * r.y; };
    uint32_t best = cur, bu;
    uint64_t bs = score(cur, &bu);
    for (uint32_t q = 0; q < cs.n_cand; q++) {
        uint32_t u;
        const uint64_t s = score(cs.cand[q], &u);
        if (cand_better(s, u, cs.cand[q], bs, bu, best)) { best = cs.cand[q]; bs = s; bu = u; }
    }
    return best;
}

bool replaced(uint32_t y, const NodeTabDev &tab, const ChangeSetDev &cs) { return y >= tab.n_total || (cs.flag[y] & kChgReplace); }

}  // namespace

void launch_dir_rebalance_changes(const Launch &L, const DirDev &dir, const NodeTabDev &tab, const ChangeSetDev &cs, uint64_t *r1_slot, uint64_t *r1_key,
                                  unsigned long long *nr1, unsigned long long *moved) {
    for (uint64_t i = 0; i <= dir.mask; i++) {
        DirSlot &s = dir.slots[i];
        const uint32_t y = node_of(s);
        if (s.key == kEmptyKey || y >= tab.n_total) continue;
        if (replaced(y, tab, cs)) { r1_slot[*nr1] = i; r1_key[*nr1] = s.key; ++*nr1; continue; }
        const uint32_t to = best_of(s.key, y, tab, cs);
        if (to != y) { s.val = (s.val & ~0xFFFFFFFFull) | to; ++*moved; }
    }
    count(L);
}

void launch_dir_scatter_changes(const Launch &L, const DirDev &dir, const uint64_t *r1_slot, const uint32_t *to, uint64_t n, unsigned long long *moved) {
    if (!n) return;
    for (uint64_t i = 0; i < n; i++) {
        DirSlot &s = dir.slots[r1_slot[i]];
        if (to[i] != node_of(s)) { s.val = (s.val & ~0xFFFFFFFFull) | to[i]; ++*moved; }
    }
    count(L);
}

void launch_rebalance_changes(const Launch &L, const uint64_t *keys, uint32_t *idx, uint64_t n, const NodeTabDev &tab, const ChangeSetDev &cs,
                              uint32_t *counters, uint32_t *sel, uint32_t *sel_old, unsigned long long *nsel, unsigned long long *moved) {
    if (!n) return;
    if (counters)
        for (uint32_t j = 0; j < tab.n_total; j++) if (cs.flag[j] & kChgReplace) counters[j] = 0;
    for (uint64_t i = 0; i < n; i++) {
        const uint32_t y = idx[i];
        if (replaced(y, tab, cs)) { sel[*nsel] = (uint32_t)i; sel_old[*nsel] = y; ++*nsel; continue; }
        const uint32_t to = best_of(keys[i], y, tab, cs);
        if (to == y) continue;
        idx[i] = to;
        ++*moved;
        if (counters) { counters[y]--; counters[to]++; }
    }
    count(L);
}

void launch_count_changed(const Launch &L, const uint32_t *idx, const uint32_t *sel, const uint32_t *sel_old, uint64_t n_sel, unsigned long long *moved) {
    if (!n_sel) return;
    for (uint64_t i = 0; i < n_sel; i++) *moved += idx[sel[i]] != sel_old[i];
    count(L);
}

}  // namespace rio

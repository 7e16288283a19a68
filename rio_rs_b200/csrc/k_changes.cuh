// k_changes.cuh -- launchers of the change-set rebalance under the flat policy (k_directory.cu, DESIGN.md 3.10).
#pragma once
#include "kernels.cuh"

namespace rio {

// What a change set does to each interned node, one byte per node, built on the host from the previous and current weights.
constexpr uint8_t kChgReplace = 1;     // not live now, or live with a grown r: its entries are re-placed over the live set (R1)
constexpr uint8_t kChgCandidate = 2;   // joined or gained weight: every other entry compares it with its incumbent (R2)
struct ChangeSetDev {
    const uint8_t *flag;     // n_total bytes (tab.n_total)
    const uint32_t *cand;    // the kChgCandidate nodes, n_cand of them
    uint32_t n_cand;
};

// Declared weak, as in k_ranked.cuh: the engine's host code can be linked without these launchers (the change-set calls then
// answer with an error under the flat policy); librio_cuda.so always links them.
//
// Directory, one pass over the slots: R2 entries are rewritten in place and counted in d_moved; R1 entries are appended to
// (d_r1_slot, d_r1_key), their number to d_nr1.  Slots with RIO_NONE or an index >= n_total are left alone, as JOIN does.
__attribute__((weak)) void launch_dir_rebalance_changes(const Launch &L, const DirDev &dir, const NodeTabDev &tab, const ChangeSetDev &cs,
                                                        uint64_t *d_r1_slot, uint64_t *d_r1_key, unsigned long long *d_nr1, unsigned long long *d_moved);
// ... then, once d_to holds the flat placement of the gathered keys: write back the nodes that changed (low word only), count them
__attribute__((weak)) void launch_dir_scatter_changes(const Launch &L, const DirDev &dir, const uint64_t *d_r1_slot, const uint32_t *d_to, uint64_t n,
                                                      unsigned long long *d_moved);
// Resident set: R2 in place (idx, counters, d_moved); R1 objects (and RIO_NONE / out-of-range ones) appended to d_sel with their
// old node in d_sel_old; the counters of kChgReplace nodes are zeroed, since every object on them is selected.  d_counters nullable.
// With cs.n_cand == 0 no entry can take the R2 branch, and the launcher runs a 4 B/object scan of idx instead of the 12 B/object pass.
__attribute__((weak)) void launch_rebalance_changes(const Launch &L, const uint64_t *d_keys, uint32_t *d_idx, uint64_t n, const NodeTabDev &tab,
                                                    const ChangeSetDev &cs, uint32_t *d_counters, uint32_t *d_sel, uint32_t *d_sel_old,
                                                    unsigned long long *d_nsel, unsigned long long *d_moved);
// after the selection was re-placed: count the selected objects whose node differs from d_sel_old
__attribute__((weak)) void launch_count_changed(const Launch &L, const uint32_t *d_idx, const uint32_t *d_sel, const uint32_t *d_sel_old, uint64_t n_sel,
                                                unsigned long long *d_moved);

}  // namespace rio

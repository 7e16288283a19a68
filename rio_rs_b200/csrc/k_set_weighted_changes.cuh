// k_set_weighted_changes.cuh -- launchers of weighted bounded sets kept within load capacity (DESIGN.md 3.21): the weight writes by
// key (a key -> position table of the written keys, then one pass over the set's keys) and the merge of the HRW2 change-set pass (each
// object against a fresh walk of its key).  The rest of the call runs on existing launchers.
#pragma once
#include "kernels.cuh"
#include "k_changes.cuh"

namespace rio {

// Declared weak, as in k_bounded_weighted.cuh: the engine's host code can be linked without these launchers (set_write_weights_by_key
// and set_rebalance_changes_bounded_weighted then answer with an error); librio_cuda.so always links them.
//
// The by-key table: 1 << lg slots (2m <= 1 << lg), d_table[s] = the key held (kEmptyKey: free, every slot on entry) and d_pos[s] its
// position in d_keys (0 on entry), linear probing from churn_slot (k_key_probe.cuh).  Each key is claimed by a 64-bit CAS and its
// position merged with atomicMax, so a key listed several times keeps its last position.  A key equal to kEmptyKey is not stored:
// *d_empty_pos (0 on entry) becomes 1 + its last position instead.
__attribute__((weak)) void launch_weight_keys_build(const Launch &L, const uint64_t *d_keys, uint64_t m, unsigned long long *d_table, uint32_t *d_pos,
                                                    uint32_t lg, uint32_t *d_empty_pos);
// One pass over the set's n rows: a row whose key is in the table gets d_weights[i] = d_w[position]; *d_written += the rows written.
__attribute__((weak)) void launch_weight_keys_apply(const Launch &L, const uint64_t *d_set_keys, uint64_t n, const unsigned long long *d_table,
                                                    const uint32_t *d_pos, uint32_t lg, const uint32_t *d_empty_pos, const uint32_t *d_w,
                                                    uint32_t *d_weights, unsigned long long *d_written);
// The HRW2 change-set pass with candidates: d_walk[i] is object i's walk over the live set.  Object i with node y = d_idx[i] takes
// d_walk[i] if y is RIO_NONE, past n_total or kChgReplace (S1), or if d_walk[i] is a kChgCandidate node (S2); otherwise it keeps y.
// Only rows whose node changes are written.  d_flag holds n_total bytes.
__attribute__((weak)) void launch_merge_walk_changes(const Launch &L, uint32_t *d_idx, const uint32_t *d_walk, uint64_t n, const uint8_t *d_flag,
                                                     uint32_t n_total);

}  // namespace rio

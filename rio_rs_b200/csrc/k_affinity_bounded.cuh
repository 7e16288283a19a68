// k_affinity_bounded.cuh -- launcher of the bounded-load affinity rounds (DESIGN.md 3.16): a spill round gathers the spilled objects'
// feature rows (launch_gather_rows), places them with the affinity launcher of the call's path over the open nodes, and writes the
// new nodes back with launch_scatter_idx.
#pragma once
#include "kernels.cuh"

namespace rio {

// Declared weak, as in k_affinity_set.cuh: the engine's host code can be linked without this launcher (the bounded affinity calls then
// answer with an error); librio_cuda.so always links it.
//
// d_idx[d_sel[i]] = d_vals[i] for i < n_sel.  The counters are not touched: the spill selection took the objects off their old nodes
// and the affinity launch that produced d_vals added them to their new ones.
__attribute__((weak)) void launch_scatter_idx(const Launch &L, const uint32_t *d_vals, const uint32_t *d_sel, uint64_t n_sel, uint32_t *d_idx);

}  // namespace rio

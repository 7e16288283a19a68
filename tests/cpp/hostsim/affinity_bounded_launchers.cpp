// affinity_bounded_launchers.cpp -- TEST INFRASTRUCTURE: host restatement of the launcher declared in csrc/k_affinity_bounded.cuh,
// linked beside launchers.cpp and the affinity-set doubles (for launch_gather_rows) by tests/test_gpu_bounded_affinity.py so that the
// bounded affinity entry points of csrc/engine.cu run without a GPU.  Like launchers.cpp: it does, sequentially and in the plainest
// way, what the kernel is SPECIFIED to do (DESIGN.md 3.16), and says nothing about the kernel.
#include "../../../rio_rs_b200/csrc/k_affinity_bounded.cuh"

namespace rio {

void launch_scatter_idx(const Launch &L, const uint32_t *vals, const uint32_t *sel, uint64_t n_sel, uint32_t *idx) {
    if (!n_sel) return;
    for (uint64_t i = 0; i < n_sel; i++) idx[sel[i]] = vals[i];
    if (L.launch_counter) ++*L.launch_counter;
}

}  // namespace rio

// affinity_ranked_launchers.cpp -- TEST INFRASTRUCTURE: host restatements of the ranked affinity launchers declared in
// csrc/k_affinity_ranked.cuh, linked beside launchers.cpp by tests/test_gpu_affinity_ranked.py so that the ranked affinity entry
// points of csrc/engine.cu run without a GPU.
//
// Like launchers.cpp: each function does, sequentially and in the plainest way, what the kernel is SPECIFIED to do (DESIGN.md 3.9);
// the costs are summed exactly as launchers.cpp's launch_assign_affinity sums them, so rank 1 is that double's answer.  Nothing here
// says anything about the kernels, which are proven on the GPU against the fp64 oracle.
#include <algorithm>
#include <utility>
#include <vector>

#include "../../../rio_rs_b200/csrc/k_affinity_ranked.cuh"
#include "../../../rio_rs_b200/csrc/spec.cuh"

namespace rio {

// the live nodes in increasing (cost, node index) order, the first `ranks` of them, kNone past the live set
void launch_assign_affinity_ranked(const Launch &L, const float *fobj, uint64_t n, const float *fnode, const uint32_t *live, uint32_t n_total, uint32_t K,
                                   uint32_t ranks, uint32_t *out) {
    if (!n) return;
    std::vector<std::pair<float, uint32_t>> c;
    for (uint64_t i = 0; i < n; i++) {
        c.clear();
        for (uint32_t j = 0; j < n_total; j++) {
            if (!live[j]) continue;
            float acc = 0.f;
            for (uint32_t k = 0; k < K; k++) acc += fobj[i * K + k] * fnode[(size_t)j * K + k];
            c.emplace_back(-acc, j);
        }
        std::sort(c.begin(), c.end());
        for (uint32_t r = 0; r < ranks; r++) out[i * ranks + r] = r < c.size() ? c[r].second : kNone;
    }
    if (L.launch_counter) ++*L.launch_counter;
}

cudaError_t launch_assign_affinity_umma_ranked(const Launch &, const float *, uint64_t, const float *, const float *, const uint32_t *, uint32_t, uint32_t,
                                               uint32_t, uint32_t *, uint32_t *) {
    return cudaErrorInvalidValue;   // never selected: launchers.cpp's affinity_umma_max_nodes() is 0
}

}  // namespace rio

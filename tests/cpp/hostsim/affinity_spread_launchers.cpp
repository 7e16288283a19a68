// affinity_spread_launchers.cpp -- TEST INFRASTRUCTURE: host restatements of the failure-domain affinity launchers declared in
// csrc/k_affinity_spread.cuh, linked beside launchers.cpp and affinity_ranked_launchers.cpp by tests/test_gpu_affinity_spread.py so
// that the failure-domain affinity entry points of csrc/engine.cu run without a GPU.
//
// Like launchers.cpp: each function does, sequentially and in the plainest way, what the kernel is SPECIFIED to do (DESIGN.md 3.14);
// the costs are summed exactly as launchers.cpp's launch_assign_affinity sums them, so rank 1 is that double's answer.  Nothing here
// says anything about the kernels, which are proven on the GPU against the fp64 oracle.
#include <algorithm>
#include <cmath>
#include <tuple>
#include <vector>

#include "../../../rio_rs_b200/csrc/k_affinity_spread.cuh"
#include "../../../rio_rs_b200/csrc/spec.cuh"

namespace rio {

// the live nodes in increasing (cost, node index) order; the first node of each domain not listed yet, `ranks` of them, kNone past
// the live domains
void launch_assign_affinity_spread(const Launch &L, const float *fobj, uint64_t n, const float *fnode, const uint32_t *live, uint32_t n_total, uint32_t K,
                                   const uint32_t *ndom, uint32_t ranks, uint32_t *out) {
    if (!n) return;
    if (hostsim_misaligned(fobj, HOSTSIM_DECLARED_ALIGN(affinity_feats_align(K)))) return;
    std::vector<std::tuple<float, uint32_t>> c;
    std::vector<uint32_t> listed;
    for (uint64_t i = 0; i < n; i++) {
        c.clear();
        for (uint32_t j = 0; j < n_total; j++) {
            if (!live[j]) continue;
            float acc = 0.f;
            for (uint32_t k = 0; k < K; k++) acc = std::fmaf(fobj[i * K + k], fnode[(size_t)j * K + k], acc);
            c.emplace_back(-acc, j);
        }
        std::sort(c.begin(), c.end());
        listed.clear();
        for (const auto &e : c) {
            if (listed.size() == ranks) break;
            const uint32_t j = std::get<1>(e);
            bool seen = false;
            for (uint32_t x : listed) seen |= ndom[x] == ndom[j];
            if (!seen) listed.push_back(j);
        }
        for (uint32_t r = 0; r < ranks; r++) out[i * ranks + r] = r < listed.size() ? listed[r] : kNone;
    }
    if (L.launch_counter) ++*L.launch_counter;
}

cudaError_t launch_assign_affinity_umma_spread(const Launch &, const float *, uint64_t, const float *, const float *, const uint32_t *, const uint32_t *,
                                               uint32_t, uint32_t, uint32_t, uint32_t *, uint32_t *) {
    return cudaErrorInvalidValue;   // never selected: launchers.cpp's affinity_umma_max_nodes() is 0
}

}  // namespace rio

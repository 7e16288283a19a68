// k_affinity_spread.cuh -- launchers of the failure-domain affinity lists (DESIGN.md 3.14): each object's `ranks` lowest-cost live
// nodes in `ranks` distinct failure domains, cost = -dot(F_obj, F_node), rank 1 the unranked answer of the same path.  The
// tensor-core pair is in k_affinity_umma.cu, the CUDA-core kernel (k_assign_affinity_ranked with SPREAD) in k_assign.cu.
#pragma once
#include "kernels.cuh"
#include "k_affinity_ranked.cuh"   // affinity_ranked_groups, kMaxRanks

namespace rio {

// d_out_idx is n x ranks row-major, ranks in [1, kMaxRanks]; RIO_NONE past the number of live domains.  Domain ids are dense: equal
// ids are one domain, and no live node has kNone.
// Declared weak, like k_affinity_ranked.cuh: engine.cu links without the kernels, and then the entry points answer with an error;
// librio_cuda.so always links them.
//
// tensor-core path, the shapes launch_assign_affinity_umma_ranked takes; d_pdom holds the domain id of every compacted position
// (m_pad entries, the order of d_nidx_map), d_cols is the n x affinity_ranked_groups(ranks) scratch of column positions
__attribute__((weak)) cudaError_t launch_assign_affinity_umma_spread(const Launch &L, const float *d_fobj, uint64_t n, const float *d_fnode_c,
                                                                     const float *d_fnode_g, const uint32_t *d_nidx_map, const uint32_t *d_pdom,
                                                                     uint32_t n_live, uint32_t m_pad, uint32_t ranks, uint32_t *d_cols,
                                                                     uint32_t *d_out_idx);
// CUDA-core path, any K; d_ndom holds the domain id of every interned index (n_total entries, kNone for nodes that are not live)
__attribute__((weak)) void launch_assign_affinity_spread(const Launch &L, const float *d_fobj, uint64_t n, const float *d_fnode, const uint32_t *d_live,
                                                         uint32_t n_total, uint32_t K, const uint32_t *d_ndom, uint32_t ranks, uint32_t *d_out_idx);

}  // namespace rio

// k_affinity_ranked.cuh -- launchers of the ranked affinity lists (DESIGN.md 3.9): each object's `ranks` lowest-cost live nodes,
// cost = -dot(F_obj, F_node), in increasing (cost, node index) order.  The tensor-core pair is in k_affinity_umma.cu, the CUDA-core
// kernel in k_assign.cu.
#pragma once
#include "kernels.cuh"
#include "k_ranked.cuh"   // kMaxRanks

namespace rio {

// Groups of 8 compacted node positions the tensor-core pass keeps per object for a list of `ranks` (1, 2, 4 or 8; the kernels are
// instantiated for these).  The scratch between the two passes holds n x affinity_ranked_groups(ranks) u32.
inline uint32_t affinity_ranked_groups(uint32_t ranks) { return ranks <= 1 ? 1u : ranks <= 2 ? 2u : ranks <= 4 ? 4u : 8u; }

// d_out_idx is n x ranks row-major, ranks in [1, kMaxRanks]; RIO_NONE pads a list longer than the live set.  Rank 1 is what the
// unranked launcher of the same path (launch_assign_affinity_umma / launch_assign_affinity) writes.
// Declared weak, like the launchers of k_ranked.cuh: engine.cu links without the kernels, and then the ranked affinity entry points
// answer with an error; librio_cuda.so always links them.
//
// tensor-core path, K == 16, the shapes launch_assign_affinity_umma takes; d_groups is the n x affinity_ranked_groups(ranks) scratch
__attribute__((weak)) cudaError_t launch_assign_affinity_umma_ranked(const Launch &L, const float *d_fobj, uint64_t n, const float *d_fnode_c,
                                                                     const float *d_fnode_g, const uint32_t *d_nidx_map, uint32_t n_live,
                                                                     uint32_t m_pad, uint32_t ranks, uint32_t *d_groups, uint32_t *d_out_idx);
// CUDA-core path, any K
__attribute__((weak)) void launch_assign_affinity_ranked(const Launch &L, const float *d_fobj, uint64_t n, const float *d_fnode, const uint32_t *d_live,
                                                         uint32_t n_total, uint32_t K, uint32_t ranks, uint32_t *d_out_idx);

}  // namespace rio

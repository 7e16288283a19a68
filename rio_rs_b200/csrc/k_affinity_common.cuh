// k_affinity_common.cuh -- what the change-set passes under the affinity cost share (k_affinity_set.cu, k_set_bounded_affinity.cu):
// the (cost, index) order, one object's fp32 cost in the fmaf order of every affinity kernel, and the shared-memory staging rule of
// DESIGN.md 3.15.
// Included by .cu files only: everything is internal to the including translation unit.
#pragma once
#include "kernels.cuh"
#include "spec.cuh"

namespace rio {

namespace {

// the most dynamic shared memory the pass is given: the flag bytes and the candidates' indices and feature rows are staged when they fit
constexpr uint32_t kAffSetSmemBudget = 96u * 1024u;

// (c, j) before (c', j'), an empty slot (j' == kNone) last: the order of k_assign_affinity_ranked's strict comparisons
__device__ __forceinline__ bool aff_before(float c, uint32_t j, float c2, uint32_t j2) { return j2 == kNone || c < c2 || (c == c2 && j < j2); }

// One object's features and its fp32 cost against a node row: the fmaf order of every affinity kernel (k = 0..K-1 from 0.f), negated.
// KC = 16 keeps the row in registers and reads node rows as float4; KC = 0 takes any K at run time.
template <int KC>
struct ObjRow {
    float f[KC ? KC : 1];
    const float *g;
    uint32_t K;
    __device__ __forceinline__ void load(const float *fobj, uint64_t i, uint32_t K_) {
        K = K_;
        g = fobj + i * K_;
        if constexpr (KC != 0) {
            const float4 *row = reinterpret_cast<const float4 *>(g);
#pragma unroll
            for (int k4 = 0; k4 < KC / 4; k4++) {
                const float4 v = __ldg(row + k4);
                f[4 * k4 + 0] = v.x; f[4 * k4 + 1] = v.y; f[4 * k4 + 2] = v.z; f[4 * k4 + 3] = v.w;
            }
        }
    }
    // node rows of the handle's table: read-only path
    __device__ __forceinline__ float cost_ro(const float *nr) const {
        float acc = 0.f;
        if constexpr (KC != 0) {
            const float4 *v4 = reinterpret_cast<const float4 *>(nr);
#pragma unroll
            for (int k4 = 0; k4 < KC / 4; k4++) {
                const float4 v = __ldg(v4 + k4);
                acc = fmaf(f[4 * k4 + 0], v.x, acc); acc = fmaf(f[4 * k4 + 1], v.y, acc);
                acc = fmaf(f[4 * k4 + 2], v.z, acc); acc = fmaf(f[4 * k4 + 3], v.w, acc);
            }
        } else {
            for (uint32_t k = 0; k < K; k++) acc = fmaf(__ldg(g + k), __ldg(nr + k), acc);
        }
        return -acc;
    }
    // candidate rows: shared memory when staged, else global memory (generic loads)
    __device__ __forceinline__ float cost(const float *nr) const {
        float acc = 0.f;
        if constexpr (KC != 0) {
            const float4 *v4 = reinterpret_cast<const float4 *>(nr);
#pragma unroll
            for (int k4 = 0; k4 < KC / 4; k4++) {
                const float4 v = v4[k4];
                acc = fmaf(f[4 * k4 + 0], v.x, acc); acc = fmaf(f[4 * k4 + 1], v.y, acc);
                acc = fmaf(f[4 * k4 + 2], v.z, acc); acc = fmaf(f[4 * k4 + 3], v.w, acc);
            }
        } else {
            for (uint32_t k = 0; k < K; k++) acc = fmaf(__ldg(g + k), nr[k], acc);
        }
        return -acc;
    }
};

// Shared-memory layout when staged: [n_cand x K fp32 candidate rows][n_cand x u32 candidates][n_total flag bytes].
inline size_t aff_changes_smem(uint32_t n_total, uint32_t n_cand, uint32_t K) {
    return (size_t)n_cand * K * 4 + (size_t)n_cand * 4 + n_total;
}

}  // namespace

}  // namespace rio

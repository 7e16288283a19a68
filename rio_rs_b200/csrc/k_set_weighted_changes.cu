// k_set_weighted_changes.cu -- weighted bounded sets kept within load capacity (DESIGN.md 3.21): the key -> position table and the
// apply pass of set_write_weights_by_key, and the merge of the HRW2 change-set pass.  In a translation unit of its own, so that no
// existing kernel's code depends on it.
#include "kernels.cuh"
#include "k_set_weighted_changes.cuh"
#include "k_key_probe.cuh"
#include "spec.cuh"

namespace rio {

namespace {

constexpr uint32_t kMergeMaxSmem = 48 * 1024;   // node flag bytes staged in shared memory up to this many nodes (no opt-in needed)

// one thread per written key; a duplicate finds its own key and merges its position
__global__ void __launch_bounds__(256)
k_weight_keys_build(const uint64_t *__restrict__ keys, uint64_t m, unsigned long long *__restrict__ table, uint32_t *__restrict__ pos, uint32_t lg,
                    uint32_t *__restrict__ empty_pos) {
    const uint64_t mask = (1ull << lg) - 1, stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < m; t += stride) {
        const unsigned long long k = __ldg(keys + t);
        if (k == kEmptyKey) { atomicMax(empty_pos, (uint32_t)t + 1); continue; }
        for (uint64_t s = churn_slot(k, lg);; s = (s + 1) & mask) {
            const unsigned long long old = atomicCAS(table + s, kEmptyKey, k);
            if (old == kEmptyKey || old == k) { atomicMax(pos + s, (uint32_t)t); break; }
        }
    }
}

// One thread per row: 8 B of key and a probe of the (L2-resident) table, 4 B of weight gathered and 4 B written per matched row, one
// atomic per warp for the count.  Whole warps run every trip, so the ballot sees every lane.
__global__ void __launch_bounds__(256)
k_weight_keys_apply(const uint64_t *__restrict__ keys, uint64_t n, const unsigned long long *__restrict__ table, const uint32_t *__restrict__ pos,
                    uint32_t lg, const uint32_t *__restrict__ empty_pos, const uint32_t *__restrict__ w, uint32_t *__restrict__ weights,
                    unsigned long long *written) {
    const uint64_t mask = (1ull << lg) - 1;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        uint32_t at = kNone;
        if (i < n) {
            const unsigned long long k = __ldg(keys + i);
            if (k == kEmptyKey) {
                const uint32_t e = __ldg(empty_pos);
                if (e) at = e - 1;
            } else {
                for (uint64_t s = churn_slot(k, lg);; s = (s + 1) & mask) {
                    const unsigned long long t = __ldg(table + s);
                    if (t == k) { at = __ldg(pos + s); break; }
                    if (t == kEmptyKey) break;
                }
            }
            if (at != kNone) weights[i] = __ldg(w + at);
        }
        const unsigned hits = __ballot_sync(0xFFFFFFFFu, at != kNone);
        if ((threadIdx.x & 31) == 0 && hits) atomicAdd(written, (unsigned long long)__popc(hits));
    }
}

// 8 B read per object, 4 B written per object that changes node; the flag bytes staged per block when they fit
template <bool SMEM>
__global__ void __launch_bounds__(256)
k_merge_walk_changes(uint32_t *__restrict__ idx, const uint32_t *__restrict__ walk, uint64_t n, const uint8_t *__restrict__ flag_in, uint32_t n_total) {
    extern __shared__ uint8_t sflag[];
    const uint8_t *flag = flag_in;
    if (SMEM) {
        for (uint32_t j = threadIdx.x; j < n_total; j += blockDim.x) sflag[j] = __ldg(flag_in + j);
        __syncthreads();
        flag = sflag;
    }
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t y = idx[i], f = __ldg(walk + i);
        if (f == y) continue;
        const bool s1 = y >= n_total || (flag[y] & kChgReplace);
        if (s1 || (f < n_total && (flag[f] & kChgCandidate))) idx[i] = f;
    }
}

int grid_of(uint64_t items, const Launch &L, int per_sm) {
    const uint64_t blocks = (items + 255) / 256, cap = (uint64_t)L.sm_count * per_sm;
    return (int)(blocks < 1 ? 1 : blocks < cap ? blocks : cap);
}

}  // namespace

void launch_weight_keys_build(const Launch &L, const uint64_t *d_keys, uint64_t m, unsigned long long *d_table, uint32_t *d_pos, uint32_t lg,
                              uint32_t *d_empty_pos) {
    if (!m) return;
    k_weight_keys_build<<<grid_of(m, L, 8), 256, 0, L.stream>>>(d_keys, m, d_table, d_pos, lg, d_empty_pos);
    RIO_COUNT_LAUNCH(L);
}

void launch_weight_keys_apply(const Launch &L, const uint64_t *d_set_keys, uint64_t n, const unsigned long long *d_table, const uint32_t *d_pos,
                              uint32_t lg, const uint32_t *d_empty_pos, const uint32_t *d_w, uint32_t *d_weights, unsigned long long *d_written) {
    if (!n) return;
    k_weight_keys_apply<<<grid_of(n, L, 8), 256, 0, L.stream>>>(d_set_keys, n, d_table, d_pos, lg, d_empty_pos, d_w, d_weights, d_written);
    RIO_COUNT_LAUNCH(L);
}

void launch_merge_walk_changes(const Launch &L, uint32_t *d_idx, const uint32_t *d_walk, uint64_t n, const uint8_t *d_flag, uint32_t n_total) {
    if (!n) return;
    if (n_total <= kMergeMaxSmem)
        k_merge_walk_changes<true><<<grid_of(n, L, 8), 256, n_total, L.stream>>>(d_idx, d_walk, n, d_flag, n_total);
    else
        k_merge_walk_changes<false><<<grid_of(n, L, 8), 256, 0, L.stream>>>(d_idx, d_walk, n, d_flag, n_total);
    RIO_COUNT_LAUNCH(L);
}

}  // namespace rio

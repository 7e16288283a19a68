// k_bounded_weighted.cu -- weighted bounded-load placement (DESIGN.md 3.19): the weight sum, the load histogram, the weighted spill
// selection, the loads of the re-placed objects, and the weight column's row moves of set_erase.  In a translation unit of its own, so
// that no existing kernel's code depends on it.
#include "kernels.cuh"
#include "k_bounded_weighted.cuh"
#include "k_rank_common.cuh"
#include "spec.cuh"

namespace rio {

namespace {

constexpr uint32_t kLoadSmemBins = 8192;

__device__ __forceinline__ uint32_t weight_at(const uint32_t *w, uint64_t i) { return w ? __ldg(w + i) : 1u; }

// 4 B per row, one u64 atomic per warp
__global__ void __launch_bounds__(256)
k_weight_sum(const uint32_t *__restrict__ w, uint64_t n, unsigned long long *__restrict__ sum) {
    unsigned long long s = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) s += __ldg(w + i);
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
    if ((threadIdx.x & 31) == 0 && s) atomicAdd(sum, s);
}

// 8 B per row (idx + w).  With bins (n_total <= kLoadSmemBins) the block sums into shared memory and adds each non-zero bin once;
// either way a warp's lanes on one node make one atomic.  Whole warps run every trip, so the warp-wide intrinsics see every lane.
__global__ void __launch_bounds__(256)
k_load_histogram(const uint32_t *__restrict__ idx, const uint32_t *__restrict__ w, uint64_t n, uint32_t *__restrict__ loads, uint32_t n_total,
                 uint32_t bins) {
    extern __shared__ uint32_t sh[];
    for (uint32_t j = threadIdx.x; j < bins; j += blockDim.x) sh[j] = 0;
    __syncthreads();
    uint32_t *dst = bins ? sh : loads;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        uint32_t j = kNone, wi = 0;
        if (i < n) {
            j = __ldg(idx + i);
            if (j >= n_total) j = kNone;
            else wi = weight_at(w, i);
        }
        warp_load_add(dst, j, wi);
    }
    if (!bins) return;
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < bins; j += blockDim.x) { const uint32_t v = sh[j]; if (v) atomicAdd(&loads[j], v); }
}

// k_select_spill with weights: a row's weight is read only when its hash hits, and a weight-0 row never spills
__global__ void __launch_bounds__(256)
k_select_spill_weighted(const uint64_t *__restrict__ keys, const uint32_t *__restrict__ idx, const uint32_t *__restrict__ w, uint64_t n,
                        const uint32_t *__restrict__ thr, const uint8_t *__restrict__ over, uint32_t round, uint32_t *__restrict__ sel,
                        unsigned long long *nsel, uint32_t *__restrict__ loads) {
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        bool hit = false;
        if (i < n) {
            const uint32_t j = __ldg(idx + i);
            if (j != kNone && __ldg(over + j) && spill_hash(__ldg(keys + i), round) < __ldg(thr + j)) {
                const uint32_t wi = weight_at(w, i);
                hit = wi != 0;
                if (hit && loads) atomicSub(&loads[j], wi);
            }
        }
        const unsigned m = __ballot_sync(0xFFFFFFFFu, hit);
        if (m) {
            const unsigned lane = threadIdx.x & 31, leader = __ffs(m) - 1;
            unsigned long long b = 0;
            if (lane == leader) b = atomicAdd(nsel, (unsigned long long)__popc(m));
            b = __shfl_sync(0xFFFFFFFFu, b, leader);
            if (hit) sel[b + __popc(m & ((1u << lane) - 1))] = (uint32_t)i;
        }
    }
}

// 12 B per spilled row (sel, idx, w)
__global__ void __launch_bounds__(256)
k_add_loads_sel(const uint32_t *__restrict__ sel, uint64_t n_sel, const uint32_t *__restrict__ idx, const uint32_t *__restrict__ w,
                uint32_t *__restrict__ loads, uint32_t n_total) {
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n_sel; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t t = base + threadIdx.x;
        uint32_t j = kNone, wi = 0;
        if (t < n_sel) {
            const uint32_t i = __ldg(sel + t);
            j = __ldg(idx + i);
            if (j >= n_total) j = kNone;
            else wi = weight_at(w, i);
        }
        warp_load_add(loads, j, wi);
    }
}

// one thread per pair; holes lie below the new size and movers at or above it, so no pair reads a row another pair writes
__global__ void __launch_bounds__(256)
k_churn_move_weights(const uint32_t *__restrict__ holes, const uint32_t *__restrict__ movers, const unsigned long long *__restrict__ pairs,
                     uint32_t *__restrict__ w) {
    const uint64_t P = __ldg(pairs);
    for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < P; j += (uint64_t)gridDim.x * blockDim.x)
        w[__ldg(holes + j)] = w[__ldg(movers + j)];
}

int grid_of(uint64_t items, const Launch &L, int per_sm) {
    const uint64_t blocks = (items + 255) / 256, cap = (uint64_t)L.sm_count * per_sm;
    return (int)(blocks < 1 ? 1 : blocks < cap ? blocks : cap);
}

}  // namespace

void launch_weight_sum(const Launch &L, const uint32_t *d_w, uint64_t n, unsigned long long *d_sum) {
    if (!n) return;
    k_weight_sum<<<grid_of(n, L, 8), 256, 0, L.stream>>>(d_w, n, d_sum);
    RIO_COUNT_LAUNCH(L);
}

void launch_load_histogram(const Launch &L, const uint32_t *d_idx, const uint32_t *d_w, uint64_t n, uint32_t *d_loads, uint32_t n_total) {
    if (!n) return;
    const uint32_t bins = n_total <= kLoadSmemBins ? n_total : 0;
    k_load_histogram<<<grid_of(n, L, 4), 256, (size_t)bins * 4, L.stream>>>(d_idx, d_w, n, d_loads, n_total, bins);
    RIO_COUNT_LAUNCH(L);
}

void launch_select_spill_weighted(const Launch &L, const uint64_t *d_keys, const uint32_t *d_idx, const uint32_t *d_w, uint64_t n, const uint32_t *d_thr,
                                  const uint8_t *d_over, uint32_t round, uint32_t *d_sel, unsigned long long *d_nsel, uint32_t *d_loads) {
    if (!n) return;
    k_select_spill_weighted<<<grid_of(n, L, 8), 256, 0, L.stream>>>(d_keys, d_idx, d_w, n, d_thr, d_over, round, d_sel, d_nsel, d_loads);
    RIO_COUNT_LAUNCH(L);
}

void launch_add_loads_sel(const Launch &L, const uint32_t *d_sel, uint64_t n_sel, const uint32_t *d_idx, const uint32_t *d_w, uint32_t *d_loads,
                          uint32_t n_total) {
    if (!n_sel) return;
    k_add_loads_sel<<<grid_of(n_sel, L, 8), 256, 0, L.stream>>>(d_sel, n_sel, d_idx, d_w, d_loads, n_total);
    RIO_COUNT_LAUNCH(L);
}

void launch_churn_move_weights(const Launch &L, const uint32_t *d_holes, const uint32_t *d_movers, uint64_t max_pairs, const unsigned long long *d_pairs,
                               uint32_t *d_w) {
    if (!max_pairs) return;
    k_churn_move_weights<<<grid_of(max_pairs, L, 8), 256, 0, L.stream>>>(d_holes, d_movers, d_pairs, d_w);
    RIO_COUNT_LAUNCH(L);
}

}  // namespace rio

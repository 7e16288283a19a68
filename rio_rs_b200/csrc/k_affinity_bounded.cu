// k_affinity_bounded.cu -- the write-back of a bounded-load affinity round (DESIGN.md 3.16).  In a translation unit of its own, so
// that no existing kernel's code depends on it.
#include "kernels.cuh"
#include "k_affinity_bounded.cuh"

namespace rio {

namespace {

__global__ void __launch_bounds__(256)
k_scatter_idx(const uint32_t *__restrict__ vals, const uint32_t *__restrict__ sel, uint64_t n_sel, uint32_t *__restrict__ idx) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_sel; i += (uint64_t)gridDim.x * blockDim.x) idx[__ldg(sel + i)] = __ldg(vals + i);
}

}  // namespace

void launch_scatter_idx(const Launch &L, const uint32_t *d_vals, const uint32_t *d_sel, uint64_t n_sel, uint32_t *d_idx) {
    if (!n_sel) return;
    const uint64_t blocks = (n_sel + 255) / 256, cap = (uint64_t)L.sm_count * 8;
    k_scatter_idx<<<(int)(blocks < cap ? blocks : cap), 256, 0, L.stream>>>(d_vals, d_sel, n_sel, d_idx);
    RIO_COUNT_LAUNCH(L);
}

}  // namespace rio

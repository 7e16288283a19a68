// k_set_bounded_affinity.cu -- the change-set pass of a bounded-load affinity set (DESIGN.md 3.17) and the count of objects whose node
// differs from the one they held before the call.  In a translation unit of its own, so that no existing kernel's code depends on it.
#include "kernels.cuh"
#include "k_set_bounded_affinity.cuh"
#include "k_affinity_common.cuh"
#include "k_rank_common.cuh"

namespace rio {

namespace {

// Pass 0 of 3.17, in place on idx: 4 B read + 4 B of prev written per object and its node's flag byte; with candidates an S2 object also
// reads its 4K B of features and costs its node and every candidate (one dot product each).  The trip loop is block-uniform, so the
// counter updates and the S1 append can ballot.
template <int KC>
__global__ void __launch_bounds__(kRankThreads, 2)
k_rebalance_changes_bounded_affinity(const float *__restrict__ fobj, uint32_t K, uint32_t *__restrict__ idx, uint32_t *__restrict__ prev, uint64_t n,
                                     const float *__restrict__ fnode, uint32_t n_total, ChangeSetDev cs, uint32_t staged, uint32_t *__restrict__ counters,
                                     uint32_t *__restrict__ sel, unsigned long long *nsel) {
    extern __shared__ __align__(16) unsigned char smem_aff[];
    const uint8_t *flag = cs.flag;
    const uint32_t *cand = cs.cand;
    const float *crow = nullptr;   // candidate q's row at crow + q * K
    if (staged) {
        float *r = reinterpret_cast<float *>(smem_aff);
        uint32_t *c = reinterpret_cast<uint32_t *>(r + (size_t)cs.n_cand * K);
        uint8_t *f = reinterpret_cast<uint8_t *>(c + cs.n_cand);
        for (uint32_t t = threadIdx.x; t < cs.n_cand * K; t += blockDim.x) r[t] = __ldg(fnode + (size_t)__ldg(cs.cand + t / K) * K + t % K);
        for (uint32_t t = threadIdx.x; t < cs.n_cand; t += blockDim.x) c[t] = __ldg(cs.cand + t);
        for (uint32_t t = threadIdx.x; t < n_total; t += blockDim.x) f[t] = __ldg(cs.flag + t);
        __syncthreads();
        flag = f; cand = c; crow = r;
    }
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t b = (uint64_t)blockIdx.x * blockDim.x; b < n; b += stride) {
        const uint64_t i = b + threadIdx.x;
        bool s1 = false;
        uint32_t from = kNone, to = kNone;   // this object's counter updates
        if (i < n) {
            const uint32_t y = idx[i];
            prev[i] = y;
            s1 = y >= n_total || (flag[y] & kChgReplace) != 0;   // kNone is past every table
            if (s1) {
                if (y < n_total) from = y;
            } else if (cs.n_cand) {
                ObjRow<KC> o;
                o.load(fobj, i, K);
                float bc = o.cost_ro(fnode + (size_t)y * K);
                uint32_t bj = y;
                for (uint32_t q = 0; q < cs.n_cand; q++) {
                    const uint32_t j = cand[q];
                    const float c = o.cost(staged ? crow + (size_t)q * K : fnode + (size_t)j * K);
                    if (aff_before(c, j, bc, bj)) { bc = c; bj = j; }
                }
                if (bj != y) { idx[i] = bj; from = y; to = bj; }
            }
        }
        warp_count_add(counters, from, 0xFFFFFFFFu);
        warp_count_add(counters, to, 1u);
        if (__ballot_sync(0xFFFFFFFFu, s1) == 0) continue;
        const unsigned long long p = warp_reserve(nsel, s1 ? 1u : 0u);
        if (s1) sel[p] = (uint32_t)i;
    }
}

__global__ void __launch_bounds__(256)
k_count_diff(const uint32_t *__restrict__ a, const uint32_t *__restrict__ b, uint64_t n, unsigned long long *count) {
    unsigned long long local = 0;
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t n4 = n / 4;
    const uint4 *a4 = reinterpret_cast<const uint4 *>(a), *b4 = reinterpret_cast<const uint4 *>(b);
    for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n4; t += stride) {
        const uint4 x = __ldg(a4 + t), y = __ldg(b4 + t);
        local += (x.x != y.x) + (x.y != y.y) + (x.z != y.z) + (x.w != y.w);
    }
    for (uint64_t t = n4 * 4 + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += stride) local += __ldg(a + t) != __ldg(b + t);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xFFFFFFFFu, local, o);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(count, local);
}

template <int KC>
void rebalance_changes_bounded_affinity(const Launch &L, const float *d_fobj, uint32_t K, uint32_t *d_idx, uint32_t *d_prev, uint64_t n, const float *d_fnode,
                                        uint32_t n_total, const ChangeSetDev &cs, uint32_t *d_counters, uint32_t *d_sel, unsigned long long *d_nsel) {
    const size_t want = aff_changes_smem(n_total, cs.n_cand, K);
    const uint32_t staged = want <= kAffSetSmemBudget;
    launch_rank_kernel<k_rebalance_changes_bounded_affinity<KC>>(L, staged ? want : 0, kAffSetSmemBudget, n, d_fobj, K, d_idx, d_prev, n, d_fnode, n_total, cs,
                                                                 staged, d_counters, d_sel, d_nsel);
}

}  // namespace

void launch_rebalance_changes_bounded_affinity(const Launch &L, const float *d_fobj, uint32_t K, uint32_t *d_idx, uint32_t *d_prev, uint64_t n,
                                               const float *d_fnode, uint32_t n_total, const ChangeSetDev &cs, uint32_t *d_counters, uint32_t *d_sel,
                                               unsigned long long *d_nsel) {
    if (!n) return;
    if (K == 16) rebalance_changes_bounded_affinity<16>(L, d_fobj, K, d_idx, d_prev, n, d_fnode, n_total, cs, d_counters, d_sel, d_nsel);
    else rebalance_changes_bounded_affinity<0>(L, d_fobj, K, d_idx, d_prev, n, d_fnode, n_total, cs, d_counters, d_sel, d_nsel);
    RIO_COUNT_LAUNCH(L);
}

void launch_count_diff(const Launch &L, const uint32_t *d_a, const uint32_t *d_b, uint64_t n, unsigned long long *d_count) {
    if (!n) return;
    const uint64_t blocks = (n / 4 + 255) / 256 + 1, cap = (uint64_t)L.sm_count * 8;
    k_count_diff<<<(int)(blocks < cap ? blocks : cap), 256, 0, L.stream>>>(d_a, d_b, n, d_count);
    RIO_COUNT_LAUNCH(L);
}

}  // namespace rio

// k_affinity_set.cu -- the change-set pass of the affinity resident sets (DESIGN.md 3.15) and the feature-row gather of their S1
// recomputation.  In a translation unit of its own, so that no existing kernel's code depends on it.
#include "kernels.cuh"
#include "k_affinity_set.cuh"
#include "k_affinity_common.cuh"
#include "k_rank_common.cuh"
#include "spec.cuh"

namespace rio {

namespace {

// Insert (c, j) into the list (lc, lj) kept in (cost, index) order; SPREAD: with the domain-aware rule of DESIGN.md 3.12 (a listed
// entry of the same domain that is before it drops the candidate; otherwise the shift stops at the same-domain entry it replaces)
template <int R, bool SPREAD>
__device__ __forceinline__ void aff_insert(float (&lc)[R], uint32_t (&lj)[R], uint32_t (&ld)[R], float c, uint32_t j, uint32_t d) {
    if (!aff_before(c, j, lc[R - 1], lj[R - 1])) return;
    if (SPREAD) {
        bool keep = true;
#pragma unroll
        for (int y = 0; y < R; y++) keep &= !(ld[y] == d && aff_before(lc[y], lj[y], c, j));
        if (!keep) return;
    }
    const uint32_t dc = d;
    bool go = true;
#pragma unroll
    for (int y = 0; y < R; y++) {
        const bool sw = go && aff_before(c, j, lc[y], lj[y]);
        const float tc = lc[y];
        const uint32_t tj = lj[y], td = ld[y];
        lc[y] = sw ? c : tc; lj[y] = sw ? j : tj; ld[y] = sw ? d : td;
        c = sw ? tc : c; j = sw ? tj : j; d = sw ? td : d;
        if (SPREAD) go = go && !(sw && td == dc);
    }
}

// The change-set pass of DESIGN.md 3.15, 4R B/object without candidates, 4R + 4K with (S2 rows only).  S1 objects (a member in REPLACE
// or past the table, or no member) are appended to sel.  An S2 list that is full and has no candidate member keeps its order, and a
// candidate enters only by going before its last member: one dot product for that member and one per candidate.  Only then, or when
// the list is short, is every member and candidate costed and inserted.  The trip loop is block-uniform, so the S1 append can ballot.
template <int KC, int R, bool SPREAD>
__global__ void __launch_bounds__(kRankThreads, 2)
k_rebalance_changes_affinity(const float *__restrict__ fobj, uint32_t K, uint32_t *__restrict__ lists, uint64_t n, const float *__restrict__ fnode,
                             uint32_t n_total, ChangeSetDev cs, uint32_t staged, const uint32_t *__restrict__ ndom, RankedCmp cmp,
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
    uint32_t n_moved = 0, n_changed = 0;
    for (uint64_t b = (uint64_t)blockIdx.x * blockDim.x; b < n; b += stride) {
        const uint64_t i = b + threadIdx.x;
        bool s1 = false;
        if (i < n) {
            uint32_t l[R];
#pragma unroll
            for (int x = 0; x < R; x++) l[x] = lists[i * R + x];
            bool member_cand = false, full = true;
            s1 = l[0] == kNone;   // no member: the list is recomputed
#pragma unroll
            for (int x = 0; x < R; x++) {
                if (l[x] == kNone) { full = false; continue; }
                if (l[x] >= n_total) { s1 = true; continue; }
                const uint8_t f = flag[l[x]];
                s1 |= (f & kChgReplace) != 0;
                member_cand |= (f & kChgCandidate) != 0;
            }
            if (!s1 && cs.n_cand) {
                ObjRow<KC> o;
                o.load(fobj, i, K);
                bool merge = member_cand || !full;
                if (!merge) {
                    const float cl = o.cost_ro(fnode + (size_t)l[R - 1] * K);
                    for (uint32_t q = 0; q < cs.n_cand && !merge; q++) merge = aff_before(o.cost(staged ? crow + (size_t)q * K : fnode + (size_t)cand[q] * K), cand[q], cl, l[R - 1]);
                }
                if (merge) {
                    float lc[R];
                    uint32_t lj[R], ld[R];
#pragma unroll
                    for (int x = 0; x < R; x++) { lc[x] = 0.f; lj[x] = kNone; ld[x] = kNone; }
#pragma unroll
                    for (int x = 0; x < R; x++) {
                        if (l[x] == kNone) continue;
                        aff_insert<R, SPREAD>(lc, lj, ld, o.cost_ro(fnode + (size_t)l[x] * K), l[x], SPREAD ? __ldg(ndom + l[x]) : 0u);
                    }
                    for (uint32_t q = 0; q < cs.n_cand; q++) {
                        const uint32_t j = cand[q];
                        bool in_l = false;
#pragma unroll
                        for (int x = 0; x < R; x++) in_l |= l[x] == j;
                        if (in_l) continue;   // a listed candidate counts once
                        aff_insert<R, SPREAD>(lc, lj, ld, o.cost(staged ? crow + (size_t)q * K : fnode + (size_t)cand[q] * K), j, SPREAD ? __ldg(ndom + j) : 0u);
                    }
                    ranked_store<R, true>(lists + i * R, lj, i, cmp, n_moved, n_changed);
                }
            }
        }
        if (__ballot_sync(0xFFFFFFFFu, s1) == 0) continue;
        const unsigned long long p = warp_reserve(nsel, s1 ? 1u : 0u);
        if (s1) sel[p] = (uint32_t)i;
    }
    ranked_flush<true>(cmp, n_moved, n_changed);
}

// n_sel x K floats by sel; float4 copies when K is a multiple of 4
__global__ void __launch_bounds__(256)
k_gather_rows(const float *__restrict__ rows, uint32_t K, const uint32_t *__restrict__ sel, uint64_t n_sel, float *__restrict__ out) {
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    if ((K & 3) == 0) {
        const uint32_t K4 = K / 4;
        const float4 *r4 = reinterpret_cast<const float4 *>(rows);
        float4 *o4 = reinterpret_cast<float4 *>(out);
        for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_sel * K4; t += stride)
            o4[t] = __ldg(r4 + (uint64_t)__ldg(sel + t / K4) * K4 + t % K4);
    } else {
        for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_sel * K; t += stride)
            out[t] = __ldg(rows + (uint64_t)__ldg(sel + t / K) * K + t % K);
    }
}

template <int KC, int R, bool SPREAD>
void rebalance_changes_affinity(const Launch &L, const float *d_fobj, uint32_t K, uint32_t *d_lists, uint64_t n, const float *d_fnode, uint32_t n_total,
                                const ChangeSetDev &cs, const uint32_t *d_ndom, const RankedCmp &cmp, uint32_t *d_sel, unsigned long long *d_nsel) {
    const size_t want = aff_changes_smem(n_total, cs.n_cand, K);
    const uint32_t staged = want <= kAffSetSmemBudget;
    launch_rank_kernel<k_rebalance_changes_affinity<KC, R, SPREAD>>(L, staged ? want : 0, kAffSetSmemBudget, n, d_fobj, K, d_lists, n, d_fnode, n_total, cs,
                                                                     staged, d_ndom, cmp, d_sel, d_nsel);
}

}  // namespace

void launch_rebalance_changes_affinity(const Launch &L, const float *d_fobj, uint32_t K, uint32_t *d_lists, uint32_t ranks, uint32_t *d_idx, uint64_t n,
                                       const float *d_fnode, uint32_t n_total, const ChangeSetDev &cs, const uint32_t *d_ndom, uint32_t *d_counters,
                                       uint32_t *d_sel, unsigned long long *d_nsel, unsigned long long *d_moved, unsigned long long *d_changed) {
    if (!n) return;
    const RankedCmp cmp{d_idx, d_counters, n_total, d_moved, d_changed};
    if (with_ranks(ranks, [&](auto r) {
            if (d_ndom) {
                if (K == 16) rebalance_changes_affinity<16, r, true>(L, d_fobj, K, d_lists, n, d_fnode, n_total, cs, d_ndom, cmp, d_sel, d_nsel);
                else rebalance_changes_affinity<0, r, true>(L, d_fobj, K, d_lists, n, d_fnode, n_total, cs, d_ndom, cmp, d_sel, d_nsel);
            } else {
                if (K == 16) rebalance_changes_affinity<16, r, false>(L, d_fobj, K, d_lists, n, d_fnode, n_total, cs, d_ndom, cmp, d_sel, d_nsel);
                else rebalance_changes_affinity<0, r, false>(L, d_fobj, K, d_lists, n, d_fnode, n_total, cs, d_ndom, cmp, d_sel, d_nsel);
            }
        }))
        RIO_COUNT_LAUNCH(L);
}

void launch_gather_rows(const Launch &L, const float *d_rows, uint32_t K, const uint32_t *d_sel, uint64_t n_sel, float *d_out) {
    if (!n_sel) return;
    const uint64_t items = n_sel * ((K & 3) == 0 ? K / 4 : K), blocks = (items + 255) / 256, cap = (uint64_t)L.sm_count * 8;
    k_gather_rows<<<(int)(blocks < cap ? blocks : cap), 256, 0, L.stream>>>(d_rows, K, d_sel, n_sel, d_out);
    RIO_COUNT_LAUNCH(L);
}

}  // namespace rio

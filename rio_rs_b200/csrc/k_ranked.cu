// k_ranked.cu -- ranked placement lists (DESIGN.md 3.9): each object's first R distinct nodes under the handle's policy.
//
// rank_1 is the assignment itself; rank_r is the same policy's placement over the live set minus rank_1..rank_{r-1}.
//   * flat weighted rendezvous (3.4): the scores do not depend on the exclusions, so the list is the first R elements of the
//     order (E(u)*r, ~u, j).  One pass over the class-sorted table keeps, per weight class, the best R of "larger u, then lower
//     node index" (no logarithm per pair) and merges those R into the object's list with one E(u)*r each at the class end.
//   * HRW2 (3.8): rank r walks the trie again.  A trie node whose subtree holds none of the r-1 excluded nodes keeps its stored
//     threshold; where it holds some, the contest is re-derived from the subtree weights minus the excluded weight on each side
//     with the exact compare LEFT <=> (v+1)(wl'+wr') <= 2^31 wl' (a 64x64->128 product, no division).  A bucket's chain skips
//     excluded members and takes each member's "rest" from the bucket weight without the excluded ones.
// One thread per object; the excluded nodes (index, bucket leaf, weight) stay in registers, R is a template parameter.
#include "k_rank_common.cuh"
#include "k_ranked.cuh"
#include "k_ranked_changes.cuh"
#include "spec.cuh"

namespace rio {

namespace {

constexpr uint32_t kRankSmemBudget = 200u * 1024u;

// ---- flat weighted rendezvous ------------------------------------------------------------------------------------------
template <int R, bool SMEM>
__global__ void __launch_bounds__(kRankThreads)
k_assign_hrw_ranked(const uint64_t *__restrict__ keys, uint64_t n, NodeTabDev tab, uint32_t *__restrict__ out_idx) {
    extern __shared__ __align__(16) unsigned char smem_rank[];
    const uint4 *rec = reinterpret_cast<const uint4 *>(tab.recs);
    if (SMEM) {
        stage16(smem_rank, tab.recs, tab.n_live * 16u);
        __syncthreads();
        rec = reinterpret_cast<const uint4 *>(smem_rank);
    }
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const ObjHash o = obj_hash(__ldg(keys + i));
        uint64_t gs[R];                  // the object's list so far, best first: (score, u, node index)
        uint32_t gu[R], gj[R];
#pragma unroll
        for (int x = 0; x < R; x++) { gs[x] = ~0ull; gu[x] = 0; gj[x] = kNone; }
        for (uint32_t c = 0; c < tab.n_classes; c++) {
            const ClassRec cr = tab.classes[c];
            const uint32_t end = tab.classes[c + 1].start;
            // best R of the class as (u << 32 | ~node index): larger is better; 0 = empty (no node index is 0xFFFFFFFF)
            uint64_t ck[R];
#pragma unroll
            for (int x = 0; x < R; x++) ck[x] = 0;
            for (uint32_t q = cr.start; q < end; q++) {
                const uint4 r = SMEM ? rec[q] : __ldg(rec + q);
                uint64_t k = ((uint64_t)pair_hash(o, r.x, r.z, r.w) << 32) | (uint32_t)~r.y;
                if (k > ck[R - 1]) {
#pragma unroll
                    for (int x = 0; x < R; x++) { const uint64_t t = ck[x]; const bool sw = k > t; ck[x] = sw ? k : t; k = sw ? t : k; }
                }
            }
            // class complete: one E(u)*r per class candidate, merged into the list in the order of cand_better
#pragma unroll
            for (int x = 0; x < R; x++) {
                if (!ck[x]) break;
                uint32_t u = (uint32_t)(ck[x] >> 32), j = ~(uint32_t)ck[x];
                uint64_t s = (uint64_t)elog(u) * cr.invw;
                if (!cand_better(s, u, j, gs[R - 1], gu[R - 1], gj[R - 1])) break;   // the class's later candidates rank lower still
#pragma unroll
                for (int y = 0; y < R; y++) {
                    const bool sw = cand_better(s, u, j, gs[y], gu[y], gj[y]);
                    const uint64_t ts = gs[y]; const uint32_t tu = gu[y], tj = gj[y];
                    gs[y] = sw ? s : ts; gu[y] = sw ? u : tu; gj[y] = sw ? j : tj;
                    s = sw ? ts : s; u = sw ? tu : u; j = sw ? tj : j;
                }
            }
        }
        uint32_t *dst = out_idx + i * R;
#pragma unroll
        for (int x = 0; x < R; x++) dst[x] = gj[x];
    }
}

// ---- HRW2 ----------------------------------------------------------------------------------------------------------------
// Compare mode (CMP, DESIGN.md 3.11): out_idx holds the stored lists of a resident set.  Each walk is compared with the stored row,
// only changed rows are written, and the set's primary index and counters follow column 0.  The extra argument comes last, so the
// plain instantiations keep their parameter layout and code.  RankedCmp and the epilogue (ranked_store, ranked_flush) are in
// k_rank_common.cuh.
template <int R, bool SMEM, bool CMP>
__global__ void __launch_bounds__(kRankThreads)
k_assign_trie_ranked(const uint64_t *__restrict__ keys, uint64_t n, TrieDev t, TrieRankDev rk, const __grid_constant__ LevelConsts lc,
                     uint32_t *__restrict__ out_idx, const RankedCmp cmp) {
    extern __shared__ __align__(16) unsigned char smem_rank[];
    const unsigned char *blob = reinterpret_cast<const unsigned char *>(t.blob);
    const unsigned long long *W = rk.wsum;
    const uint2 *node = rk.node;
    if (SMEM) {   // [blob][side table]: both multiples of 16 bytes
        stage16(smem_rank, t.blob, t.blob_bytes);
        stage16(smem_rank + t.blob_bytes, rk.wsum, rk.bytes);
        __syncthreads();
        blob = smem_rank;
        W = reinterpret_cast<const unsigned long long *>(smem_rank + t.blob_bytes);
        node = reinterpret_cast<const uint2 *>(smem_rank + t.blob_bytes + (16u << t.bits));
    }
    const uint32_t *tab32 = reinterpret_cast<const uint32_t *>(blob);
    const uint32_t bits = t.bits;
    uint32_t n_moved = 0, n_changed = 0;   // compare mode only (a thread walks far fewer than 2^32 objects)
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const ObjHash o = obj_hash(__ldg(keys + i));
        uint32_t res[R], xleaf[R], xw[R];   // ranks so far: node index, heap index of its bucket, weight
#pragma unroll
        for (int r = 0; r < R; r++) {
            uint32_t nid = kNone;
            if ((uint32_t)r < rk.n_members) {
                uint32_t hi = 1;
                uint32_t on = (1u << r) - 1u;   // the excluded nodes inside the current subtree: all of them at the root
                for (uint32_t l = 0; l < bits; l++) {
                    const uint32_t u = contest_u(o, lc.s0[l], lc.m2[l], lc.h2[l]);
                    uint32_t right;
                    if (!on) {
                        right = u > tab32[hi] ? 1u : 0u;
                    } else {
                        const uint32_t sh = bits - 1u - l;
                        unsigned long long exl = 0, exr = 0;
                        uint32_t onr = 0;
#pragma unroll
                        for (int x = 0; x < r; x++) {
                            if (!((on >> x) & 1u)) continue;
                            if ((xleaf[x] >> sh) & 1u) { exr += xw[x]; onr |= 1u << x; }
                            else exl += xw[x];
                        }
                        right = contest_left_exact(u >> 1, W[2 * hi] - exl, W[2 * hi + 1] - exr) ? 0u : 1u;
                        on = right ? onr : (on & ~onr);
                    }
                    hi = 2 * hi + right;
                }
                uint32_t w = tab32[hi];
                if (!on) {
                    // no excluded member in the bucket: the walk of k_assign_trie
                    while ((int32_t)w <= -2) {
                        const unsigned char *p = blob + (w & 0x7FFFFFFFu);
                        const uint4 c = *reinterpret_cast<const uint4 *>(p);
                        const uint2 nn = *reinterpret_cast<const uint2 *>(p + 16);
                        if (contest_u(o, c.x, c.y, c.z) <= c.w) { w = nn.x; break; }
                        w = nn.y;
                    }
                    nid = w;
                } else {
                    // the bucket's chain without its excluded members: "m_k against the rest" with rest = the bucket's remaining
                    // weight after m_k; the walk only enters buckets with a remaining member, so one is always taken
                    unsigned long long remain = W[hi];
#pragma unroll
                    for (int x = 0; x < r; x++) if ((on >> x) & 1u) remain -= xw[x];
                    while ((int32_t)w <= -2) {
                        const unsigned char *p = blob + (w & 0x7FFFFFFFu);
                        const uint4 c = *reinterpret_cast<const uint4 *>(p);
                        const uint2 nn = *reinterpret_cast<const uint2 *>(p + 16);
                        bool excluded = false;
#pragma unroll
                        for (int x = 0; x < r; x++) excluded |= ((on >> x) & 1u) && res[x] == nn.x;
                        if (!excluded) {
                            const uint32_t wm = node[nn.x].y;
                            remain -= wm;
                            if (contest_left_exact(contest_u(o, c.x, c.y, c.z) >> 1, wm, remain)) { w = nn.x; break; }
                        }
                        w = nn.y;
                    }
                    nid = w;
                }
            }
            res[r] = nid;
            if (r + 1 < R && nid != kNone) {
                const uint2 nd = node[nid];
                xleaf[r] = (1u << bits) + nd.x;
                xw[r] = nd.y;
            }
        }
        ranked_store<R, CMP>(out_idx + i * R, res, i, cmp, n_moved, n_changed);
    }
    ranked_flush<CMP>(cmp, n_moved, n_changed);
}

template <int R>
void hrw_ranked(const Launch &L, const uint64_t *d_keys, uint64_t n, const NodeTabDev &tab, uint32_t *d_out) {
    const size_t smem = (size_t)tab.n_live * 16;
    if (smem <= 96u * 1024u) {
        launch_rank_kernel<k_assign_hrw_ranked<R, true>>(L, smem, kRankSmemBudget, n, d_keys, n, tab, d_out);
    } else {
        launch_rank_kernel<k_assign_hrw_ranked<R, false>>(L, 0, kRankSmemBudget, n, d_keys, n, tab, d_out);
    }
}

template <int R, bool CMP = false>
void trie_ranked(const Launch &L, const uint64_t *d_keys, uint64_t n, const TrieDev &t, const TrieRankDev &rk, uint32_t *d_out, const RankedCmp &cmp = {}) {
    static const LevelConsts lc = level_consts();
    const size_t smem = (size_t)t.blob_bytes + rk.bytes;
    if (smem <= kRankSmemBudget) {
        launch_rank_kernel<k_assign_trie_ranked<R, true, CMP>>(L, smem, kRankSmemBudget, n, d_keys, n, t, rk, lc, d_out, cmp);
    } else {
        launch_rank_kernel<k_assign_trie_ranked<R, false, CMP>>(L, 0, kRankSmemBudget, n, d_keys, n, t, rk, lc, d_out, cmp);
    }
}

}  // namespace

void launch_assign_hrw_ranked(const Launch &L, const uint64_t *d_keys, uint64_t n, const NodeTabDev &tab, uint32_t ranks, uint32_t *d_out_idx) {
    if (!n) return;
    if (with_ranks(ranks, [&](auto r) { hrw_ranked<r>(L, d_keys, n, tab, d_out_idx); })) RIO_COUNT_LAUNCH(L);
}

void launch_assign_trie_ranked(const Launch &L, const uint64_t *d_keys, uint64_t n, const TrieDev &t, const TrieRankDev &rk, uint32_t ranks,
                               uint32_t *d_out_idx) {
    if (!n) return;
    if (with_ranks(ranks, [&](auto r) { trie_ranked<r>(L, d_keys, n, t, rk, d_out_idx); })) RIO_COUNT_LAUNCH(L);
}

void launch_reassign_trie_ranked(const Launch &L, const uint64_t *d_keys, uint64_t n, const TrieDev &t, const TrieRankDev &rk, uint32_t ranks, uint32_t *d_lists,
                                 uint32_t *d_idx, uint32_t *d_counters, uint32_t n_total, unsigned long long *d_moved, unsigned long long *d_changed) {
    if (!n) return;
    const RankedCmp cmp{d_idx, d_counters, n_total, d_moved, d_changed};
    if (with_ranks(ranks, [&](auto r) { trie_ranked<r, true>(L, d_keys, n, t, rk, d_lists, cmp); })) RIO_COUNT_LAUNCH(L);
}

}  // namespace rio

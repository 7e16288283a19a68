// k_spread.cu -- failure-domain ranked lists (DESIGN.md 3.12): each object's first R nodes in R distinct domains.
//
// rank_1 is the assignment itself; rank_r is the same policy's placement over the live set minus every node of the domains of
// rank_1..rank_{r-1}.
//   * flat weighted rendezvous (3.4): the scores do not depend on the exclusions, so the list is the order (E(u)*r, ~u, j) with
//     only the first node of each domain kept.  The class-sorted pass of k_assign_hrw_ranked keeps, per class and then per object,
//     the best R entries of distinct domains: a candidate whose domain is listed replaces that entry if it is better and is dropped
//     otherwise; a candidate of a new domain must beat the R-th entry.  The domain of a record is read on the insert path only.
//   * HRW2 (3.8): rank r walks the trie again with r-1 whole domains excluded.  Per excluded domain the thread keeps the range of
//     its members (sorted by bucket) inside the current subtree; one binary search per level splits it at the level's bucket bit,
//     and two prefix differences give the excluded weight on each side of the exact contest of k_assign_trie_ranked.
#include "k_rank_common.cuh"
#include "k_spread.cuh"
#include "k_spread_changes.cuh"
#include "k_ranked.cuh"
#include "spec.cuh"

namespace rio {

namespace {

constexpr uint32_t kSpreadSmemBudget = 200u * 1024u;   // the budget of the ranked walk (k_ranked.cu)

// ---- flat weighted rendezvous ------------------------------------------------------------------------------------------
template <int R, bool SMEM>
__global__ void __launch_bounds__(kRankThreads)
k_assign_hrw_spread(const uint64_t *__restrict__ keys, uint64_t n, NodeTabDev tab, const uint32_t *__restrict__ pos_dom, uint32_t *__restrict__ out_idx) {
    extern __shared__ __align__(16) unsigned char smem_spread[];
    const uint4 *rec = reinterpret_cast<const uint4 *>(tab.recs);
    const uint32_t *dom = pos_dom;
    if (SMEM) {   // [records][domain per record, padded to 16 bytes]
        stage16(smem_spread, tab.recs, tab.n_live * 16u);
        stage16(smem_spread + tab.n_live * 16u, pos_dom, (tab.n_live * 4u + 15u) & ~15u);
        __syncthreads();
        rec = reinterpret_cast<const uint4 *>(smem_spread);
        dom = reinterpret_cast<const uint32_t *>(smem_spread + tab.n_live * 16u);
    }
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const ObjHash o = obj_hash(__ldg(keys + i));
        uint64_t gs[R];                  // the object's list so far, best first: (score, u, node index, domain)
        uint32_t gu[R], gj[R], gd[R];
#pragma unroll
        for (int x = 0; x < R; x++) { gs[x] = ~0ull; gu[x] = 0; gj[x] = kNone; gd[x] = kNone; }
        for (uint32_t c = 0; c < tab.n_classes; c++) {
            const ClassRec cr = tab.classes[c];
            const uint32_t end = tab.classes[c + 1].start;
            // best R of the class in distinct domains as (u << 32 | ~node index): larger is better; 0 = empty
            uint64_t ck[R];
            uint32_t cd[R];
#pragma unroll
            for (int x = 0; x < R; x++) { ck[x] = 0; cd[x] = kNone; }
            for (uint32_t q = cr.start; q < end; q++) {
                const uint4 r = SMEM ? rec[q] : __ldg(rec + q);
                uint64_t k = ((uint64_t)pair_hash(o, r.x, r.z, r.w) << 32) | (uint32_t)~r.y;
                if (k > ck[R - 1]) {   // a listed entry of the same domain is better than ck[R-1]: nothing below it can enter
                    uint32_t d = SMEM ? dom[q] : __ldg(dom + q);
                    bool keep = true;
#pragma unroll
                    for (int x = 0; x < R; x++) keep &= !(cd[x] == d && ck[x] > k);
                    if (keep) {   // insert; the shift stops at the entry of the same domain it replaces, if there is one
                        const uint32_t dc = d;
                        bool go = true;
#pragma unroll
                        for (int x = 0; x < R; x++) {
                            const uint64_t t = ck[x]; const uint32_t td = cd[x];
                            const bool sw = go && k > t;
                            ck[x] = sw ? k : t; cd[x] = sw ? d : td;
                            k = sw ? t : k; d = sw ? td : d;
                            go = go && !(sw && td == dc);
                        }
                    }
                }
            }
            // class complete: one E(u)*r per class candidate, merged into the list with the same rule in the order of cand_better
#pragma unroll
            for (int x = 0; x < R; x++) {
                if (!ck[x]) break;
                uint32_t u = (uint32_t)(ck[x] >> 32), j = ~(uint32_t)ck[x], d = cd[x];
                uint64_t s = (uint64_t)elog(u) * cr.invw;
                if (!cand_better(s, u, j, gs[R - 1], gu[R - 1], gj[R - 1])) break;   // the class's later candidates rank lower still
                // spread_insert of k_rank_common.cuh, written out: called here it changes this kernel's register allocation at R = 1
                bool keep = true;
#pragma unroll
                for (int y = 0; y < R; y++) keep &= !(gd[y] == d && cand_better(gs[y], gu[y], gj[y], s, u, j));
                if (!keep) continue;
                const uint32_t dc = d;
                bool go = true;
#pragma unroll
                for (int y = 0; y < R; y++) {
                    const bool sw = go && cand_better(s, u, j, gs[y], gu[y], gj[y]);
                    const uint64_t ts = gs[y]; const uint32_t tu = gu[y], tj = gj[y], td = gd[y];
                    gs[y] = sw ? s : ts; gu[y] = sw ? u : tu; gj[y] = sw ? j : tj; gd[y] = sw ? d : td;
                    s = sw ? ts : s; u = sw ? tu : u; j = sw ? tj : j; d = sw ? td : d;
                    go = go && !(sw && td == dc);
                }
            }
        }
        uint32_t *dst = out_idx + i * R;
#pragma unroll
        for (int x = 0; x < R; x++) dst[x] = gj[x];
    }
}

// ---- HRW2 ----------------------------------------------------------------------------------------------------------------
// Compare mode (CMP, DESIGN.md 3.13): out_idx holds the stored lists of a spread resident set, written back only where the walk
// differs, as in the compare mode of k_assign_trie_ranked.  The extra argument comes last, so the plain instantiations keep their code.
// The compare instantiations ask for one CTA per SM as their occupancy floor: without that hint ptxas spills at R = 6 to stay at 64
// registers; with it R = 6 takes 66 and nothing spills (the plain ones have no such hint, as before).
template <int R, bool SMEM, bool CMP>
__global__ void __launch_bounds__(kRankThreads, CMP ? 1 : 0)
k_assign_trie_spread(const uint64_t *__restrict__ keys, uint64_t n, TrieDev t, SpreadTabDev sp, const __grid_constant__ LevelConsts lc,
                     uint32_t *__restrict__ out_idx, const RankedCmp cmp) {
    extern __shared__ __align__(16) unsigned char smem_spread[];
    const unsigned char *blob = reinterpret_cast<const unsigned char *>(t.blob);
    const unsigned char *side = sp.base;
    if (SMEM) {   // [blob][W and node]: the bytes k_assign_trie_ranked stages, so both walks fit the same number of CTAs per SM
        stage16(smem_spread, t.blob, t.blob_bytes);
        stage16(smem_spread + t.blob_bytes, sp.base, sp.o_ndom);
        __syncthreads();
        blob = smem_spread;
        side = smem_spread + t.blob_bytes;
    }
    const uint32_t *tab32 = reinterpret_cast<const uint32_t *>(blob);
    const unsigned long long *W = reinterpret_cast<const unsigned long long *>(side);
    const uint2 *node = reinterpret_cast<const uint2 *>(side + sp.o_node);
    // the domain part (~20 B per live node) is read through the read-only path: it is touched only where an excluded domain has
    // members in the subtree, and staging it would cost the walk a CTA per SM at M = 1024
    const unsigned long long *pre = reinterpret_cast<const unsigned long long *>(sp.base + sp.o_pre);
    const uint32_t *ndom = reinterpret_cast<const uint32_t *>(sp.base + sp.o_ndom);
    const uint32_t *mb = reinterpret_cast<const uint32_t *>(sp.base + sp.o_mb);
    const uint32_t *dstart = reinterpret_cast<const uint32_t *>(sp.base + sp.o_dstart);
    const uint32_t bits = t.bits;
    uint32_t n_moved = 0, n_changed = 0;   // compare mode only (a thread walks far fewer than 2^32 objects)
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const ObjHash o = obj_hash(__ldg(keys + i));
        uint32_t res[R], xd[R];   // ranks so far: node index, its dense domain
#pragma unroll
        for (int r = 0; r < R; r++) {
            uint32_t nid = kNone;
            if ((uint32_t)r < sp.n_domains) {
                // [lo, hi): the members of excluded domain x inside the current subtree, in bucket order; all of them at the root
                uint32_t lo[R], hi[R];
#pragma unroll
                for (int x = 0; x < r; x++) { lo[x] = __ldg(dstart + xd[x]); hi[x] = __ldg(dstart + xd[x] + 1); }
                uint32_t on = (1u << r) - 1u;   // excluded domains with members in the current subtree
                uint32_t h = 1;
                for (uint32_t l = 0; l < bits; l++) {
                    const uint32_t u = contest_u(o, lc.s0[l], lc.m2[l], lc.h2[l]);
                    uint32_t right;
                    if (!on) {
                        right = u > tab32[h] ? 1u : 0u;
                    } else {
                        const uint32_t sh = bits - 1u - l;
                        unsigned long long exl = 0, exr = 0;
                        uint32_t mid[R];
#pragma unroll
                        for (int x = 0; x < r; x++) {
                            if (!((on >> x) & 1u)) continue;
                            // the subtree's buckets share the bits above sh: its members with bit sh set (the right child) come last
                            uint32_t a = lo[x], b = hi[x];
                            while (a < b) {
                                const uint32_t m = (a + b) >> 1;
                                if ((__ldg(mb + m) >> sh) & 1u) b = m; else a = m + 1;
                            }
                            mid[x] = a;
                            const unsigned long long pa = __ldg(pre + a);
                            exl += pa - __ldg(pre + lo[x]);
                            exr += __ldg(pre + hi[x]) - pa;
                        }
                        right = contest_left_exact(u >> 1, W[2 * h] - exl, W[2 * h + 1] - exr) ? 0u : 1u;
#pragma unroll
                        for (int x = 0; x < r; x++) {
                            if (!((on >> x) & 1u)) continue;
                            if (right) lo[x] = mid[x]; else hi[x] = mid[x];
                            if (lo[x] == hi[x]) on &= ~(1u << x);
                        }
                    }
                    h = 2 * h + right;
                }
                uint32_t w = tab32[h];
                if (!on) {
                    // no excluded member in the bucket: the walk of k_assign_trie
                    while ((int32_t)w <= -2) {
                        const unsigned char *p = blob + (w & 0x7FFFFFFFu);
                        const uint4 c = *reinterpret_cast<const uint4 *>(p);
                        const uint2 nn = *reinterpret_cast<const uint2 *>(p + 16);
                        if (contest_u(o, c.x, c.y, c.z) <= c.w) { w = nn.x; break; }
                        w = nn.y;
                    }
                } else {
                    // the bucket's chain without the members of excluded domains, "m_k against the rest" over the remaining weight;
                    // the walk only enters buckets with a remaining member, so one is always taken
                    unsigned long long remain = W[h];
#pragma unroll
                    for (int x = 0; x < r; x++) if ((on >> x) & 1u) remain -= __ldg(pre + hi[x]) - __ldg(pre + lo[x]);
                    while ((int32_t)w <= -2) {
                        const unsigned char *p = blob + (w & 0x7FFFFFFFu);
                        const uint4 c = *reinterpret_cast<const uint4 *>(p);
                        const uint2 nn = *reinterpret_cast<const uint2 *>(p + 16);
                        const uint32_t dm = __ldg(ndom + nn.x);
                        bool excluded = false;
#pragma unroll
                        for (int x = 0; x < r; x++) excluded |= ((on >> x) & 1u) && xd[x] == dm;
                        if (!excluded) {
                            const uint32_t wm = node[nn.x].y;
                            remain -= wm;
                            if (contest_left_exact(contest_u(o, c.x, c.y, c.z) >> 1, wm, remain)) { w = nn.x; break; }
                        }
                        w = nn.y;
                    }
                }
                nid = w;
            }
            res[r] = nid;
            if (r + 1 < R && nid != kNone) xd[r] = __ldg(ndom + nid);
        }
        ranked_store<R, CMP>(out_idx + i * R, res, i, cmp, n_moved, n_changed);
    }
    ranked_flush<CMP>(cmp, n_moved, n_changed);
}

template <int R>
void hrw_spread(const Launch &L, const uint64_t *d_keys, uint64_t n, const NodeTabDev &tab, const SpreadTabDev &sp, uint32_t *d_out) {
    const uint32_t *pos_dom = reinterpret_cast<const uint32_t *>(sp.base + sp.trie_bytes);
    const size_t smem = (size_t)tab.n_live * 16 + ((size_t)tab.n_live * 4 + 15) / 16 * 16;
    if (smem <= 96u * 1024u) {
        launch_rank_kernel<k_assign_hrw_spread<R, true>>(L, smem, kSpreadSmemBudget, n, d_keys, n, tab, pos_dom, d_out);
    } else {
        launch_rank_kernel<k_assign_hrw_spread<R, false>>(L, 0, kSpreadSmemBudget, n, d_keys, n, tab, pos_dom, d_out);
    }
}

template <int R, bool CMP = false>
void trie_spread(const Launch &L, const uint64_t *d_keys, uint64_t n, const TrieDev &t, const SpreadTabDev &sp, uint32_t *d_out, const RankedCmp &cmp = {}) {
    static const LevelConsts lc = level_consts();
    const size_t smem = (size_t)t.blob_bytes + sp.o_ndom;
    if (smem <= kSpreadSmemBudget) {
        launch_rank_kernel<k_assign_trie_spread<R, true, CMP>>(L, smem, kSpreadSmemBudget, n, d_keys, n, t, sp, lc, d_out, cmp);
    } else {
        launch_rank_kernel<k_assign_trie_spread<R, false, CMP>>(L, 0, kSpreadSmemBudget, n, d_keys, n, t, sp, lc, d_out, cmp);
    }
}

}  // namespace

void launch_assign_hrw_spread(const Launch &L, const uint64_t *d_keys, uint64_t n, const NodeTabDev &tab, const SpreadTabDev &sp, uint32_t ranks,
                              uint32_t *d_out_idx) {
    if (!n) return;
    if (with_ranks(ranks, [&](auto r) { hrw_spread<r>(L, d_keys, n, tab, sp, d_out_idx); })) RIO_COUNT_LAUNCH(L);
}

void launch_assign_trie_spread(const Launch &L, const uint64_t *d_keys, uint64_t n, const TrieDev &t, const SpreadTabDev &sp, uint32_t ranks,
                               uint32_t *d_out_idx) {
    if (!n) return;
    if (with_ranks(ranks, [&](auto r) { trie_spread<r>(L, d_keys, n, t, sp, d_out_idx); })) RIO_COUNT_LAUNCH(L);
}

void launch_reassign_trie_spread(const Launch &L, const uint64_t *d_keys, uint64_t n, const TrieDev &t, const SpreadTabDev &sp, uint32_t ranks, uint32_t *d_lists,
                                 uint32_t *d_idx, uint32_t *d_counters, uint32_t n_total, unsigned long long *d_moved, unsigned long long *d_changed) {
    if (!n) return;
    const RankedCmp cmp{d_idx, d_counters, n_total, d_moved, d_changed};
    if (with_ranks(ranks, [&](auto r) { trie_spread<r, true>(L, d_keys, n, t, sp, d_lists, cmp); })) RIO_COUNT_LAUNCH(L);
}

}  // namespace rio

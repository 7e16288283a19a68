// ranked_launchers.cpp -- TEST INFRASTRUCTURE: host restatements of the ranked-list launchers declared in csrc/k_ranked.cuh, linked
// beside launchers.cpp by tests/test_gpu_ranked.py so that the ranked entry points of csrc/engine.cu run without a GPU.
//
// Like launchers.cpp: each function does, sequentially and in the plainest way, what the kernel is SPECIFIED to do (DESIGN.md 3.9) on
// the tables the engine builds; it says nothing about the kernels, which are proven on the GPU against the oracle.
#include <algorithm>
#include <vector>

#include "../../../rio_rs_b200/csrc/k_ranked.cuh"
#include "../../../rio_rs_b200/csrc/spec.cuh"
#include "../../../rio_rs_b200/csrc/trie_table.hpp"

namespace rio {

namespace {

inline void count(const Launch &L) { if (L.launch_counter) ++*L.launch_counter; }

const ContestRec *levels() {
    static const std::vector<ContestRec> v = trie_level_constants(16);
    return v.data();
}

// LEFT iff v < floor(2^31 wl / (wl + wr)); an empty side is a forced outcome
bool left(uint32_t v, uint64_t wl, uint64_t wr) { return wl && (!wr || v < (uint64_t)(((unsigned __int128)wl << 31) / (wl + wr))); }

}  // namespace

// rank r = the flat weighted rendezvous (3.4) over the live set minus ranks 1..r-1
void launch_assign_hrw_ranked(const Launch &L, const uint64_t *keys, uint64_t n, const NodeTabDev &tab, uint32_t ranks, uint32_t *out) {
    if (!n) return;
    for (uint64_t i = 0; i < n; i++) {
        const ObjHash o = obj_hash(keys[i]);
        uint32_t *row = out + i * ranks;
        for (uint32_t r = 0; r < ranks; r++) {
            uint64_t best_sc = 0;
            uint32_t best_u = 0, best_i = kNone;
            for (uint32_t c = 0; c < tab.n_classes; c++)
                for (uint32_t q = tab.classes[c].start; q < tab.classes[c + 1].start; q++) {
                    const NodeRec &nr = tab.recs[q];
                    if (std::find(row, row + r, nr.nidx) != row + r) continue;
                    const uint32_t u = pair_hash(o, nr.s0, nr.s1, nr.s2);
                    const uint64_t sc = (uint64_t)elog(u) * tab.classes[c].invw;
                    if (best_i == kNone || cand_better(sc, u, nr.nidx, best_sc, best_u, best_i)) { best_sc = sc; best_u = u; best_i = nr.nidx; }
                }
            row[r] = best_i;
        }
    }
    count(L);
}

// HRW2: the walk with every contest whose subtree holds an excluded node re-derived from the subtree weights minus the excluded
// weight, and a bucket's chain without its excluded members
void launch_assign_trie_ranked(const Launch &L, const uint64_t *keys, uint64_t n, const TrieDev &t, const TrieRankDev &rk, uint32_t ranks, uint32_t *out) {
    if (!n) return;
    const uint32_t *blob = reinterpret_cast<const uint32_t *>(t.blob), nb = 1u << t.bits;
    for (uint64_t i = 0; i < n; i++) {
        const ObjHash o = obj_hash(keys[i]);
        uint32_t *row = out + i * ranks;
        for (uint32_t r = 0; r < ranks; r++) {
            if (r >= rk.n_members) { row[r] = kNone; continue; }
            auto ex_weight = [&](uint32_t heap, uint32_t depth) {   // excluded weight under the trie node `heap` at `depth`
                uint64_t s = 0;
                for (uint32_t x = 0; x < r; x++) if (((nb + rk.node[row[x]].x) >> (t.bits - depth)) == heap) s += rk.node[row[x]].y;
                return s;
            };
            uint32_t hi = 1;
            for (uint32_t l = 0; l < t.bits; l++) {
                const uint32_t v = contest_u(o, levels()[l].s0, levels()[l].m2, levels()[l].h2) >> 1;
                const bool go_left = left(v, rk.wsum[2 * hi] - ex_weight(2 * hi, l + 1), rk.wsum[2 * hi + 1] - ex_weight(2 * hi + 1, l + 1));
                hi = 2 * hi + (go_left ? 0u : 1u);
            }
            uint32_t w = blob[hi];
            uint64_t remain = rk.wsum[hi] - ex_weight(hi, t.bits);
            while ((int32_t)w <= -2) {
                const uint32_t *p = blob + (w & 0x7FFFFFFFu) / 4;
                if (std::find(row, row + r, p[4]) == row + r) {
                    const uint32_t wm = rk.node[p[4]].y;
                    remain -= wm;
                    if (left(contest_u(o, p[0], p[1], p[2]) >> 1, wm, remain)) { w = p[4]; break; }
                }
                w = p[5];
            }
            row[r] = w;
        }
    }
    count(L);
}

}  // namespace rio

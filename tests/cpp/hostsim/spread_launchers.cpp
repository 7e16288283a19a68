// spread_launchers.cpp -- TEST INFRASTRUCTURE: host restatements of the failure-domain ranked launchers declared in csrc/k_spread.cuh,
// linked beside launchers.cpp by tests/test_gpu_spread.py so that the spread entry points of csrc/engine.cu run without a GPU.
//
// Like ranked_launchers.cpp: each function does, sequentially and in the plainest way, what the kernel is SPECIFIED to do (DESIGN.md
// 3.12) on the tables the engine builds; it says nothing about the kernels, which are proven on the GPU against the oracle.
#include <algorithm>
#include <vector>

#include "../../../rio_rs_b200/csrc/k_spread.cuh"
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

template <class T> const T *part(const SpreadTabDev &sp, uint32_t off) { return reinterpret_cast<const T *>(sp.base + off); }

}  // namespace

// rank r = the flat weighted rendezvous (3.4) over the live set minus the domains of ranks 1..r-1
void launch_assign_hrw_spread(const Launch &L, const uint64_t *keys, uint64_t n, const NodeTabDev &tab, const SpreadTabDev &sp, uint32_t ranks,
                              uint32_t *out) {
    if (!n) return;
    const uint32_t *pos_dom = part<uint32_t>(sp, sp.trie_bytes);
    for (uint64_t i = 0; i < n; i++) {
        const ObjHash o = obj_hash(keys[i]);
        uint32_t *row = out + i * ranks;
        std::vector<uint32_t> gone;   // domains of the ranks so far
        for (uint32_t r = 0; r < ranks; r++) {
            uint64_t best_sc = 0;
            uint32_t best_u = 0, best_i = kNone, best_d = kNone;
            for (uint32_t c = 0; c < tab.n_classes; c++)
                for (uint32_t q = tab.classes[c].start; q < tab.classes[c + 1].start; q++) {
                    if (std::find(gone.begin(), gone.end(), pos_dom[q]) != gone.end()) continue;
                    const NodeRec &nr = tab.recs[q];
                    const uint32_t u = pair_hash(o, nr.s0, nr.s1, nr.s2);
                    const uint64_t sc = (uint64_t)elog(u) * tab.classes[c].invw;
                    if (best_i == kNone || cand_better(sc, u, nr.nidx, best_sc, best_u, best_i)) { best_sc = sc; best_u = u; best_i = nr.nidx; best_d = pos_dom[q]; }
                }
            row[r] = best_i;
            gone.push_back(best_d);
        }
    }
    count(L);
}

// HRW2: the walk with every contest re-derived from the subtree weights minus the weight of the excluded domains' members in each
// subtree, and a bucket's chain without those members
void launch_assign_trie_spread(const Launch &L, const uint64_t *keys, uint64_t n, const TrieDev &t, const SpreadTabDev &sp, uint32_t ranks,
                               uint32_t *out) {
    if (!n) return;
    const uint32_t *blob = reinterpret_cast<const uint32_t *>(t.blob), nb = 1u << t.bits;
    const uint64_t *W = part<uint64_t>(sp, 0);
    const uint2 *node = part<uint2>(sp, sp.o_node);
    const uint32_t *ndom = part<uint32_t>(sp, sp.o_ndom);
    std::vector<uint32_t> live;   // the node part is padded to 16 bytes: a padding entry has weight 0
    for (uint32_t j = 0; j < (sp.o_ndom - sp.o_node) / 8; j++) if (node[j].y) live.push_back(j);
    std::vector<uint64_t> exw(2 * (size_t)nb, 0);   // per trie node: weight of the excluded members below it
    std::vector<uint32_t> touched;
    for (uint64_t i = 0; i < n; i++) {
        const ObjHash o = obj_hash(keys[i]);
        uint32_t *row = out + i * ranks;
        for (uint32_t r = 0; r < ranks; r++) {
            if (r >= sp.n_domains) { row[r] = kNone; continue; }
            auto excluded = [&](uint32_t j) {
                for (uint32_t x = 0; x < r; x++) if (ndom[row[x]] == ndom[j]) return true;
                return false;
            };
            for (uint32_t hp : touched) exw[hp] = 0;
            touched.clear();
            for (uint32_t j : live)
                if (excluded(j))
                    for (uint32_t hp = nb + node[j].x; hp; hp >>= 1) { exw[hp] += node[j].y; touched.push_back(hp); }
            uint32_t hi = 1;
            for (uint32_t l = 0; l < t.bits; l++) {
                const uint32_t v = contest_u(o, levels()[l].s0, levels()[l].m2, levels()[l].h2) >> 1;
                const bool go_left = left(v, W[2 * hi] - exw[2 * hi], W[2 * hi + 1] - exw[2 * hi + 1]);
                hi = 2 * hi + (go_left ? 0u : 1u);
            }
            uint32_t w = blob[hi];
            uint64_t remain = W[hi] - exw[hi];
            while ((int32_t)w <= -2) {
                const uint32_t *p = blob + (w & 0x7FFFFFFFu) / 4;
                if (!excluded(p[4])) {
                    const uint32_t wm = node[p[4]].y;
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

// trie_table.hpp -- the HRW2 table (DESIGN.md 3.8 / 4.1) as ONE host-side builder and ONE host-side walk, plain C++.
//
// Two users: engine.cu (build_tab: the blob is copied into the pinned staging area and walked on the device by k_trie.cu) and
// client.cpp (librio_client.so: a client resolves its first hop on its own CPU by walking the very same blob).  Clients and
// servers therefore cannot disagree about the table, and the CPU test-suite of the client library (tests/test_client_first_hop.py,
// against the oracle) exercises the builder the GPU path depends on.
//
// Blob layout (all offsets in bytes, 32-bit little-endian words):
//   [0, 4 << bits)                 thresholds T3 of the trie nodes in heap order (index 1 = root; word 0 unused)
//   [4 << bits, 8 << bits)         leaf words, one per bucket: a node index | 0x80000000 + byte offset of the bucket's first chain
//                                  record | kNone (no live node in the bucket)
//   off_crec (16-byte aligned)     chain records, 32 bytes each, k-1 for a bucket of k nodes: {s0, m2, h2, T3} of the member-keyed
//                                  contest "this member against the rest", then {this member's node index, next, 0, 0}; next = the
//                                  LAST member's node index when only that one is left (it would always be taken), else
//                                  0x80000000 + byte offset of the next record
#pragma once
#include <algorithm>
#include <cstdint>
#include <memory>
#include <vector>

#include "spec.cuh"

namespace rio {

struct TrieMember {
    uint64_t seed;     // seed(address), DESIGN.md 3.1
    uint32_t idx;      // the index a walk returns for this member
    uint32_t weight;   // > 0 (only live members are listed)
};

struct TrieBlob {
    std::vector<uint32_t> words;   // the blob; words.size() * 4 == blob_bytes, a multiple of 16
    uint32_t blob_bytes = 0;
    uint32_t off_crec = 0;         // byte offset of the first chain record
    uint32_t n_chain = 0;          // chain records
    uint32_t bits = 0;
    std::vector<uint64_t> wsum;    // heap of subtree weights the thresholds were derived from (index 1 = root, buckets at [2^bits, 2^(bits+1)));
                                   // not part of the blob: the ranked walk (DESIGN.md 3.9) re-derives the contests that exclusions change
};

// T3 of a contest (spec.cuh contest_t3) for the common case "both weights and their sum below 2^32": floor(2^31 wl / (wl + wr)) by one
// double-precision division and an exact integer correction instead of a 64-bit hardware division (~25-40 ns each on server CPUs; a
// table rebuild does one per trie node with two non-empty subtrees and one per chain record).  q0 is within 1 of the true quotient (the
// operands are exact in a double, the quotient <= 2^31 has 22 bits of slack), the two loops make it exact; everything else falls back
// to the reference form.  tests/test_client_first_hop.py compares both forms on edge and random operands.
inline uint32_t contest_t3_fast(uint64_t wl, uint64_t wr) {
    if (wl == 0) return 0u;
    if (wr == 0) return 0xFFFFFFFFu;
    const uint64_t s = wl + wr;
    if (s >= (1ull << 32)) return contest_t3(wl, wr);
    const uint64_t num = wl << 31;                                  // < 2^63
    uint64_t q = (uint64_t)((double)num / (double)s);
    while (q * s > num) q--;                                        // q * s <= 2^31 * 2^32: no overflow
    while ((q + 1) * s <= num) q++;
    return q ? (uint32_t)(2 * q - 1) : 0u;
}

// Members in any order: positions and chains are ordered by (pos(seed), idx), so the table is a function of the member SET.
inline TrieBlob build_trie_blob(const std::vector<TrieMember> &members, uint32_t bits) {
    const uint32_t nb = 1u << bits;
    struct Mem { uint64_t pos; uint64_t seed; uint32_t idx, w; };
    // Order by (pos, idx) without a full sort: the bucket is the top `bits` bits of pos, so members are dropped into their buckets by
    // counting (two linear passes) and only the few buckets that hold more than one member are sorted.
    std::vector<uint32_t> bstart((size_t)nb + 1, 0);
    std::vector<Mem> all;
    all.reserve(members.size());
    for (const TrieMember &m : members) {
        if (!m.weight) continue;
        const uint64_t pos = mix64(m.seed ^ kSaltPos);
        all.push_back(Mem{pos, m.seed, m.idx, m.weight});
        bstart[(bits ? (uint32_t)(pos >> (64 - bits)) : 0u) + 1]++;
    }
    for (uint32_t k = 0; k < nb; k++) bstart[k + 1] += bstart[k];
    std::unique_ptr<Mem[]> mem(new Mem[all.size() ? all.size() : 1]);     // every element is written below
    {
        std::vector<uint32_t> fill(bstart.begin(), bstart.end() - 1);
        for (const Mem &m : all) mem[fill[bits ? (uint32_t)(m.pos >> (64 - bits)) : 0u]++] = m;
    }
    std::vector<uint64_t> wsum((size_t)2 * nb, 0);                 // heap of subtree weights, leaves at [nb, 2nb)
    uint32_t n_rec = 0;                                            // chain records: k-1 for a bucket of k >= 2 members
    for (uint32_t k = 0; k < nb; k++) {
        const uint32_t lo = bstart[k], hi = bstart[k + 1];
        if (hi - lo > 1) {
            std::sort(mem.get() + lo, mem.get() + hi, [](const Mem &a, const Mem &b) { return a.pos != b.pos ? a.pos < b.pos : a.idx < b.idx; });
            n_rec += hi - lo - 1;
        }
        uint64_t sum = 0;
        for (uint32_t q = lo; q < hi; q++) sum += mem[q].w;
        wsum[nb + k] = sum;
    }
    for (uint32_t i = nb - 1; i >= 1; i--) wsum[i] = wsum[2 * i] + wsum[2 * i + 1];
    TrieBlob b;
    b.bits = bits;
    b.off_crec = (uint32_t)(((size_t)2 * nb * 4 + 15) / 16 * 16);
    b.n_chain = n_rec;
    b.blob_bytes = std::max<uint32_t>(16u, b.off_crec + n_rec * 32u);
    b.words.assign(b.blob_bytes / 4, 0u);                          // thresholds, leaves and records are written in place
    uint32_t *w32 = b.words.data();
    for (uint32_t i = 1; i < nb; i++) w32[i] = contest_t3_fast(wsum[2 * i], wsum[2 * i + 1]);
    uint32_t rec_off = b.off_crec;                                 // byte offset of the next chain record
    for (uint32_t k = 0; k < nb; k++) {
        const uint32_t lo = bstart[k], hi = bstart[k + 1];
        if (lo == hi) { w32[nb + k] = kNone; continue; }
        if (hi - lo == 1) { w32[nb + k] = mem[lo].idx; continue; }
        w32[nb + k] = 0x80000000u | rec_off;                       // the chain's first record
        uint64_t rest = wsum[nb + k];
        for (uint32_t q = lo; q + 1 < hi; q++, rec_off += 32u) {   // the last member needs no record: it is always taken
            rest -= mem[q].w;
            const ContestRec r = contest_rec(mem[q].seed);
            uint32_t *d = w32 + rec_off / 4;
            d[0] = r.s0; d[1] = r.m2; d[2] = r.h2; d[3] = contest_t3_fast(mem[q].w, rest);
            d[4] = mem[q].idx;
            d[5] = q + 2 == hi ? mem[hi - 1].idx : 0x80000000u | (rec_off + 32u);
        }
    }
    b.wsum = std::move(wsum);
    return b;
}

// Per-level contest constants (pseudo-node seeds c_l): spec constants, the same for every table.
inline std::vector<ContestRec> trie_level_constants(uint32_t levels) {
    std::vector<ContestRec> v(levels);
    for (uint32_t l = 0; l < levels; l++) v[l] = contest_rec(level_seed(l));
    return v;
}

// One object's walk over the blob on the host -- statement for statement what k_trie.cu's trie_leaf_index + trie_resolve_leaf do.
inline uint32_t trie_walk_host(const uint32_t *blob, uint32_t bits, const ContestRec *level, ObjHash o) {
    uint32_t i = 1;
    for (uint32_t l = 0; l < bits; l++) i = 2 * i + (contest_u(o, level[l].s0, level[l].m2, level[l].h2) > blob[i] ? 1u : 0u);
    uint32_t w = blob[i];
    if ((int32_t)w > -2) return w;                 // node index (top bit clear) or kNone
    for (;;) {
        const uint32_t *p = blob + (w & 0x7FFFFFFFu) / 4;
        if (contest_u(o, p[0], p[1], p[2]) <= p[3]) return p[4];
        if ((int32_t)p[5] >= 0) return p[5];
        w = p[5];
    }
}

}  // namespace rio

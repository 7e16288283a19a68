// k_trie.cu -- HRW2, the hierarchical weighted rendezvous with fan-out 2 (DESIGN.md 3.8 / 5.4).
//
// Per object: one mix64 for the hashed pair (b, ab), then `bits` contests down a binary trie over node positions
// (per contest: IMAD, IMAD for u = 2v+1, one LDS.32 of the node's threshold, ISETP, index update), one leaf word,
// and -- only in buckets that hold more than one node -- a short chain of member-keyed contests.  At M = 1024 that
// is ~13 contests instead of the 1024 pair hashes of the flat grid, so the kernel is bound by HBM (12 B/object) and
// the shared-memory gathers, not by the integer pipes.
//
// The whole table (thresholds, leaves, chain records; <= ~40 KB at bits = 12) is ONE contiguous blob that a single
// elected thread brings into shared memory with cp.async.bulk (TMA, mbarrier complete_tx); keys are read two per
// 128-bit load; node indices leave as 64-bit stores.
#include "kernels.cuh"
#include "spec.cuh"
#include "bounded_tail.cuh"

#include <cstdlib>

namespace rio {

namespace {

constexpr int kTrieThreads = 256;
constexpr uint32_t kMaxLevels = 16;          // trie_bits <= 14; the table has two spare entries

// Per-level contest constants (pseudo-node seeds c_l, DESIGN.md 3.8): spec constants, identical for every handle.
__constant__ uint32_t c_lvl_s0[kMaxLevels];
__constant__ uint32_t c_lvl_m2[kMaxLevels];
__constant__ uint32_t c_lvl_h2[kMaxLevels];

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// Bring `bytes` (multiple of 16) from global to shared memory with the TMA bulk-copy engine and wait for it.
// Called by every thread of the block; one thread issues.  `bar` is an 8-byte shared mbarrier used once (phase 0).
__device__ __forceinline__ void stage_blob_tma(void *smem_dst, const void *gsrc, uint32_t bytes, unsigned long long *bar) {
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(bar)) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
        // chunks of at most 32 KB: one bulk copy each, all completing on the same mbarrier
        for (uint32_t off = 0; off < bytes; off += 32768u) {
            const uint32_t len = min(32768u, bytes - off);
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         ::"r"(smem_u32(reinterpret_cast<unsigned char *>(smem_dst) + off)),
                           "l"(reinterpret_cast<const unsigned char *>(gsrc) + off), "r"(len), "r"(smem_u32(bar))
                         : "memory");
        }
    }
    uint32_t done = 0;
    while (!done) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(smem_u32(bar)), "r"(0u) : "memory");
    }
}

// off' = 2 off + sel as ONE multiply-add: keeps the update on the FMA pipe (the ALU pipe carries the compare and the select)
__device__ __forceinline__ uint32_t walk_step(uint32_t off, uint32_t sel) {
    uint32_t r;
    asm("mad.lo.u32 %0, %1, 2, %2;" : "=r"(r) : "r"(off), "r"(sel));
    return r;
}

// One object's walk.  tab32 = thresholds [0, 2^bits) then leaves [2^bits, 2^(bits+1)); the running heap index i starts
// at 1, so after `bits` contests tab32[i] IS the leaf word.  RIGHT iff u > T3 (u = 2v+1, T3 = max(2T-1, 0)).
template <int BITS>
__device__ __forceinline__ uint32_t trie_leaf_index(ObjHash o, const uint32_t *__restrict__ tab32, uint32_t bits_rt) {
    uint32_t i = 1;
    if (BITS > 0) {
#pragma unroll
        for (int l = 0; l < BITS; l++) {
            const uint32_t u = contest_u(o, c_lvl_s0[l], c_lvl_m2[l], c_lvl_h2[l]);
            i = 2 * i + (u > tab32[i] ? 1u : 0u);
        }
    } else {
        for (uint32_t l = 0; l < bits_rt; l++) {
            const uint32_t u = contest_u(o, c_lvl_s0[l], c_lvl_m2[l], c_lvl_h2[l]);
            i = 2 * i + (u > tab32[i] ? 1u : 0u);
        }
    }
    return i;
}

// leaf word: kNone = empty bucket (only without live nodes), top bit = chain start (low bits: BYTE offset of the first
// chain record inside the blob), else the node index.  A chain of k members has k-1 records of 32 bytes:
// {s0, m2, h2, T3} {this member's node index, next, 0, 0}; `next` is the LAST member's node index when only that one is
// left (it would always be taken) and 0x80000000 | byte offset of the next record otherwise.
__device__ __forceinline__ uint32_t trie_resolve_leaf(ObjHash o, uint32_t leaf, const unsigned char *__restrict__ blob) {
    if ((int32_t)leaf > -2) return leaf;           // node index (top bit clear) or kNone
    uint32_t w = leaf;
    for (;;) {
        const unsigned char *p = blob + (w & 0x7FFFFFFFu);
        const uint4 r = *reinterpret_cast<const uint4 *>(p);
        const uint2 nn = *reinterpret_cast<const uint2 *>(p + 16);
        if (contest_u(o, r.x, r.y, r.z) <= r.w) return nn.x;
        if ((int32_t)nn.y >= 0) return nn.y;
        w = nn.y;
    }
}

struct TrieSmem {
    const uint32_t *tab32;          // == the blob: thresholds, leaves, then the chain records
    const unsigned char *blob;
    uint32_t *hist;
};

// Shared-memory layout: [blob (tab32 | chain records)] [hist bins] [mbarrier].  Falls back to the table in global memory
// (through the read-only path) when the blob does not fit beside the histogram.
template <bool SMEM>
__device__ __forceinline__ TrieSmem trie_stage(const TrieDev &t, uint32_t hist_bins) {
    extern __shared__ __align__(128) unsigned char smem_trie[];
    constexpr bool in_smem = SMEM;
    TrieSmem s;
    uint32_t off = 0;
    if (in_smem) {
        s.tab32 = reinterpret_cast<const uint32_t *>(smem_trie);
        s.blob = smem_trie;
        off = t.blob_bytes;
    } else {
        const unsigned char *g = reinterpret_cast<const unsigned char *>(t.blob);
        s.tab32 = reinterpret_cast<const uint32_t *>(g);
        s.blob = g;
    }
    s.hist = reinterpret_cast<uint32_t *>(smem_trie + off);
    for (uint32_t j = threadIdx.x; j < hist_bins; j += blockDim.x) s.hist[j] = 0;
    unsigned long long *bar = reinterpret_cast<unsigned long long *>(smem_trie + off + ((hist_bins * 4u + 15u) & ~15u));
    if (in_smem) stage_blob_tma(smem_trie, t.blob, t.blob_bytes, bar);   // contains the __syncthreads that publishes hist = 0
    else __syncthreads();
    return s;
}

// ---- dense assign: thread owns 2 consecutive objects per 128-bit key load, OPT/2 such loads per tile ----------------
// MODE 0: plain assign (+ fused histogram).  MODE 1: re-assign and compare with the previous assignment (rebalance):
// only changed indices are written, `moved` counts them.
template <int BITS, int OPT, int MODE, bool SMEM, int MINB = (SMEM ? 5 : 3)>
__global__ void __launch_bounds__(kTrieThreads, MINB)
k_assign_trie(const uint64_t *__restrict__ keys, uint64_t n, TrieDev t, uint32_t *__restrict__ out_idx, uint32_t *__restrict__ counters,
              uint32_t hist_bins, unsigned long long *__restrict__ moved, const __grid_constant__ BoundedTail tail) {
    static_assert(OPT % 2 == 0, "two objects per 128-bit load");
    constexpr bool in_smem = SMEM;
    constexpr int SEG = OPT / 2;
    const uint64_t tile_objs = (uint64_t)kTrieThreads * OPT;
    const uint64_t n_tiles = (n + tile_objs - 1) / tile_objs;
    unsigned long long n_moved = 0;
    // keys of the NEXT tile are requested before the current tile is walked: the walk (~170 instructions per object)
    // hides the HBM latency of the stream even at 5 CTAs per SM
    ulonglong2 kk[SEG];
    // A tile that lies wholly inside [0, n) -- all but the last -- takes the straight path: no per-load / per-store bound checks
    auto load_tile = [&](uint64_t tile) {
        const uint64_t f0 = tile * tile_objs + 2 * threadIdx.x;
        if ((tile + 1) * tile_objs <= n) {
            const ulonglong2 *src = reinterpret_cast<const ulonglong2 *>(keys + f0);   // keys is 256-byte aligned, f0 is even
#pragma unroll
            for (int g = 0; g < SEG; g++) kk[g] = __ldg(src + g * kTrieThreads);
            return;
        }
#pragma unroll
        for (int g = 0; g < SEG; g++) {
            const uint64_t f = f0 + (uint64_t)g * (2 * kTrieThreads);
            kk[g] = make_ulonglong2(0, 0);
            if (f + 1 < n) kk[g] = __ldg(reinterpret_cast<const ulonglong2 *>(keys + f));
            else if (f < n) kk[g].x = __ldg(keys + f);
        }
    };
    // Programmatic dependent launch: this grid may be scheduled while the previous kernel of the stream is still draining.  The
    // table (written by copies only, never by a kernel) is staged first; nothing a previous KERNEL may have produced -- keys,
    // counters, indices -- is touched before griddepcontrol.wait, which returns once that kernel has completed and flushed.
    // Both instructions are no-ops for a launch without the attribute.
    const TrieSmem s = trie_stage<SMEM>(t, hist_bins);
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (blockIdx.x < n_tiles) load_tile(blockIdx.x);
    for (uint64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const uint64_t base = tile * tile_objs;
        const bool full_tile = base + tile_objs <= n;
        ObjHash o[OPT];
#pragma unroll
        for (int g = 0; g < SEG; g++) {
            o[2 * g] = obj_hash(kk[g].x);
            o[2 * g + 1] = obj_hash(kk[g].y);
        }
        if (tile + gridDim.x < n_tiles) load_tile(tile + gridDim.x);
        uint32_t leaf[OPT];
        if (in_smem) {
            // byte offset of the walk inside the table: off' = 2 off + (RIGHT ? 4 : 0), starting at heap index 1
            const unsigned char *tb = reinterpret_cast<const unsigned char *>(s.tab32);
            uint32_t off[OPT];
#pragma unroll
            for (int k = 0; k < OPT; k++) off[k] = 4;
            // level-major: the OPT walks of a thread interleave, so every LDS has OPT-1 independent ones behind it
            if (BITS > 0) {
                // The seven thresholds of levels 0-2 travel as kernel parameters (constant bank, uniform registers): those
                // contests cost selects instead of shared-memory wavefronts -- the LDS data pipe is this kernel's limiter
                constexpr int TOP = BITS >= 3 ? 3 : 0;
                if (TOP) {
#pragma unroll
                    for (int k = 0; k < OPT; k++) {
                        const bool c0 = contest_u(o[k], c_lvl_s0[0], c_lvl_m2[0], c_lvl_h2[0]) > t.top[1];
                        const bool c1 = contest_u(o[k], c_lvl_s0[1], c_lvl_m2[1], c_lvl_h2[1]) > (c0 ? t.top[3] : t.top[2]);
                        const uint32_t t2 = c0 ? (c1 ? t.top[7] : t.top[6]) : (c1 ? t.top[5] : t.top[4]);
                        const bool c2 = contest_u(o[k], c_lvl_s0[2], c_lvl_m2[2], c_lvl_h2[2]) > t2;
                        off[k] = 32u + (c0 ? 16u : 0u) + (c1 ? 8u : 0u) + (c2 ? 4u : 0u);
                    }
                }
#pragma unroll
                for (int l = TOP; l < BITS; l++) {
#pragma unroll
                    for (int k = 0; k < OPT; k++) {
                        const uint32_t u = contest_u(o[k], c_lvl_s0[l], c_lvl_m2[l], c_lvl_h2[l]);
                        const uint32_t thr = *reinterpret_cast<const uint32_t *>(tb + off[k]);
                        off[k] = walk_step(off[k], u > thr ? 4u : 0u);
                    }
                }
            } else {
                for (uint32_t l = 0; l < t.bits; l++) {
#pragma unroll
                    for (int k = 0; k < OPT; k++) {
                        const uint32_t u = contest_u(o[k], c_lvl_s0[l], c_lvl_m2[l], c_lvl_h2[l]);
                        const uint32_t thr = *reinterpret_cast<const uint32_t *>(tb + off[k]);
                        off[k] = walk_step(off[k], u > thr ? 4u : 0u);
                    }
                }
            }
#pragma unroll
            for (int k = 0; k < OPT; k++) leaf[k] = *reinterpret_cast<const uint32_t *>(tb + off[k]);
        } else {
#pragma unroll
            for (int k = 0; k < OPT; k++) leaf[k] = __ldg(s.tab32 + trie_leaf_index<0>(o[k], s.tab32, t.bits));
        }
        uint32_t nid[OPT];
#pragma unroll
        for (int k = 0; k < OPT; k++) nid[k] = trie_resolve_leaf(o[k], leaf[k], s.blob);
        if (MODE == 0 && full_tile) {
            uint2 *dst = reinterpret_cast<uint2 *>(out_idx + base + 2 * threadIdx.x);
#pragma unroll
            for (int g = 0; g < SEG; g++) dst[g * kTrieThreads] = make_uint2(nid[2 * g], nid[2 * g + 1]);
            // kNone leaves exist only when NO node is live (the walk never enters an empty subtree otherwise): one test covers the tile
            if (counters && nid[0] != kNone) {
                if (hist_bins) {
#pragma unroll
                    for (int k = 0; k < OPT; k++) atomicAdd(&s.hist[nid[k]], 1u);
                } else {
#pragma unroll
                    for (int k = 0; k < OPT; k++) atomicAdd(&counters[nid[k]], 1u);
                }
            }
            continue;
        }
#pragma unroll
        for (int g = 0; g < SEG; g++) {
            const uint64_t first = base + (uint64_t)g * (2 * kTrieThreads) + 2 * threadIdx.x;
            if (first >= n) continue;
            const bool two = first + 1 < n;
            if (MODE == 1) {
                uint2 old = make_uint2(kNone, kNone);
                if (two) old = *reinterpret_cast<const uint2 *>(out_idx + first);
                else old.x = out_idx[first];
                const bool c0 = old.x != nid[2 * g], c1 = two && old.y != nid[2 * g + 1];
                if (c0 | c1) {
                    if (two) *reinterpret_cast<uint2 *>(out_idx + first) = make_uint2(nid[2 * g], nid[2 * g + 1]);
                    else out_idx[first] = nid[2 * g];
                }
                n_moved += (unsigned)c0 + (unsigned)c1;
            } else {
                if (two) *reinterpret_cast<uint2 *>(out_idx + first) = make_uint2(nid[2 * g], nid[2 * g + 1]);
                else out_idx[first] = nid[2 * g];
            }
            if (counters) {
                if (hist_bins) {
                    if (nid[2 * g] != kNone) atomicAdd(&s.hist[nid[2 * g]], 1u);
                    if (two && nid[2 * g + 1] != kNone) atomicAdd(&s.hist[nid[2 * g + 1]], 1u);
                } else {
                    if (nid[2 * g] != kNone) atomicAdd(&counters[nid[2 * g]], 1u);
                    if (two && nid[2 * g + 1] != kNone) atomicAdd(&counters[nid[2 * g + 1]], 1u);
                }
            }
        }
    }
    if (MODE == 1) {
#pragma unroll
        for (int sh = 16; sh > 0; sh >>= 1) n_moved += __shfl_xor_sync(0xFFFFFFFFu, n_moved, sh);
        if ((threadIdx.x & 31) == 0 && n_moved) atomicAdd(moved, n_moved);
    }
    if (hist_bins && counters) {
        __syncthreads();
        for (uint32_t j = threadIdx.x; j < hist_bins; j += blockDim.x) { const uint32_t v = s.hist[j]; if (v) atomicAdd(&counters[j], v); }
    }
    if (MODE == 0 && tail.enabled) {
        // the pass's exchange + capacity check, in whichever CTA finishes last: its atomics on `counters` are ordered before its
        // ticket, and the last CTA reads the counters through L2 after taking the last ticket
        __shared__ uint32_t s_last;
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) s_last = atomicAdd(tail.ticket, 1u) == gridDim.x - 1;
        __syncthreads();
        if (s_last) {
            if (threadIdx.x == 0) *tail.ticket = 0;
            __threadfence();
            exchange_and_check_block(tail, counters);
        }
    }
}

// ---- gathered assign (a compact list of object positions: bounded-load spill rounds, place_batch) ---------------
template <bool SMEM>
__global__ void __launch_bounds__(kTrieThreads, 4)
k_assign_trie_sel(const uint64_t *__restrict__ keys, const uint32_t *__restrict__ sel, uint64_t n_sel, TrieDev t, uint32_t *__restrict__ out_idx,
                  uint32_t *__restrict__ counters, uint32_t hist_bins) {
    const TrieSmem s = trie_stage<SMEM>(t, hist_bins);
    for (uint64_t q = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; q < n_sel; q += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t oi = __ldg(sel + q);
        const ObjHash o = obj_hash(__ldg(keys + oi));
        const uint32_t i = trie_leaf_index<0>(o, s.tab32, t.bits);
        const uint32_t nid = trie_resolve_leaf(o, s.tab32[i], s.blob);
        out_idx[oi] = nid;
        if (counters && nid != kNone) { if (hist_bins) atomicAdd(&s.hist[nid], 1u); else atomicAdd(&counters[nid], 1u); }
    }
    if (hist_bins && counters) {
        __syncthreads();
        for (uint32_t j = threadIdx.x; j < hist_bins; j += blockDim.x) { const uint32_t v = s.hist[j]; if (v) atomicAdd(&counters[j], v); }
    }
}

// ---- directory-wide re-placement under HRW2 (eager rebalance after a membership event): streaming over the slots,
// every placed key is walked again and rewritten only if its node changed.  16 B/slot, HBM bound. -------------------
template <bool SMEM>
__global__ void __launch_bounds__(kTrieThreads, 4)
k_dir_reassign_trie(DirDev dir, TrieDev t, unsigned long long *__restrict__ moved) {
    const TrieSmem s = trie_stage<SMEM>(t, 0);
    const uint4 *slots = reinterpret_cast<const uint4 *>(dir.slots);
    const uint64_t cap = dir.mask + 1;
    unsigned long long n_moved = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint4 v = slots[i];
        const unsigned long long key = ((unsigned long long)v.y << 32) | v.x;
        if (key == kEmptyKey || v.z == kNone) continue;
        const ObjHash o = obj_hash(key);
        const uint32_t li = trie_leaf_index<0>(o, s.tab32, t.bits);
        const uint32_t nid = trie_resolve_leaf(o, s.tab32[li], s.blob);
        if (nid != v.z) { reinterpret_cast<uint32_t *>(&dir.slots[i].val)[0] = nid; n_moved++; }
    }
#pragma unroll
    for (int sh = 16; sh > 0; sh >>= 1) n_moved += __shfl_xor_sync(0xFFFFFFFFu, n_moved, sh);
    if ((threadIdx.x & 31) == 0 && n_moved) atomicAdd(moved, n_moved);
}

constexpr uint32_t kTrieSmemBudget = 200u * 1024u;   // blob + histogram + barrier must fit under this to be staged

struct TrieLaunchShape { uint32_t hist_bins; uint32_t in_smem; size_t smem; int ctas_per_sm; };
TrieLaunchShape trie_shape(const TrieDev &t, bool want_hist, uint32_t n_total, int want_ctas) {
    TrieLaunchShape sh{};
    sh.hist_bins = (want_hist && n_total <= 8192) ? n_total : 0;
    const size_t tail = ((size_t)sh.hist_bins * 4 + 15) / 16 * 16 + 16;
    sh.in_smem = (t.blob_bytes + tail <= kTrieSmemBudget) ? 1u : 0u;
    sh.smem = (sh.in_smem ? t.blob_bytes : 0) + tail;
    int c = want_ctas;
    while (c > 1 && (size_t)c * (sh.smem + 1024) > 227u * 1024u) c--;
    sh.ctas_per_sm = c;
    return sh;
}

bool g_lvl_uploaded[64] = {};

}  // namespace

// Per-level constants are spec constants: upload once per device.
void trie_upload_level_constants(int device) {
    if (device >= 0 && device < 64 && g_lvl_uploaded[device]) return;
    uint32_t s0[kMaxLevels], m2[kMaxLevels], h2[kMaxLevels];
    for (uint32_t l = 0; l < kMaxLevels; l++) {
        const ContestRec r = contest_rec(level_seed(l));
        s0[l] = r.s0; m2[l] = r.m2; h2[l] = r.h2;
    }
    cudaMemcpyToSymbol(c_lvl_s0, s0, sizeof s0);
    cudaMemcpyToSymbol(c_lvl_m2, m2, sizeof m2);
    cudaMemcpyToSymbol(c_lvl_h2, h2, sizeof h2);
    if (device >= 0 && device < 64) g_lvl_uploaded[device] = true;
}

uint64_t trie_wave_objects(int sm_count) { return (uint64_t)sm_count * 5 * kTrieThreads * 4; }

#define RIO_TRIE_LAUNCH(KERNEL, GRID, SMEM, ...)                                                                       \
    do {                                                                                                               \
        static bool attr_set[64] = {};   /* per device; the attribute call costs ~1 us of host time per launch otherwise */ \
        int dev__ = 0;                                                                                                 \
        cudaGetDevice(&dev__);                                                                                         \
        if (dev__ < 0 || dev__ >= 64 || !attr_set[dev__]) {                                                            \
            cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTrieSmemBudget + 1024);    \
            if (dev__ >= 0 && dev__ < 64) attr_set[dev__] = true;                                                      \
        }                                                                                                              \
        KERNEL<<<(GRID), kTrieThreads, (SMEM), L.stream>>>(__VA_ARGS__);                                               \
    } while (0)

// The dense walk is launched with programmatic stream serialization: its CTAs take the SM slots the previous kernel's CTAs free
// one by one and stage their table while that kernel drains (RIO_TRIE_PDL=0 turns the attribute off, for A/B runs).
#define RIO_TRIE_LAUNCH_PDL(KERNEL, GRID, SMEM, ...)                                                                   \
    do {                                                                                                               \
        static bool attr_set[64] = {};                                                                                 \
        static const bool pdl = [] { const char *e = getenv("RIO_TRIE_PDL"); return !(e && e[0] == '0'); }();          \
        int dev__ = 0;                                                                                                 \
        cudaGetDevice(&dev__);                                                                                         \
        if (dev__ < 0 || dev__ >= 64 || !attr_set[dev__]) {                                                            \
            cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTrieSmemBudget + 1024);    \
            if (dev__ >= 0 && dev__ < 64) attr_set[dev__] = true;                                                      \
        }                                                                                                              \
        cudaLaunchConfig_t cfg__ = {};                                                                                 \
        cfg__.gridDim = dim3((unsigned)(GRID)); cfg__.blockDim = dim3(kTrieThreads);                                   \
        cfg__.dynamicSmemBytes = (SMEM); cfg__.stream = L.stream;                                                      \
        cudaLaunchAttribute at__[1];                                                                                   \
        at__[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                                               \
        at__[0].val.programmaticStreamSerializationAllowed = 1;                                                        \
        cfg__.attrs = at__; cfg__.numAttrs = pdl ? 1 : 0;                                                              \
        cudaLaunchKernelEx(&cfg__, KERNEL, __VA_ARGS__);                                                               \
    } while (0)

void launch_assign_trie(const Launch &L, const uint64_t *d_keys, uint64_t n, const TrieDev &t, uint32_t *d_out_idx, uint32_t *d_counters,
                        const uint32_t *d_sel, uint64_t n_sel, uint32_t n_total, const BoundedTail *tail) {
    BoundedTail no_tail{};
    const BoundedTail &tl = tail ? *tail : no_tail;
    const uint64_t n_work = d_sel ? n_sel : n;
    if (!n_work) return;
    if (d_sel) {
        const TrieLaunchShape sh = trie_shape(t, d_counters != nullptr, n_total, 4);
        const uint64_t blocks = (n_work + kTrieThreads - 1) / kTrieThreads, cap = (uint64_t)L.sm_count * sh.ctas_per_sm;
        const int grid = (int)(blocks < cap ? blocks : cap);
        if (sh.in_smem) RIO_TRIE_LAUNCH(k_assign_trie_sel<true>, grid, sh.smem, d_keys, d_sel, n_work, t, d_out_idx, d_counters, sh.hist_bins);
        else RIO_TRIE_LAUNCH(k_assign_trie_sel<false>, grid, sh.smem, d_keys, d_sel, n_work, t, d_out_idx, d_counters, sh.hist_bins);
    } else {
        constexpr int OPT = 4;
#ifdef RIO_ASSIGN_TUNING   // A/B points of the walk kernel (RIO_BUILD_TUNING=1, tools/tune_trie.py): "<objects per thread><CTAs per SM>"
        if (const char *tn = getenv("RIO_TRIE_TUNE")) {
            const int code = atoi(tn);
            auto go = [&](auto kern, int opt, int minb) {
                const TrieLaunchShape sh2 = trie_shape(t, d_counters != nullptr, n_total, minb);
                const uint64_t tiles2 = (n_work + (uint64_t)kTrieThreads * opt - 1) / ((uint64_t)kTrieThreads * opt), cap2 = (uint64_t)L.sm_count * sh2.ctas_per_sm;
                cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTrieSmemBudget + 1024);
                kern<<<(int)(tiles2 < cap2 ? tiles2 : cap2), kTrieThreads, sh2.smem, L.stream>>>(d_keys, n_work, t, d_out_idx, d_counters, sh2.hist_bins, nullptr, tl);
            };
            bool done = true;
            switch (code) {
                case 25: go(k_assign_trie<12, 2, 0, true, 5>, 2, 5); break;
                case 28: go(k_assign_trie<12, 2, 0, true, 8>, 2, 8); break;
                case 44: go(k_assign_trie<12, 4, 0, true, 4>, 4, 4); break;
                case 45: go(k_assign_trie<12, 4, 0, true, 5>, 4, 5); break;
                case 63: go(k_assign_trie<12, 6, 0, true, 3>, 6, 3); break;
                case 64: go(k_assign_trie<12, 6, 0, true, 4>, 6, 4); break;
                case 83: go(k_assign_trie<12, 8, 0, true, 3>, 8, 3); break;
                default: done = false;
            }
            if (done && t.bits == 12) { RIO_COUNT_LAUNCH(L); return; }
        }
#endif
        const TrieLaunchShape sh = trie_shape(t, d_counters != nullptr, n_total, 5);
        uint64_t cap = (uint64_t)L.sm_count * sh.ctas_per_sm;
        if (L.spare_ctas > 0 && cap > (uint64_t)L.spare_ctas + 1) cap -= (uint64_t)L.spare_ctas;
        const uint64_t tiles = (n_work + (uint64_t)kTrieThreads * OPT - 1) / ((uint64_t)kTrieThreads * OPT);
        const int grid = (int)(tiles < cap ? tiles : cap);
        unsigned long long *no_moved = nullptr;
        if (!sh.in_smem) RIO_TRIE_LAUNCH_PDL((k_assign_trie<0, OPT, 0, false>), grid, sh.smem, d_keys, n_work, t, d_out_idx, d_counters, sh.hist_bins, no_moved, tl);
        else if (t.bits == 12) RIO_TRIE_LAUNCH_PDL((k_assign_trie<12, OPT, 0, true>), grid, sh.smem, d_keys, n_work, t, d_out_idx, d_counters, sh.hist_bins, no_moved, tl);
        else RIO_TRIE_LAUNCH_PDL((k_assign_trie<0, OPT, 0, true>), grid, sh.smem, d_keys, n_work, t, d_out_idx, d_counters, sh.hist_bins, no_moved, tl);
    }
    RIO_COUNT_LAUNCH(L);
}

// Re-assign a dense set after the table changed; writes only changed indices, counts them, rebuilds the counters.
void launch_reassign_trie(const Launch &L, const uint64_t *d_keys, uint64_t n, const TrieDev &t, uint32_t *d_idx, uint32_t *d_counters,
                          uint32_t n_total, unsigned long long *d_moved) {
    if (!n) return;
    constexpr int OPT = 4;
 const TrieLaunchShape sh = trie_shape(t, d_counters != nullptr, n_total, 5);
    const uint64_t tiles = (n + (uint64_t)kTrieThreads * OPT - 1) / ((uint64_t)kTrieThreads * OPT), cap = (uint64_t)L.sm_count * sh.ctas_per_sm;
    const int grid = (int)(tiles < cap ? tiles : cap);
    if (!sh.in_smem) RIO_TRIE_LAUNCH((k_assign_trie<0, OPT, 1, false>), grid, sh.smem, d_keys, n, t, d_idx, d_counters, sh.hist_bins, d_moved, BoundedTail{});
    else if (t.bits == 12) RIO_TRIE_LAUNCH((k_assign_trie<12, OPT, 1, true>), grid, sh.smem, d_keys, n, t, d_idx, d_counters, sh.hist_bins, d_moved, BoundedTail{});
    else RIO_TRIE_LAUNCH((k_assign_trie<0, OPT, 1, true>), grid, sh.smem, d_keys, n, t, d_idx, d_counters, sh.hist_bins, d_moved, BoundedTail{});
    RIO_COUNT_LAUNCH(L);
}

void launch_dir_reassign_trie(const Launch &L, const DirDev &dir, const TrieDev &t, unsigned long long *d_moved) {
    const TrieLaunchShape sh = trie_shape(t, false, 0, 4);
    const uint64_t blocks = (dir.mask + 1 + kTrieThreads - 1) / kTrieThreads, cap = (uint64_t)L.sm_count * sh.ctas_per_sm;
    const int grid = (int)(blocks < cap ? blocks : cap);
    if (sh.in_smem) RIO_TRIE_LAUNCH(k_dir_reassign_trie<true>, grid, sh.smem, dir, t, d_moved);
    else RIO_TRIE_LAUNCH(k_dir_reassign_trie<false>, grid, sh.smem, dir, t, d_moved);
    RIO_COUNT_LAUNCH(L);
}

}  // namespace rio

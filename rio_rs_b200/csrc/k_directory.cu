// k_directory.cu -- the placement directory in HBM (batched LocalObjectPlacement, local.rs:12-68) and the
// streaming rebalance kernels.  Integer/byte work, HBM-bound: one 16-byte slot per probe (a 32-byte sector holds
// two slots), 128-bit loads on the scans, warp-aggregated counters.
#include "kernels.cuh"
#include "k_changes.cuh"
#include "k_ranked_changes.cuh"
#include "k_spread_changes.cuh"
#include "k_set_commit.cuh"
#include "k_rank_common.cuh"
#include "spec.cuh"
#include "bounded_tail.cuh"

namespace rio {

namespace {

inline int grid_for(uint64_t work_items, int threads, int sm_count, int blocks_per_sm) {
    uint64_t blocks = (work_items + threads - 1) / threads;
    uint64_t cap = (uint64_t)sm_count * blocks_per_sm;
    if (blocks < 1) blocks = 1;
    return (int)(blocks < cap ? blocks : cap);
}

__device__ __forceinline__ unsigned long long norm_key(uint64_t k) {
    // kEmptyKey is reserved for free slots: fold it onto its neighbour (documented, DESIGN.md 4.2)
    return k == kEmptyKey ? kEmptyKey - 1 : k;
}
__device__ __forceinline__ uint64_t home_slot(unsigned long long key, const DirDev &d) {
    return (key * kGolden64) >> d.shift;   // Fibonacci hashing: keys may be raw user u64s
}

__device__ __forceinline__ void warp_add(unsigned long long *ctr, bool pred) {
    const unsigned m = __ballot_sync(0xFFFFFFFFu, pred);
    if (m && (threadIdx.x & 31) == (unsigned)(__ffs(m) - 1)) atomicAdd(ctr, (unsigned long long)__popc(m));
}

// End-of-kernel variant for high hit rates: each thread accumulates locally over its grid-stride loop, then one atomic per warp.
__device__ __forceinline__ void warp_flush(unsigned long long *ctr, unsigned long long local) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xFFFFFFFFu, local, o);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(ctr, local);
}

__global__ void k_dir_init(DirSlot *slots, uint64_t cap) {
    uint4 *p = reinterpret_cast<uint4 *>(slots);
    const uint4 e = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0u);  // key = EMPTY, val = (0 << 32) | NONE
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (uint64_t)gridDim.x * blockDim.x) p[i] = e;
}

// The directory's answer for a normalised key whose home slot sl holds x (the first probe, already loaded): the node of its slot,
// kNone for an absent or removed key.
__device__ __forceinline__ uint32_t dir_answer(const uint4 *slots, const DirDev &dir, unsigned long long key, uint64_t sl, uint4 x) {
    uint32_t res = kNone;
    for (uint64_t probes = 0; probes <= dir.mask; probes++) {
        const unsigned long long k = ((unsigned long long)x.y << 32) | x.x;
        if (k == key) { res = x.z; break; }
        if (k == kEmptyKey) break;
        sl = (sl + 1) & dir.mask;
        x = slots[sl];
    }
    return res;
}

// lookup (local.rs:42-49).  Random 16-byte probes are latency bound (ncu: long_scoreboard), so every thread keeps four
// independent first probes in flight; the rare longer probe sequences are finished one by one afterwards.
constexpr int kLookupIlp = 4;
__global__ void __launch_bounds__(256)
k_dir_lookup(DirDev dir, const uint64_t *__restrict__ keys, uint64_t n, uint32_t *__restrict__ out) {
    const uint4 *slots = reinterpret_cast<const uint4 *>(dir.slots);
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < n; i0 += stride * kLookupIlp) {
        unsigned long long key[kLookupIlp];
        uint64_t s[kLookupIlp];
        uint4 v[kLookupIlp];
#pragma unroll
        for (int q = 0; q < kLookupIlp; q++) {
            const uint64_t i = i0 + q * stride;
            key[q] = norm_key(i < n ? __ldg(keys + i) : 0);
            s[q] = home_slot(key[q], dir);
        }
#pragma unroll
        for (int q = 0; q < kLookupIlp; q++) v[q] = slots[s[q]];   // four independent 16-byte probes in flight
#pragma unroll
        for (int q = 0; q < kLookupIlp; q++) {
            const uint64_t i = i0 + q * stride;
            if (i >= n) continue;
            out[i] = dir_answer(slots, dir, key[q], s[q], v[q]);
        }
    }
}

// ---- delta commit of a resident set (DESIGN.md 3.20) ----
// The diff pass: one block per kCommitRows rows, row lo + q * 256 + t in thread t's q-th probe, so each warp reads 32 consecutive keys
// and idx per probe round.  As in k_dir_lookup every thread keeps kLookupIlp first probes in flight.  Per row: 8 B of key, 4 B of idx,
// one probe (a 32-byte sector), one flag byte written; 4 B of `from` for a selected row only, so an unchanged set writes no more.
static_assert(kCommitRows == 256 * kLookupIlp, "a block of the diff pass is 256 threads x kLookupIlp rows");
__global__ void __launch_bounds__(256)
k_commit_diff(DirDev dir, const uint64_t *__restrict__ keys, const uint32_t *__restrict__ idx, uint64_t n, uint8_t *__restrict__ flag,
              uint32_t *__restrict__ from, uint32_t *__restrict__ block_cnt) {
    const uint4 *slots = reinterpret_cast<const uint4 *>(dir.slots);
    const uint64_t i0 = (uint64_t)blockIdx.x * kCommitRows + threadIdx.x;
    unsigned long long key[kLookupIlp];
    uint64_t s[kLookupIlp];
    uint32_t to[kLookupIlp];
    uint4 v[kLookupIlp];
#pragma unroll
    for (int q = 0; q < kLookupIlp; q++) {
        const uint64_t i = i0 + q * 256;
        key[q] = norm_key(i < n ? __ldg(keys + i) : 0);
        to[q] = i < n ? __ldg(idx + i) : kNone;
        s[q] = home_slot(key[q], dir);
    }
#pragma unroll
    for (int q = 0; q < kLookupIlp; q++) v[q] = slots[s[q]];
    uint32_t cnt = 0;
#pragma unroll
    for (int q = 0; q < kLookupIlp; q++) {
        const uint64_t i = i0 + q * 256;
        bool sel = false;
        if (i < n) {
            const uint32_t res = dir_answer(slots, dir, key[q], s[q], v[q]);
            sel = res != to[q];
            flag[i] = sel ? 1 : 0;
            if (sel) from[i] = res;
        }
        cnt += (uint32_t)__syncthreads_count(sel);
    }
    if (threadIdx.x == 0) block_cnt[blockIdx.x] = cnt;
}

// One block: the exclusive offsets of the blocks' selected counts and their total.  Thread t sums a contiguous run of blocks, so the
// counts are read twice (8 B per kCommitRows rows).
__global__ void __launch_bounds__(1024)
k_commit_scan(const uint32_t *__restrict__ block_cnt, uint64_t nb, uint32_t *__restrict__ block_off, unsigned long long *__restrict__ total) {
    __shared__ uint32_t ws[32];
    const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const uint64_t per = (nb + 1023) / 1024, b0 = threadIdx.x * per, b1 = b0 + per < nb ? b0 + per : nb;
    uint32_t mine = 0;
    for (uint64_t b = b0; b < b1; b++) mine += __ldg(block_cnt + b);
    uint32_t x = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, x, o);
        if (lane >= (unsigned)o) x += t;
    }
    if (lane == 31) ws[w] = x;
    __syncthreads();
    if (w == 0) {
        uint32_t y = ws[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, y, o);
            if (lane >= (unsigned)o) y += t;
        }
        ws[lane] = y;
    }
    __syncthreads();
    uint32_t off = x - mine + (w ? ws[w - 1] : 0u);
    for (uint64_t b = b0; b < b1; b++) {
        block_off[b] = off;
        off += __ldg(block_cnt + b);
    }
    if (threadIdx.x == 0) *total = ws[31];
}

// The manifest: one block per kCommitRows rows, with the diff pass's row layout.  Positions come from the block's offset, the selected
// rows of the earlier probe rounds and warps of the block (ballots), and the thread's rank in its warp, so the manifest is in row order
// with no atomics.  A block with nothing selected reads only its count.
__global__ void __launch_bounds__(256)
k_commit_list(const uint64_t *__restrict__ keys, const uint32_t *__restrict__ idx, uint64_t n, const uint8_t *__restrict__ flag,
              const uint32_t *__restrict__ from, const uint32_t *__restrict__ block_cnt, const uint32_t *__restrict__ block_off,
              uint64_t *__restrict__ out_rows, uint64_t *__restrict__ out_keys, uint32_t *__restrict__ out_from, uint32_t *__restrict__ out_to) {
    __shared__ uint32_t wc[kLookupIlp][8];
    if (__ldg(block_cnt + blockIdx.x) == 0) return;
    const unsigned lane = threadIdx.x & 31, w = threadIdx.x >> 5, below = (1u << lane) - 1u;
    const uint64_t i0 = (uint64_t)blockIdx.x * kCommitRows + threadIdx.x;
    bool sel[kLookupIlp];
    unsigned bal[kLookupIlp];
#pragma unroll
    for (int q = 0; q < kLookupIlp; q++) {
        const uint64_t i = i0 + q * 256;
        sel[q] = i < n && flag[i] != 0;
        bal[q] = __ballot_sync(0xFFFFFFFFu, sel[q]);
        if (lane == 0) wc[q][w] = __popc(bal[q]);
    }
    __syncthreads();
    uint32_t base = __ldg(block_off + blockIdx.x);
#pragma unroll
    for (int q = 0; q < kLookupIlp; q++) {
        uint32_t before = 0, all = 0;
        for (unsigned u = 0; u < 8; u++) {
            const uint32_t c = wc[q][u];
            before += u < w ? c : 0u;
            all += c;
        }
        if (sel[q]) {
            const uint64_t i = i0 + q * 256;
            const uint32_t p = base + before + __popc(bal[q] & below);
            out_rows[p] = i;
            out_keys[p] = __ldg(keys + i);
            out_from[p] = __ldg(from + i);
            out_to[p] = __ldg(idx + i);
        }
        base += all;
    }
}

// update (local.rs:22-40), batched.  Claim-or-find the slot with a 64-bit CAS on the key, then order duplicate keys with a
// 64-bit atomicMax on (seq << 32 | node): seq = seq_base + position + 1 grows monotonically across batches, so within a batch
// the last one in array order wins and a later batch always beats an earlier one.  Readers look at the low word only.  When
// the 32-bit sequence space is about to wrap the host runs k_dir_clear_seq once (a streaming pass).
__global__ void __launch_bounds__(256)
k_dir_upsert(DirDev dir, const uint64_t *__restrict__ keys, const uint32_t *__restrict__ idx, uint32_t const_idx, uint64_t n, uint32_t seq_base,
             unsigned long long *new_keys, uint32_t *error) {
    unsigned long long n_fresh = 0;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        if (i < n) {
            const unsigned long long key = norm_key(__ldg(keys + i));
            const uint32_t node = idx ? __ldg(idx + i) : const_idx;
            uint64_t s = home_slot(key, dir);
            bool placed = false;
            for (uint64_t probes = 0; probes <= dir.mask; probes++) {
                unsigned long long k = *reinterpret_cast<volatile unsigned long long *>(&dir.slots[s].key);
                if (k == kEmptyKey) {
                    k = atomicCAS(&dir.slots[s].key, kEmptyKey, key);
                    if (k == kEmptyKey) { n_fresh++; k = key; }
                }
                if (k == key) { placed = true; break; }
                s = (s + 1) & dir.mask;
            }
            if (placed) atomicMax(&dir.slots[s].val, ((unsigned long long)(seq_base + (uint32_t)i + 1u) << 32) | node);
            else atomicExch(error, 1u);   // table full: the host sizes the table so this cannot happen
        }
    }
    warp_flush(new_keys, n_fresh);   // whole warp reaches this point (the base loop is block-uniform)
}
__global__ void __launch_bounds__(256) k_dir_clear_seq(DirDev dir) {
    const uint64_t cap = dir.mask + 1;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (uint64_t)gridDim.x * blockDim.x)
        reinterpret_cast<uint32_t *>(&dir.slots[i].val)[1] = 0;
}

// clean_server (local.rs:51-58): streaming scan, the GPU analogue of retain(|_, v| *v != address)
__global__ void __launch_bounds__(256)
k_dir_clean_node(DirDev dir, uint32_t node, unsigned long long *removed) {
    uint4 *slots = reinterpret_cast<uint4 *>(dir.slots);
    const uint64_t cap = dir.mask + 1;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < cap; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        bool hit = false;
        if (i < cap) {
            const uint4 v = slots[i];
            hit = v.z == node && (v.x & v.y) != 0xFFFFFFFFu;
            if (hit) reinterpret_cast<uint32_t *>(&dir.slots[i].val)[0] = kNone;
        }
        warp_add(removed, hit);
    }
}
// same, for a set of nodes flagged in a byte map (place_batch cleans every dead node it met in one pass)
__global__ void __launch_bounds__(256)
k_dir_clean_flagged(DirDev dir, const uint8_t *__restrict__ flag, uint32_t n_total, unsigned long long *removed) {
    uint4 *slots = reinterpret_cast<uint4 *>(dir.slots);
    const uint64_t cap = dir.mask + 1;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < cap; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        bool hit = false;
        if (i < cap) {
            const uint4 v = slots[i];
            hit = v.z < n_total && (v.x & v.y) != 0xFFFFFFFFu && __ldg(flag + v.z);
            if (hit) reinterpret_cast<uint32_t *>(&dir.slots[i].val)[0] = kNone;
        }
        warp_add(removed, hit);
    }
}

// grow: re-insert every placed key of `from` into the (empty) table `to`; unplaced keys are dropped
__global__ void __launch_bounds__(256)
k_dir_rehash(DirDev from, DirDev to, unsigned long long *new_keys, uint32_t *error) {
    const uint4 *src = reinterpret_cast<const uint4 *>(from.slots);
    const uint64_t cap = from.mask + 1;
    unsigned long long n_moved = 0;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < cap; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        bool moved = false;
        if (i < cap) {
            const uint4 v = src[i];
            const unsigned long long key = ((unsigned long long)v.y << 32) | v.x;
            if (key != kEmptyKey && v.z != kNone) {
                uint64_t s = home_slot(key, to);
                for (uint64_t probes = 0; probes <= to.mask; probes++) {
                    const unsigned long long k = atomicCAS(&to.slots[s].key, kEmptyKey, key);
                    if (k == kEmptyKey) { to.slots[s].val = v.z; moved = true; break; }   // keys of `from` are distinct
                    s = (s + 1) & to.mask;
                }
                if (!moved) atomicExch(error, 1u);
            }
        }
        n_moved += moved;
    }
    warp_flush(new_keys, n_moved);
}

__global__ void __launch_bounds__(256)
k_dir_count(DirDev dir, unsigned long long *placed, uint32_t *counters, uint32_t n_total) {
    const uint4 *slots = reinterpret_cast<const uint4 *>(dir.slots);
    const uint64_t cap = dir.mask + 1;
    unsigned long long n_hit = 0;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < cap; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        if (i < cap) {
            const uint4 v = slots[i];
            const bool hit = (v.x & v.y) != 0xFFFFFFFFu && v.z != kNone;
            if (hit && counters && v.z < n_total) atomicAdd(&counters[v.z], 1u);
            n_hit += hit;
        }
    }
    warp_flush(placed, n_hit);
}

// ---- rebalance ---------------------------------------------------------------------------------------
// JOIN(new): an object moves iff the new node beats its incumbent under the spec order (score, ~u, j); both
// candidates are one pair hash each (the incumbent's is recomputed from (key, idx) instead of being stored, so
// the stream is 12 B/object for a dense set, 16 B/slot for the directory).  by_idx[] gives {s0, invw, s2}.
// Returns the node the object belongs on after the join: new_idx if it beats the incumbent, the incumbent otherwise; an
// incumbent that is not live (recorded on an inactive / zero-weight / never-live address: update() may record anything) is
// re-placed by the full rendezvous over the live table, exactly what a fresh assignment would do -- not handed to the joiner.
__device__ uint32_t hrw_scalar(uint64_t key, const NodeTabDev &tab);
// Does node jn (pair hash un, factor rn) beat node jc (uc, rc) under the spec order?  Cheap bracket first: E(u) lies in
// [clz(u) << 26, (clz(u)+1) << 26], so most comparisons (the challenger wins only ~w/W of the time) are decided without
// evaluating the log polynomial at all.
__device__ __forceinline__ bool challenger_wins(uint32_t un, uint32_t rn, uint32_t jn, uint32_t uc, uint32_t rc, uint32_t jc) {
    const uint32_t ln = clz_u32(un), lc = clz_u32(uc);
    if ((uint64_t)(ln << 26) * rn > (uint64_t)((lc + 1u) << 26) * rc) return false;
    const uint64_t sn = (uint64_t)elog(un) * rn;
    const uint64_t sc = (uint64_t)elog(uc) * rc;
    return cand_better(sn, un, jn, sc, uc, jc);
}
__device__ __forceinline__ bool join_wins(uint64_t key, uint32_t cur, uint32_t new_idx, const uint4 nn, const uint4 *by_idx, bool *incumbent_dead) {
    const ObjHash o = obj_hash(key);
    const uint32_t un = pair_hash(o, nn.x, nn.z, nn.w);
    const uint4 c = by_idx[cur];   // shared memory (staged) or global
    *incumbent_dead = c.y == 0;
    if (c.y == 0) return false;
    const uint32_t uc = pair_hash(o, c.x, c.z, c.w);
    return challenger_wins(un, nn.y, new_idx, uc, c.y, cur);
}

// The incumbent's node record is a random 16-byte gather: from L1 that costs one wavefront per distinct line (up to 32 per
// warp load), so the by-index table is staged in shared memory when it fits (template SMEM; LDS.128, not generic LD).
template <bool SMEM>
__device__ __forceinline__ const uint4 *stage_by_idx(const NodeTabDev &tab) {
    extern __shared__ __align__(16) unsigned char smem_dir[];
    if (!SMEM) return tab.by_idx;
    uint4 *s = reinterpret_cast<uint4 *>(smem_dir);
    for (uint32_t j = threadIdx.x; j < tab.n_total; j += blockDim.x) s[j] = __ldg(tab.by_idx + j);
    __syncthreads();
    return s;
}

// One object of a join: returns the node it belongs on afterwards (== cur when nothing changes).
__device__ __forceinline__ uint32_t join_target(uint64_t key, uint32_t cur, uint32_t new_idx, const uint4 nn, const uint4 *by_idx, const NodeTabDev &tab) {
    if (cur == new_idx || cur >= tab.n_total || !nn.y) return cur;
    bool dead;
    if (join_wins(key, cur, new_idx, nn, by_idx, &dead)) return new_idx;
    return dead ? hrw_scalar(key, tab) : cur;   // rare: the incumbent is not live
}

// Dense set, 12 B/object stream: each thread owns 4 consecutive objects per trip -- two 128-bit key loads and one 128-bit index
// load, all issued before any of them is used, and the next trip's loads are in flight while this one computes.
constexpr int kJoinOpt = 4;
template <bool SMEM>
__global__ void __launch_bounds__(256)
k_rebalance_join(const uint64_t *__restrict__ keys, uint32_t *__restrict__ idx, uint64_t n, NodeTabDev tab, uint32_t new_idx,
                 uint32_t *__restrict__ counters, unsigned long long *moved) {
    const uint4 *by_idx = stage_by_idx<SMEM>(tab);
    const uint4 nn = __ldg(tab.by_idx + new_idx);
    const uint64_t n_quads = (n + kJoinOpt - 1) / kJoinOpt, stride = (uint64_t)gridDim.x * blockDim.x;
    unsigned long long n_moved = 0;
    ulonglong2 k0, k1;
    uint4 cur4;
    auto load = [&](uint64_t q) {
        const uint64_t f = q * kJoinOpt;
        if (f + 3 < n) {
            k0 = __ldg(reinterpret_cast<const ulonglong2 *>(keys + f));
            k1 = __ldg(reinterpret_cast<const ulonglong2 *>(keys + f + 2));
            cur4 = *reinterpret_cast<const uint4 *>(idx + f);
        } else {   // ragged tail: element by element, missing ones read as "already on the new node" (skipped)
            k0.x = f < n ? __ldg(keys + f) : 0; k0.y = f + 1 < n ? __ldg(keys + f + 1) : 0; k1.x = f + 2 < n ? __ldg(keys + f + 2) : 0; k1.y = 0;
            cur4.x = f < n ? idx[f] : new_idx; cur4.y = f + 1 < n ? idx[f + 1] : new_idx; cur4.z = f + 2 < n ? idx[f + 2] : new_idx; cur4.w = new_idx;
        }
    };
    uint64_t q = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q < n_quads) load(q);
    for (; q < n_quads; q += stride) {
        const ulonglong2 a0 = k0, a1 = k1;
        const uint4 c = cur4;
        if (q + stride < n_quads) load(q + stride);
        uint4 t;
        t.x = join_target(a0.x, c.x, new_idx, nn, by_idx, tab);
        t.y = join_target(a0.y, c.y, new_idx, nn, by_idx, tab);
        t.z = join_target(a1.x, c.z, new_idx, nn, by_idx, tab);
        t.w = join_target(a1.y, c.w, new_idx, nn, by_idx, tab);
        const uint32_t tt[4] = {t.x, t.y, t.z, t.w}, cc[4] = {c.x, c.y, c.z, c.w};
        uint32_t changed = 0;
#pragma unroll
        for (int e = 0; e < 4; e++) {
            if (tt[e] != cc[e]) {
                changed++;
                if (q * kJoinOpt + e < n) idx[q * kJoinOpt + e] = tt[e];
                if (counters) { atomicSub(&counters[cc[e]], 1u); if (tt[e] != kNone) atomicAdd(&counters[tt[e]], 1u); }
            }
        }
        n_moved += changed;
    }
    warp_flush(moved, n_moved);
}

// Directory, 16 B/slot stream: four independent 128-bit slot loads per thread per trip.
template <bool SMEM>
__global__ void __launch_bounds__(256)
k_dir_rebalance_join(DirDev dir, NodeTabDev tab, uint32_t new_idx, unsigned long long *moved) {
    const uint4 *by_idx = stage_by_idx<SMEM>(tab);
    const uint4 *slots = reinterpret_cast<const uint4 *>(dir.slots);
    const uint4 nn = __ldg(tab.by_idx + new_idx);
    const uint64_t cap = dir.mask + 1, stride = (uint64_t)gridDim.x * blockDim.x;
    unsigned long long n_moved = 0;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < cap; i0 += stride * 4) {
        uint4 v[4];
#pragma unroll
        for (int e = 0; e < 4; e++) { const uint64_t i = i0 + e * stride; v[e] = i < cap ? slots[i] : make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, kNone, 0); }
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const unsigned long long key = ((unsigned long long)v[e].y << 32) | v[e].x;
            if (key == kEmptyKey || v[e].z == kNone) continue;
            const uint32_t to = join_target(key, v[e].z, new_idx, nn, by_idx, tab);
            if (to != v[e].z) { reinterpret_cast<uint32_t *>(&dir.slots[i0 + e * stride].val)[0] = to; n_moved++; }
        }
    }
    warp_flush(moved, n_moved);
}

// LEAVE(gone): pick the objects recorded on the node (4 B/object scan) into a compact list ...
__global__ void __launch_bounds__(256)
k_select_on_node(const uint32_t *__restrict__ idx, uint64_t n, uint32_t node, uint32_t *__restrict__ sel, unsigned long long *nsel) {
    // 128-bit loads, four of them in flight per thread: one thread scans 4 x 4 objects per trip (idx is 256-byte aligned)
    const uint64_t n4 = (n + 3) / 4, stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n4; base += stride * 4) {
        uint4 x[4];
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const uint64_t v = base + e * stride + threadIdx.x;
            if (v < n4 && 4 * v + 3 < n) x[e] = __ldg(reinterpret_cast<const uint4 *>(idx) + v);
            else if (v < n4) { x[e].x = __ldg(idx + 4 * v); x[e].y = 4 * v + 1 < n ? __ldg(idx + 4 * v + 1) : ~node; x[e].z = 4 * v + 2 < n ? __ldg(idx + 4 * v + 2) : ~node; x[e].w = ~node; }
            else x[e] = make_uint4(~node, ~node, ~node, ~node);
        }
        uint32_t hits4[4];
#pragma unroll
        for (int e = 0; e < 4; e++) hits4[e] = (x[e].x == node) | ((x[e].y == node) << 1) | ((x[e].z == node) << 2) | ((x[e].w == node) << 3);   // bit q: object 4v+q is on the node
        if (__ballot_sync(0xFFFFFFFFu, (hits4[0] | hits4[1] | hits4[2] | hits4[3]) != 0) == 0) continue;   // the common trip: nobody in the warp hit
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const uint64_t v = base + e * stride + threadIdx.x;
            const uint32_t hits = hits4[e];
            const unsigned m = __ballot_sync(0xFFFFFFFFu, hits != 0);
            if (m) {                                        // rare: about 4/M of the vectors
                const unsigned lane = threadIdx.x & 31;
                const uint32_t mine = __popc(hits);
                uint32_t pre = mine;                        // inclusive warp prefix sum of the hit counts
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, pre, o); if (lane >= (unsigned)o) pre += t; }
                const uint32_t total = __shfl_sync(0xFFFFFFFFu, pre, 31);
                unsigned long long b = 0;
                if (lane == 0) b = atomicAdd(nsel, (unsigned long long)total);
                b = __shfl_sync(0xFFFFFFFFu, b, 0) + (pre - mine);
#pragma unroll
                for (int qq = 0; qq < 4; qq++) if (hits >> qq & 1) sel[b++] = (uint32_t)(4 * v + qq);
            }
        }
    }
}
// ... and, for the directory, re-place them in the same pass (warp per hit would be nicer; hits are ~cap/M so a
// thread-serial walk of the class-sorted table from global/L2 is enough here).
__device__ uint32_t hrw_scalar(uint64_t key, const NodeTabDev &tab) {
    const ObjHash o = obj_hash(key);
    const uint4 *grec = reinterpret_cast<const uint4 *>(tab.recs);
    uint64_t best_sc = ~0ull; uint32_t best_u = 0, best_i = kNone;
    for (uint32_t c = 0; c < tab.n_classes; c++) {
        const ClassRec r0 = tab.classes[c], r1 = tab.classes[c + 1];
        uint32_t cu = 0, ci = kNone;
        for (uint32_t q = r0.start; q < r1.start; q++) {
            const uint4 r = __ldg(grec + q);
            const uint32_t u = pair_hash(o, r.x, r.z, r.w);
            if (ci == kNone || u > cu) { cu = u; ci = r.y; }
        }
        const uint64_t sc = (uint64_t)elog(cu) * r0.invw;
        if (ci != kNone && (best_i == kNone || cand_better(sc, cu, ci, best_sc, best_u, best_i))) { best_sc = sc; best_u = cu; best_i = ci; }
    }
    return best_i;
}
__global__ void __launch_bounds__(256)
k_dir_rebalance_leave(DirDev dir, NodeTabDev tab, uint32_t gone, unsigned long long *moved) {
    const uint4 *slots = reinterpret_cast<const uint4 *>(dir.slots);
    const uint64_t cap = dir.mask + 1;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < cap; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        bool mv = false;
        if (i < cap) {
            const uint4 v = slots[i];
            const unsigned long long key = ((unsigned long long)v.y << 32) | v.x;
            if (key != kEmptyKey && v.z == gone) {
                reinterpret_cast<uint32_t *>(&dir.slots[i].val)[0] = hrw_scalar(key, tab);
                mv = true;
            }
        }
        warp_add(moved, mv);
    }
}

// ---- change set (DESIGN.md 3.10): R1 entries (incumbent in REPLACE) are collected and re-placed by the grid kernel;
// an R2 entry goes to the best of {incumbent} u CANDIDATES, one pair hash each, decided in place.
// Shared-memory layout when staged: [n_total x uint4 by-index records][n_cand x u32 candidates][n_total flag bytes].
template <bool SMEM>
__device__ __forceinline__ ChangeSetDev stage_changes(const ChangeSetDev &cs, uint32_t n_total) {
    extern __shared__ __align__(16) unsigned char smem_dir[];
    if (!SMEM) return cs;
    uint32_t *c = reinterpret_cast<uint32_t *>(smem_dir + (size_t)n_total * 16);
    uint8_t *f = reinterpret_cast<uint8_t *>(c + cs.n_cand);
    for (uint32_t j = threadIdx.x; j < cs.n_cand; j += blockDim.x) c[j] = __ldg(cs.cand + j);
    for (uint32_t j = threadIdx.x; j < n_total; j += blockDim.x) f[j] = __ldg(cs.flag + j);
    return ChangeSetDev{f, c, cs.n_cand};   // visible after the __syncthreads of stage_by_idx
}

__device__ __forceinline__ uint32_t change_target(uint64_t key, uint32_t cur, const uint4 *by_idx, const ChangeSetDev &cs) {
    const ObjHash o = obj_hash(key);
    const uint4 c = by_idx[cur];
    uint32_t best = cur, bu = pair_hash(o, c.x, c.z, c.w), br = c.y;
    for (uint32_t q = 0; q < cs.n_cand; q++) {
        const uint32_t j = cs.cand[q];
        const uint4 r = by_idx[j];
        const uint32_t u = pair_hash(o, r.x, r.z, r.w);
        if (challenger_wins(u, r.y, j, bu, br, best)) { best = j; bu = u; br = r.y; }
    }
    return best;
}

// Directory, 16 B/slot stream: four independent 128-bit slot loads per thread per trip.  The trip loop is warp-uniform (the
// capacity is a power of two >= 1024), so the R1 append can ballot.
template <bool SMEM>
__global__ void __launch_bounds__(256)
k_dir_rebalance_changes(DirDev dir, NodeTabDev tab, ChangeSetDev cs_in, uint64_t *__restrict__ r1_slot, uint64_t *__restrict__ r1_key,
                        unsigned long long *nr1, unsigned long long *moved) {
    const ChangeSetDev cs = stage_changes<SMEM>(cs_in, tab.n_total);
    const uint4 *by_idx = stage_by_idx<SMEM>(tab);
    const uint4 *slots = reinterpret_cast<const uint4 *>(dir.slots);
    const uint64_t cap = dir.mask + 1, stride = (uint64_t)gridDim.x * blockDim.x;
    unsigned long long n_moved = 0;
    for (uint64_t i0 = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i0 < cap; i0 += stride * 4) {
        uint4 v[4];
#pragma unroll
        for (int e = 0; e < 4; e++) { const uint64_t i = i0 + e * stride; v[e] = i < cap ? slots[i] : make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, kNone, 0); }
        uint32_t r1 = 0;   // bit e: slot e goes to the R1 list
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const unsigned long long key = ((unsigned long long)v[e].y << 32) | v[e].x;
            if (key == kEmptyKey || v[e].z >= tab.n_total) continue;
            if (cs.flag[v[e].z] & kChgReplace) { r1 |= 1u << e; continue; }
            const uint32_t to = change_target(key, v[e].z, by_idx, cs);
            if (to != v[e].z) { reinterpret_cast<uint32_t *>(&dir.slots[i0 + e * stride].val)[0] = to; n_moved++; }
        }
        if (__ballot_sync(0xFFFFFFFFu, r1 != 0) == 0) continue;
        unsigned long long b = warp_reserve(nr1, __popc(r1));
#pragma unroll
        for (int e = 0; e < 4; e++)
            if (r1 >> e & 1) { r1_slot[b] = i0 + e * stride; r1_key[b] = ((unsigned long long)v[e].y << 32) | v[e].x; b++; }
    }
    warp_flush(moved, n_moved);
}

__global__ void __launch_bounds__(256)
k_dir_scatter_changes(DirDev dir, const uint64_t *__restrict__ r1_slot, const uint32_t *__restrict__ to, uint64_t n, unsigned long long *moved) {
    unsigned long long n_moved = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t *node = reinterpret_cast<uint32_t *>(&dir.slots[__ldg(r1_slot + i)].val);
        const uint32_t t = __ldg(to + i);
        if (t != *node) { *node = t; n_moved++; }
    }
    warp_flush(moved, n_moved);
}

// The counters of REPLACE nodes: every object on such a node is selected and re-placed, and the re-placement adds its result.
__device__ __forceinline__ void zero_replace_counters(const ChangeSetDev &cs, uint32_t n_total, uint32_t *counters) {
    if (!counters) return;
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n_total; j += gridDim.x * blockDim.x)
        if (__ldg(cs.flag + j) & kChgReplace) counters[j] = 0;
}

// Dense set, 12 B/object: each thread takes 4 consecutive objects per trip (two 128-bit key loads, one 128-bit index load).
// An object that is not placed (RIO_NONE, or an index past the table) is selected too: the fresh assignment places it.
template <bool SMEM>
__global__ void __launch_bounds__(256)
k_rebalance_changes(const uint64_t *__restrict__ keys, uint32_t *__restrict__ idx, uint64_t n, NodeTabDev tab, ChangeSetDev cs_in,
                    uint32_t *__restrict__ counters, uint32_t *__restrict__ sel, uint32_t *__restrict__ sel_old, unsigned long long *nsel,
                    unsigned long long *moved) {
    zero_replace_counters(cs_in, tab.n_total, counters);
    const ChangeSetDev cs = stage_changes<SMEM>(cs_in, tab.n_total);
    const uint4 *by_idx = stage_by_idx<SMEM>(tab);
    const uint64_t n_quads = (n + kJoinOpt - 1) / kJoinOpt, stride = (uint64_t)gridDim.x * blockDim.x;
    unsigned long long n_moved = 0;
    for (uint64_t qb = (uint64_t)blockIdx.x * blockDim.x; qb < n_quads; qb += stride) {   // block-uniform trips
        const uint64_t q = qb + threadIdx.x, f = q * kJoinOpt;
        uint64_t k[4] = {0, 0, 0, 0};
        uint32_t c[4] = {kNone, kNone, kNone, kNone};
        if (q < n_quads && f + 3 < n) {
            const ulonglong2 k0 = __ldg(reinterpret_cast<const ulonglong2 *>(keys + f)), k1 = __ldg(reinterpret_cast<const ulonglong2 *>(keys + f + 2));
            const uint4 c4 = *reinterpret_cast<const uint4 *>(idx + f);
            k[0] = k0.x; k[1] = k0.y; k[2] = k1.x; k[3] = k1.y;
            c[0] = c4.x; c[1] = c4.y; c[2] = c4.z; c[3] = c4.w;
        } else if (q < n_quads) {
#pragma unroll
            for (int e = 0; e < 4; e++) if (f + e < n) { k[e] = __ldg(keys + f + e); c[e] = idx[f + e]; }
        }
        uint32_t r1 = 0;
#pragma unroll
        for (int e = 0; e < 4; e++) {
            if (q >= n_quads || f + e >= n) continue;
            if (c[e] >= tab.n_total || (cs.flag[c[e]] & kChgReplace)) { r1 |= 1u << e; continue; }
            const uint32_t to = change_target(k[e], c[e], by_idx, cs);
            if (to != c[e]) {
                idx[f + e] = to;
                n_moved++;
                if (counters) { atomicSub(&counters[c[e]], 1u); atomicAdd(&counters[to], 1u); }
            }
        }
        if (__ballot_sync(0xFFFFFFFFu, r1 != 0) == 0) continue;
        unsigned long long b = warp_reserve(nsel, __popc(r1));
#pragma unroll
        for (int e = 0; e < 4; e++)
            if (r1 >> e & 1) { sel[b] = (uint32_t)(f + e); sel_old[b] = c[e]; b++; }
    }
    warp_flush(moved, n_moved);
}

// No candidates: no entry takes the R2 branch, so only the selection is left -- a 4 B/object scan of idx, the multi-node form of
// k_select_on_node (4 x 4 objects per thread per trip).
__global__ void __launch_bounds__(256)
k_select_flagged(const uint32_t *__restrict__ idx, uint64_t n, ChangeSetDev cs, uint32_t n_total, uint32_t *__restrict__ counters,
                 uint32_t *__restrict__ sel, uint32_t *__restrict__ sel_old, unsigned long long *nsel) {
    zero_replace_counters(cs, n_total, counters);
    const uint64_t n4 = (n + 3) / 4, stride = (uint64_t)gridDim.x * blockDim.x;
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n4; base += stride * 4) {
        uint4 x[4];
        uint32_t valid[4];   // bit q: object 4v+q exists
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const uint64_t v = base + e * stride + threadIdx.x;
            valid[e] = v < n4 ? (4 * v + 3 < n ? 15u : (1u << (n - 4 * v)) - 1u) : 0u;
            if (valid[e] == 15u) x[e] = __ldg(reinterpret_cast<const uint4 *>(idx) + v);
            else if (valid[e]) { x[e].x = __ldg(idx + 4 * v); x[e].y = 4 * v + 1 < n ? __ldg(idx + 4 * v + 1) : 0; x[e].z = 4 * v + 2 < n ? __ldg(idx + 4 * v + 2) : 0; x[e].w = 0; }
        }
        uint32_t hits4[4];
#pragma unroll
        for (int e = 0; e < 4; e++) {
            hits4[e] = 0;
            if (!valid[e]) continue;
            const uint32_t xs[4] = {x[e].x, x[e].y, x[e].z, x[e].w};
#pragma unroll
            for (int qq = 0; qq < 4; qq++)
                if ((valid[e] >> qq & 1) && (xs[qq] >= n_total || (cs.flag[xs[qq]] & kChgReplace))) hits4[e] |= 1u << qq;
        }
        if (__ballot_sync(0xFFFFFFFFu, (hits4[0] | hits4[1] | hits4[2] | hits4[3]) != 0) == 0) continue;
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const uint64_t v = base + e * stride + threadIdx.x;
            if (__ballot_sync(0xFFFFFFFFu, hits4[e] != 0) == 0) continue;
            unsigned long long b = warp_reserve(nsel, __popc(hits4[e]));
            const uint32_t xs[4] = {x[e].x, x[e].y, x[e].z, x[e].w};
#pragma unroll
            for (int qq = 0; qq < 4; qq++) if (hits4[e] >> qq & 1) { sel[b] = (uint32_t)(4 * v + qq); sel_old[b] = xs[qq]; b++; }
        }
    }
}

__global__ void __launch_bounds__(256)
k_count_changed(const uint32_t *__restrict__ idx, const uint32_t *__restrict__ sel, const uint32_t *__restrict__ sel_old, uint64_t n, unsigned long long *moved) {
    unsigned long long n_moved = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        n_moved += __ldg(idx + __ldg(sel + i)) != __ldg(sel_old + i);
    warp_flush(moved, n_moved);
}

// ---- ranked resident sets (DESIGN.md 3.11) -------------------------------------------------------------------------------
// Insert node j (pair hash u, factor r) into the list (gs, gu, gj), best first under the order (E(u)*r, ~u, j) of cand_better: the
// insertion network of k_assign_hrw_ranked, so ties resolve exactly as there.
template <int R>
__device__ __forceinline__ void rank_insert(uint64_t (&gs)[R], uint32_t (&gu)[R], uint32_t (&gj)[R], uint32_t u, uint32_t r, uint32_t j) {
    uint64_t s = (uint64_t)elog(u) * r;
    if (!cand_better(s, u, j, gs[R - 1], gu[R - 1], gj[R - 1])) return;
#pragma unroll
    for (int y = 0; y < R; y++) {
        const bool sw = cand_better(s, u, j, gs[y], gu[y], gj[y]);
        const uint64_t ts = gs[y]; const uint32_t tu = gu[y], tj = gj[y];
        gs[y] = sw ? s : ts; gu[y] = sw ? u : tu; gj[y] = sw ? j : tj;
        s = sw ? ts : s; u = sw ? tu : u; j = sw ? tj : j;
    }
}

// The same for a failure-domain list (DESIGN.md 3.13): node j of dense domain d, inserted with the domain-aware rule of 3.12.
template <int R>
__device__ __forceinline__ void spread_rank_insert(uint64_t (&gs)[R], uint32_t (&gu)[R], uint32_t (&gj)[R], uint32_t (&gd)[R], uint32_t u, uint32_t r,
                                                   uint32_t j, uint32_t d) {
    const uint64_t s = (uint64_t)elog(u) * r;
    if (!cand_better(s, u, j, gs[R - 1], gu[R - 1], gj[R - 1])) return;
    spread_insert<R>(gs, gu, gj, gd, s, u, j, d);
}

// Flat policy, 8 + 4R B/object: S1 objects (a list member in REPLACE or past the table) are appended to sel; an S2 list becomes the
// first R of L u CANDIDATES.  When no member of L is a candidate and L is full, its order is unchanged and a candidate enters only by
// beating L's last member: one pair hash per candidate, behind challenger_wins's clz bracket.  Only then, or when a member gained
// weight or L is short, is every member and candidate scored and merged.  The trip loop is block-uniform, so the S1 append can ballot.
// SPREAD (DESIGN.md 3.13): the lists are failure-domain lists and the merge keeps the first R domain representatives, with one dense
// domain id per scored node read from ndom (n_total x u32) through the read-only path; the gate above is exact for them as well.  The
// extra argument comes last, so the plain instantiations keep their code.
template <int R, bool SMEM, bool SPREAD>
__global__ void __launch_bounds__(256)
k_rebalance_changes_ranked(const uint64_t *__restrict__ keys, uint32_t *__restrict__ lists, uint32_t *__restrict__ idx, uint64_t n, NodeTabDev tab,
                           ChangeSetDev cs_in, uint32_t *__restrict__ counters, uint32_t *__restrict__ sel, unsigned long long *nsel,
                           unsigned long long *moved, unsigned long long *changed, const uint32_t *__restrict__ ndom) {
    const ChangeSetDev cs = stage_changes<SMEM>(cs_in, tab.n_total);
    const uint4 *by_idx = stage_by_idx<SMEM>(tab);
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    unsigned long long n_moved = 0, n_changed = 0;
    for (uint64_t b = (uint64_t)blockIdx.x * blockDim.x; b < n; b += stride) {
        const uint64_t i = b + threadIdx.x;
        bool s1 = false;
        if (i < n) {
            uint32_t l[R];
#pragma unroll
            for (int x = 0; x < R; x++) l[x] = lists[i * R + x];
            const uint64_t key = cs.n_cand ? __ldg(keys + i) : 0;   // no candidate: an S2 list cannot change, the key is not needed
            bool member_cand = false, full = true;
#pragma unroll
            for (int x = 0; x < R; x++) {
                if (l[x] == kNone) { full = false; continue; }
                if (l[x] >= tab.n_total) { s1 = true; continue; }
                const uint8_t f = cs.flag[l[x]];
                s1 |= (f & kChgReplace) != 0;
                member_cand |= (f & kChgCandidate) != 0;
            }
            if (!s1 && cs.n_cand) {
                const ObjHash o = obj_hash(key);
                bool merge = member_cand || !full;
                if (!merge) {
                    const uint4 c = by_idx[l[R - 1]];
                    const uint32_t ul = pair_hash(o, c.x, c.z, c.w);
                    for (uint32_t q = 0; q < cs.n_cand && !merge; q++) {
                        const uint32_t j = cs.cand[q];
                        const uint4 r = by_idx[j];
                        merge = challenger_wins(pair_hash(o, r.x, r.z, r.w), r.y, j, ul, c.y, l[R - 1]);
                    }
                }
                if (merge) {
                    uint64_t gs[R];
                    uint32_t gu[R], gj[R], gd[R];
#pragma unroll
                    for (int x = 0; x < R; x++) { gs[x] = ~0ull; gu[x] = 0; gj[x] = kNone; gd[x] = kNone; }
#pragma unroll
                    for (int x = 0; x < R; x++) {
                        if (l[x] == kNone) continue;
                        const uint4 r = by_idx[l[x]];
                        if (SPREAD) spread_rank_insert<R>(gs, gu, gj, gd, pair_hash(o, r.x, r.z, r.w), r.y, l[x], __ldg(ndom + l[x]));
                        else rank_insert<R>(gs, gu, gj, pair_hash(o, r.x, r.z, r.w), r.y, l[x]);
                    }
                    for (uint32_t q = 0; q < cs.n_cand; q++) {
                        const uint32_t j = cs.cand[q];
                        bool in_l = false;
#pragma unroll
                        for (int x = 0; x < R; x++) in_l |= l[x] == j;
                        if (in_l) continue;   // a member that gained weight counts once
                        const uint4 r = by_idx[j];
                        if (SPREAD) spread_rank_insert<R>(gs, gu, gj, gd, pair_hash(o, r.x, r.z, r.w), r.y, j, __ldg(ndom + j));
                        else rank_insert<R>(gs, gu, gj, pair_hash(o, r.x, r.z, r.w), r.y, j);
                    }
                    bool ch = false;
#pragma unroll
                    for (int x = 0; x < R; x++) ch |= gj[x] != l[x];
                    if (ch) {
#pragma unroll
                        for (int x = 0; x < R; x++) lists[i * R + x] = gj[x];
                        n_changed++;
                        if (gj[0] != l[0]) {
                            idx[i] = gj[0];
                            n_moved++;
                            if (counters) { if (l[0] != kNone) atomicSub(&counters[l[0]], 1u); atomicAdd(&counters[gj[0]], 1u); }
                        }
                    }
                }
            }
        }
        if (__ballot_sync(0xFFFFFFFFu, s1) == 0) continue;
        const unsigned long long p = warp_reserve(nsel, s1 ? 1u : 0u);
        if (s1) sel[p] = (uint32_t)i;
    }
    warp_flush(moved, n_moved);
    warp_flush(changed, n_changed);
}

// S1 objects after the flat ranked kernel re-ranked their gathered keys into fresh (n_sel x R): write back the rows that changed.
// The stored row still holds the old list, so its column 0 is the old rank 1.
__global__ void __launch_bounds__(256)
k_scatter_ranked(const uint32_t *__restrict__ fresh, const uint32_t *__restrict__ sel, uint64_t n_sel, uint32_t ranks, uint32_t *__restrict__ lists,
                 uint32_t *__restrict__ idx, uint32_t *__restrict__ counters, uint32_t n_total, unsigned long long *moved, unsigned long long *changed) {
    unsigned long long n_moved = 0, n_changed = 0;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_sel; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t o = __ldg(sel + i);
        uint32_t *row = lists + o * ranks;
        const uint32_t *f = fresh + i * ranks;
        const uint32_t old0 = row[0], new0 = __ldg(f);
        bool ch = false;
        for (uint32_t x = 0; x < ranks; x++) {
            const uint32_t v = __ldg(f + x);
            if (row[x] != v) { row[x] = v; ch = true; }
        }
        n_changed += ch;
        if (old0 != new0) {
            idx[o] = new0;
            n_moved++;
            if (counters) {
                if (old0 < n_total) atomicSub(&counters[old0], 1u);
                if (new0 < n_total) atomicAdd(&counters[new0], 1u);
            }
        }
    }
    warp_flush(moved, n_moved);
    warp_flush(changed, n_changed);
}

__global__ void __launch_bounds__(256)
k_ranked_primary(const uint32_t *__restrict__ lists, uint64_t n, uint32_t ranks, uint32_t *__restrict__ idx) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) idx[i] = __ldg(lists + i * ranks);
}

// bounded-load rounds: spill selection (DESIGN.md 3.5)
__global__ void __launch_bounds__(256)
k_select_spill(const uint64_t *__restrict__ keys, const uint32_t *__restrict__ idx, uint64_t n, const uint32_t *__restrict__ thr,
               const uint8_t *__restrict__ over, uint32_t round, uint32_t *__restrict__ sel, unsigned long long *nsel, uint32_t *__restrict__ counters) {
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        bool hit = false;
        if (i < n) {
            const uint32_t j = __ldg(idx + i);
            if (j != kNone && __ldg(over + j)) {
                hit = spill_hash(__ldg(keys + i), round) < __ldg(thr + j);
                if (hit && counters) atomicSub(&counters[j], 1u);
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

// place_batch: which looked-up placements must be (re)placed (service.rs:203-238)
__global__ void __launch_bounds__(256)
k_classify(const uint32_t *__restrict__ cur, uint64_t n, const uint8_t *__restrict__ node_state, uint32_t n_total, uint32_t *__restrict__ sel,
           unsigned long long *nsel, uint8_t *__restrict__ dead_flag) {
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        bool need = false;
        if (i < n) {
            const uint32_t c = __ldg(cur + i);
            if (c == kNone || c >= n_total) need = true;                                  // service.rs:241-252
            else {
                const uint8_t st = __ldg(node_state + c);
                if (!(st & kNodeLive)) { need = true; if (!(st & kNodeMalformed)) dead_flag[c] = 1; }   // :226-238 / :213-222
            }
        }
        const unsigned m = __ballot_sync(0xFFFFFFFFu, need);
        if (m) {
            const unsigned lane = threadIdx.x & 31, leader = __ffs(m) - 1;
            unsigned long long b = 0;
            if (lane == leader) b = atomicAdd(nsel, (unsigned long long)__popc(m));
            b = __shfl_sync(0xFFFFFFFFu, b, leader);
            if (need) sel[b + __popc(m & ((1u << lane) - 1))] = (uint32_t)i;
        }
    }
}

// Service::check_address_mismatch, batched (service.rs:261-298): the verdict per interned address comes in a byte table
__global__ void __launch_bounds__(256)
k_check_address(const uint32_t *__restrict__ idx, uint64_t n, const uint8_t *__restrict__ verdict_tab, uint32_t n_total, uint8_t *__restrict__ out,
                uint8_t *__restrict__ dead_flag, unsigned long long *ndead) {
    for (uint64_t base = (uint64_t)blockIdx.x * blockDim.x; base < n; base += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t i = base + threadIdx.x;
        bool dead = false;
        if (i < n) {
            const uint32_t j = __ldg(idx + i);
            const uint8_t v = j < n_total ? __ldg(verdict_tab + j) : (uint8_t)3;
            out[i] = v;
            dead = v == 2;
            if (dead) dead_flag[j] = 1;
        }
        warp_add(ndead, dead);
    }
}

__global__ void k_scatter_const(uint32_t *__restrict__ out, const uint32_t *__restrict__ sel, uint64_t n_sel, uint32_t v) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_sel; i += (uint64_t)gridDim.x * blockDim.x) out[sel[i]] = v;
}
__global__ void k_gather_keys(const uint64_t *__restrict__ keys, const uint32_t *__restrict__ sel, uint64_t n_sel, uint64_t *__restrict__ out_keys,
                              const uint32_t *__restrict__ idx, uint32_t *__restrict__ out_idx) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_sel; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t s = sel[i];
        out_keys[i] = keys[s];
        if (idx) out_idx[i] = idx[s];
    }
}

// ---- the counter exchange as ONE kernel over NVLink peer memory (DESIGN.md 6) -------------------------------------
// Every rank owns a window {slots[2][world][max_nodes] u32, flags[world] u32} that all peers have mapped through CUDA
// IPC.  push: my M counters go into slot [epoch&1][rank] of every peer's window (plain P2P stores over NVLink);
// signal: a release store of the epoch into flags[rank] of every peer; wait: spin (acquire loads, system scope) until my
// own window carries this epoch from every rank; sum.  Slots are double buffered by epoch parity: nobody can be two
// exchanges ahead, because every exchange needs everybody's flag.
__global__ void __launch_bounds__(1024)
k_exchange_p2p(const uint32_t *__restrict__ local, XchgPeers peers, uint32_t rank, uint32_t world, uint32_t M, uint32_t max_nodes, uint32_t epoch,
               uint32_t *__restrict__ out_global) {
    const size_t slot_words = (size_t)2 * world * max_nodes;
    const size_t par = (size_t)(epoch & 1u) * world * max_nodes;
    for (uint32_t p = 0; p < world; p++) {
        uint32_t *dst = peers.win[p] + par + (size_t)rank * max_nodes;
        for (uint32_t j = threadIdx.x; j < M; j += blockDim.x) dst[j] = local[j];
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < world) {
        uint32_t *flag = peers.win[threadIdx.x] + slot_words + rank;
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(epoch) : "memory");
    }
    if (threadIdx.x < world) {
        const uint32_t *mine = peers.win[rank] + slot_words + threadIdx.x;
        uint32_t v;
        do { asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(mine) : "memory"); } while ((int32_t)(v - epoch) < 0);
    }
    __syncthreads();
    const uint32_t *src = peers.win[rank] + par;
    for (uint32_t j = threadIdx.x; j < M; j += blockDim.x) {
        uint32_t s = 0;
        for (uint32_t r = 0; r < world; r++) s += src[(size_t)r * max_nodes + j];
        out_global[j] = s;
    }
}

// The counter exchange AND the bounded-load capacity check of a pass as one single-CTA kernel (bounded_tail.cuh)
// 256 threads: 8 warps fit beside the 5 x 8 warps of a resident walk kernel on any SM, so a pipelined check (auxiliary stream) never
// has to wait for the next set's persistent CTAs to drain
__global__ void __launch_bounds__(256)
k_exchange_check(const uint32_t *__restrict__ local, BoundedTail b) { exchange_and_check_block(b, local); }

}  // namespace

void launch_exchange_check(const Launch &L, const uint32_t *d_local, const BoundedTail &b) {
    k_exchange_check<<<1, 256, 0, L.stream>>>(d_local, b);
    RIO_COUNT_LAUNCH(L);
}

void launch_exchange_p2p(const Launch &L, const uint32_t *d_local, uint32_t *const *peer_windows, uint32_t rank, uint32_t world, uint32_t M, uint32_t max_nodes,
                         uint32_t epoch, uint32_t *d_out_global) {
    XchgPeers P{};
    for (uint32_t p = 0; p < world && p < 16; p++) P.win[p] = peer_windows[p];
    k_exchange_p2p<<<1, 1024, 0, L.stream>>>(d_local, P, rank, world, M, max_nodes, epoch, d_out_global);
    RIO_COUNT_LAUNCH(L);
}

void launch_dir_init(const Launch &L, DirSlot *slots, uint64_t cap) {
    k_dir_init<<<grid_for(cap, 256, L.sm_count, 8), 256, 0, L.stream>>>(slots, cap);
    RIO_COUNT_LAUNCH(L);
}
void launch_dir_lookup(const Launch &L, const DirDev &dir, const uint64_t *d_keys, uint64_t n, uint32_t *d_out) {
    if (!n) return;
    k_dir_lookup<<<grid_for((n + kLookupIlp - 1) / kLookupIlp, 256, L.sm_count, 8), 256, 0, L.stream>>>(dir, d_keys, n, d_out);
    RIO_COUNT_LAUNCH(L);
}
void launch_commit_diff(const Launch &L, const DirDev &dir, const uint64_t *d_keys, const uint32_t *d_idx, uint64_t n, uint8_t *d_flag, uint32_t *d_from,
                        uint32_t *d_block_cnt, uint32_t *d_block_off, unsigned long long *d_total) {
    if (!n) return;
    const uint64_t nb = (n + kCommitRows - 1) / kCommitRows;
    k_commit_diff<<<(unsigned)nb, 256, 0, L.stream>>>(dir, d_keys, d_idx, n, d_flag, d_from, d_block_cnt);
    RIO_COUNT_LAUNCH(L);
    k_commit_scan<<<1, 1024, 0, L.stream>>>(d_block_cnt, nb, d_block_off, d_total);
    RIO_COUNT_LAUNCH(L);
}
void launch_commit_list(const Launch &L, const uint64_t *d_keys, const uint32_t *d_idx, uint64_t n, const uint8_t *d_flag, const uint32_t *d_from,
                        const uint32_t *d_block_cnt, const uint32_t *d_block_off, uint64_t *d_rows, uint64_t *d_mkeys, uint32_t *d_mfrom, uint32_t *d_mto) {
    if (!n) return;
    k_commit_list<<<(unsigned)((n + kCommitRows - 1) / kCommitRows), 256, 0, L.stream>>>(d_keys, d_idx, n, d_flag, d_from, d_block_cnt, d_block_off, d_rows,
                                                                                       d_mkeys, d_mfrom, d_mto);
    RIO_COUNT_LAUNCH(L);
}
void launch_dir_upsert(const Launch &L, const DirDev &dir, const uint64_t *d_keys, const uint32_t *d_idx, uint32_t const_idx, uint64_t n, uint32_t seq_base,
                       unsigned long long *d_new_keys, uint32_t *d_error) {
    if (!n) return;
    k_dir_upsert<<<grid_for(n, 256, L.sm_count, 8), 256, 0, L.stream>>>(dir, d_keys, d_idx, const_idx, n, seq_base, d_new_keys, d_error);
    RIO_COUNT_LAUNCH(L);
}
void launch_dir_clear_seq(const Launch &L, const DirDev &dir) {
    k_dir_clear_seq<<<grid_for(dir.mask + 1, 256, L.sm_count, 8), 256, 0, L.stream>>>(dir);
    RIO_COUNT_LAUNCH(L);
}
void launch_dir_clean_node(const Launch &L, const DirDev &dir, uint32_t node, unsigned long long *d_removed) {
    k_dir_clean_node<<<grid_for(dir.mask + 1, 256, L.sm_count, 8), 256, 0, L.stream>>>(dir, node, d_removed);
    RIO_COUNT_LAUNCH(L);
}
void launch_dir_clean_flagged(const Launch &L, const DirDev &dir, const uint8_t *d_flag, uint32_t n_total, unsigned long long *d_removed) {
    k_dir_clean_flagged<<<grid_for(dir.mask + 1, 256, L.sm_count, 8), 256, 0, L.stream>>>(dir, d_flag, n_total, d_removed);
    RIO_COUNT_LAUNCH(L);
}
void launch_dir_rehash(const Launch &L, const DirDev &from, const DirDev &to, unsigned long long *d_new_keys, uint32_t *d_error) {
    k_dir_rehash<<<grid_for(from.mask + 1, 256, L.sm_count, 8), 256, 0, L.stream>>>(from, to, d_new_keys, d_error);
    RIO_COUNT_LAUNCH(L);
}
void launch_dir_count(const Launch &L, const DirDev &dir, unsigned long long *d_placed, uint32_t *d_counters, uint32_t n_total) {
    k_dir_count<<<grid_for(dir.mask + 1, 256, L.sm_count, 8), 256, 0, L.stream>>>(dir, d_placed, d_counters, n_total);
    RIO_COUNT_LAUNCH(L);
}
void launch_dir_rebalance_join(const Launch &L, const DirDev &dir, const NodeTabDev &tab, uint32_t new_idx, unsigned long long *d_moved) {
    const uint32_t sn = tab.n_total <= 6144 ? tab.n_total : 0;   // 96 KB of node records at most
    const int grid = grid_for((dir.mask + 1 + 3) / 4, 256, L.sm_count, sn > 2048 ? 2 : 8);
    if (sn) {
        cudaFuncSetAttribute(k_dir_rebalance_join<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 6144 * 16);
        k_dir_rebalance_join<true><<<grid, 256, (size_t)sn * 16, L.stream>>>(dir, tab, new_idx, d_moved);
    } else {
        k_dir_rebalance_join<false><<<grid, 256, 0, L.stream>>>(dir, tab, new_idx, d_moved);
    }
    RIO_COUNT_LAUNCH(L);
}
void launch_dir_rebalance_leave(const Launch &L, const DirDev &dir, const NodeTabDev &tab, uint32_t gone_idx, unsigned long long *d_moved) {
    k_dir_rebalance_leave<<<grid_for(dir.mask + 1, 256, L.sm_count, 8), 256, 0, L.stream>>>(dir, tab, gone_idx, d_moved);
    RIO_COUNT_LAUNCH(L);
}
void launch_rebalance_join(const Launch &L, const uint64_t *d_keys, uint32_t *d_idx, uint64_t n, const NodeTabDev &tab, uint32_t new_idx,
                           uint32_t *d_counters, unsigned long long *d_moved) {
    if (!n) return;
    const uint32_t sn = tab.n_total <= 6144 ? tab.n_total : 0;
    const int grid = grid_for((n + kJoinOpt - 1) / kJoinOpt, 256, L.sm_count, sn > 2048 ? 2 : 8);
    if (sn) {
        cudaFuncSetAttribute(k_rebalance_join<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 6144 * 16);
        k_rebalance_join<true><<<grid, 256, (size_t)sn * 16, L.stream>>>(d_keys, d_idx, n, tab, new_idx, d_counters, d_moved);
    } else {
        k_rebalance_join<false><<<grid, 256, 0, L.stream>>>(d_keys, d_idx, n, tab, new_idx, d_counters, d_moved);
    }
    RIO_COUNT_LAUNCH(L);
}
// The change-set passes stage the by-index records, the candidate list and the flag table when the node table fits as JOIN's
// does (<= 6144 interned nodes: at most 96 + 24 + 6 KB); otherwise every read goes to global memory.
static size_t changes_smem(const NodeTabDev &tab, const ChangeSetDev &cs) {
    return tab.n_total <= 6144 ? (size_t)tab.n_total * 17 + (size_t)cs.n_cand * 4 : 0;
}
static int changes_ctas_per_sm(size_t smem) { return smem ? (int)std::max<size_t>(1, std::min<size_t>(8, (200u << 10) / smem)) : 8; }
constexpr int kChangesMaxSmem = 6144 * 21;

void launch_dir_rebalance_changes(const Launch &L, const DirDev &dir, const NodeTabDev &tab, const ChangeSetDev &cs, uint64_t *d_r1_slot, uint64_t *d_r1_key,
                                  unsigned long long *d_nr1, unsigned long long *d_moved) {
    const size_t smem = changes_smem(tab, cs);
    const int grid = grid_for((dir.mask + 1 + 3) / 4, 256, L.sm_count, changes_ctas_per_sm(smem));
    if (smem) {
        cudaFuncSetAttribute(k_dir_rebalance_changes<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kChangesMaxSmem);
        k_dir_rebalance_changes<true><<<grid, 256, smem, L.stream>>>(dir, tab, cs, d_r1_slot, d_r1_key, d_nr1, d_moved);
    } else {
        k_dir_rebalance_changes<false><<<grid, 256, 0, L.stream>>>(dir, tab, cs, d_r1_slot, d_r1_key, d_nr1, d_moved);
    }
    RIO_COUNT_LAUNCH(L);
}
void launch_dir_scatter_changes(const Launch &L, const DirDev &dir, const uint64_t *d_r1_slot, const uint32_t *d_to, uint64_t n, unsigned long long *d_moved) {
    if (!n) return;
    k_dir_scatter_changes<<<grid_for(n, 256, L.sm_count, 8), 256, 0, L.stream>>>(dir, d_r1_slot, d_to, n, d_moved);
    RIO_COUNT_LAUNCH(L);
}
void launch_rebalance_changes(const Launch &L, const uint64_t *d_keys, uint32_t *d_idx, uint64_t n, const NodeTabDev &tab, const ChangeSetDev &cs,
                              uint32_t *d_counters, uint32_t *d_sel, uint32_t *d_sel_old, unsigned long long *d_nsel, unsigned long long *d_moved) {
    if (!n) return;
    if (!cs.n_cand) {
        k_select_flagged<<<grid_for((n + 15) / 16, 256, L.sm_count, 8), 256, 0, L.stream>>>(d_idx, n, cs, tab.n_total, d_counters, d_sel, d_sel_old, d_nsel);
        RIO_COUNT_LAUNCH(L);
        return;
    }
    const size_t smem = changes_smem(tab, cs);
    const int grid = grid_for((n + kJoinOpt - 1) / kJoinOpt, 256, L.sm_count, changes_ctas_per_sm(smem));
    if (smem) {
        cudaFuncSetAttribute(k_rebalance_changes<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kChangesMaxSmem);
        k_rebalance_changes<true><<<grid, 256, smem, L.stream>>>(d_keys, d_idx, n, tab, cs, d_counters, d_sel, d_sel_old, d_nsel, d_moved);
    } else {
        k_rebalance_changes<false><<<grid, 256, 0, L.stream>>>(d_keys, d_idx, n, tab, cs, d_counters, d_sel, d_sel_old, d_nsel, d_moved);
    }
    RIO_COUNT_LAUNCH(L);
}
void launch_count_changed(const Launch &L, const uint32_t *d_idx, const uint32_t *d_sel, const uint32_t *d_sel_old, uint64_t n_sel, unsigned long long *d_moved) {
    if (!n_sel) return;
    k_count_changed<<<grid_for(n_sel, 256, L.sm_count, 8), 256, 0, L.stream>>>(d_idx, d_sel, d_sel_old, n_sel, d_moved);
    RIO_COUNT_LAUNCH(L);
}
// The spread form stages what the ranked one does and reads the 4 B/node domain ids through the read-only path: they are touched
// only on the merge path, once per scored node, so the 6144-node staging threshold and its shared-memory size stay as they are.
template <int R, bool SPREAD = false>
static void rebalance_changes_ranked(const Launch &L, const uint64_t *d_keys, uint32_t *d_lists, uint32_t *d_idx, uint64_t n, const NodeTabDev &tab,
                                     const ChangeSetDev &cs, uint32_t *d_counters, uint32_t *d_sel, unsigned long long *d_nsel, unsigned long long *d_moved,
                                     unsigned long long *d_changed, const uint32_t *d_ndom = nullptr) {
    const size_t smem = changes_smem(tab, cs);
    const int grid = grid_for(n, 256, L.sm_count, changes_ctas_per_sm(smem));
    if (smem) {
        cudaFuncSetAttribute(k_rebalance_changes_ranked<R, true, SPREAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, kChangesMaxSmem);
        k_rebalance_changes_ranked<R, true, SPREAD><<<grid, 256, smem, L.stream>>>(d_keys, d_lists, d_idx, n, tab, cs, d_counters, d_sel, d_nsel, d_moved, d_changed,
                                                                                  d_ndom);
    } else {
        k_rebalance_changes_ranked<R, false, SPREAD><<<grid, 256, 0, L.stream>>>(d_keys, d_lists, d_idx, n, tab, cs, d_counters, d_sel, d_nsel, d_moved, d_changed,
                                                                                d_ndom);
    }
}
void launch_rebalance_changes_spread(const Launch &L, const uint64_t *d_keys, uint32_t *d_lists, uint32_t ranks, uint32_t *d_idx, uint64_t n, const NodeTabDev &tab,
                                     const ChangeSetDev &cs, const SpreadTabDev &sp, uint32_t *d_counters, uint32_t *d_sel, unsigned long long *d_nsel,
                                     unsigned long long *d_moved, unsigned long long *d_changed) {
    if (!n) return;
    const uint32_t *d_ndom = reinterpret_cast<const uint32_t *>(sp.base + sp.o_ndom);
    if (with_ranks(ranks, [&](auto r) {
            rebalance_changes_ranked<r, true>(L, d_keys, d_lists, d_idx, n, tab, cs, d_counters, d_sel, d_nsel, d_moved, d_changed, d_ndom);
        }))
        RIO_COUNT_LAUNCH(L);
}
void launch_rebalance_changes_ranked(const Launch &L, const uint64_t *d_keys, uint32_t *d_lists, uint32_t ranks, uint32_t *d_idx, uint64_t n, const NodeTabDev &tab,
                                     const ChangeSetDev &cs, uint32_t *d_counters, uint32_t *d_sel, unsigned long long *d_nsel, unsigned long long *d_moved,
                                     unsigned long long *d_changed) {
    if (!n) return;
    if (with_ranks(ranks, [&](auto r) { rebalance_changes_ranked<r>(L, d_keys, d_lists, d_idx, n, tab, cs, d_counters, d_sel, d_nsel, d_moved, d_changed); }))
        RIO_COUNT_LAUNCH(L);
}
void launch_scatter_ranked(const Launch &L, const uint32_t *d_fresh, const uint32_t *d_sel, uint64_t n_sel, uint32_t ranks, uint32_t *d_lists, uint32_t *d_idx,
                           uint32_t *d_counters, uint32_t n_total, unsigned long long *d_moved, unsigned long long *d_changed) {
    if (!n_sel) return;
    k_scatter_ranked<<<grid_for(n_sel, 256, L.sm_count, 8), 256, 0, L.stream>>>(d_fresh, d_sel, n_sel, ranks, d_lists, d_idx, d_counters, n_total, d_moved, d_changed);
    RIO_COUNT_LAUNCH(L);
}
void launch_ranked_primary(const Launch &L, const uint32_t *d_lists, uint64_t n, uint32_t ranks, uint32_t *d_idx) {
    if (!n) return;
    k_ranked_primary<<<grid_for(n, 256, L.sm_count, 8), 256, 0, L.stream>>>(d_lists, n, ranks, d_idx);
    RIO_COUNT_LAUNCH(L);
}
void launch_select_on_node(const Launch &L, const uint32_t *d_idx, uint64_t n, uint32_t node, uint32_t *d_sel, unsigned long long *d_nsel) {
    if (!n) return;
    k_select_on_node<<<grid_for((n + 15) / 16, 256, L.sm_count, 8), 256, 0, L.stream>>>(d_idx, n, node, d_sel, d_nsel);
    RIO_COUNT_LAUNCH(L);
}
void launch_select_spill(const Launch &L, const uint64_t *d_keys, const uint32_t *d_idx, uint64_t n, const uint32_t *d_thr, const uint8_t *d_over,
                         uint32_t round, uint32_t *d_sel, unsigned long long *d_nsel, uint32_t *d_counters) {
    if (!n) return;
    k_select_spill<<<grid_for(n, 256, L.sm_count, 8), 256, 0, L.stream>>>(d_keys, d_idx, n, d_thr, d_over, round, d_sel, d_nsel, d_counters);
    RIO_COUNT_LAUNCH(L);
}
void launch_classify(const Launch &L, const uint32_t *d_cur, uint64_t n, const uint8_t *d_node_state, uint32_t n_total, uint32_t *d_sel,
                     unsigned long long *d_nsel, uint8_t *d_dead_flag) {
    if (!n) return;
    k_classify<<<grid_for(n, 256, L.sm_count, 8), 256, 0, L.stream>>>(d_cur, n, d_node_state, n_total, d_sel, d_nsel, d_dead_flag);
    RIO_COUNT_LAUNCH(L);
}
void launch_check_address(const Launch &L, const uint32_t *d_idx, uint64_t n, const uint8_t *d_verdict_tab, uint32_t n_total, uint8_t *d_out, uint8_t *d_dead_flag,
                          unsigned long long *d_ndead) {
    if (!n) return;
    k_check_address<<<grid_for(n, 256, L.sm_count, 8), 256, 0, L.stream>>>(d_idx, n, d_verdict_tab, n_total, d_out, d_dead_flag, d_ndead);
    RIO_COUNT_LAUNCH(L);
}
void launch_scatter_const(const Launch &L, uint32_t *d_out, const uint32_t *d_sel, uint64_t n_sel, uint32_t v) {
    if (!n_sel) return;
    k_scatter_const<<<grid_for(n_sel, 256, L.sm_count, 8), 256, 0, L.stream>>>(d_out, d_sel, n_sel, v);
    RIO_COUNT_LAUNCH(L);
}
void launch_gather_keys(const Launch &L, const uint64_t *d_keys, const uint32_t *d_sel, uint64_t n_sel, uint64_t *d_out_keys, const uint32_t *d_idx,
                        uint32_t *d_out_idx) {
    if (!n_sel) return;
    k_gather_keys<<<grid_for(n_sel, 256, L.sm_count, 8), 256, 0, L.stream>>>(d_keys, d_sel, n_sel, d_out_keys, d_idx, d_out_idx);
    RIO_COUNT_LAUNCH(L);
}

}  // namespace rio

// k_assign.cu -- the solver hot path: N_obj x M_node score grid + per-row argmin, never materialised.
//
// Weighted rendezvous (DESIGN.md 3.4 / 5.1): one thread owns OPT objects, the block walks the class-sorted
// node table staged in shared memory (one broadcast LDS.128 per node per warp), and per (object,node) pair
// the integer work is  p = s0*b + ab (IMAD);  u = p*m + s2 (IMAD);  max (VIMNMX3 / 2)   [spec v3].
// The -log2 and the 64-bit weighted score are evaluated once per (object, weight class), not per pair.
// The kernel is integer-ALU bound (12 B of HBM traffic per object against M pair hashes), see DESIGN.md 5.1.
#include "kernels.cuh"
#include "k_affinity_ranked.cuh"
#include "k_affinity_spread.cuh"
#include "spec.cuh"
#include <cstdlib>

namespace rio {

namespace {

constexpr int kAssignThreads = 256;
constexpr int kOPT = 4;

template <int OPT>
__global__ void __launch_bounds__(kAssignThreads, 2)
k_assign_hrw(const uint64_t *__restrict__ keys, uint64_t n_work, NodeTabDev tab, uint32_t *__restrict__ out_idx,
             uint32_t *__restrict__ counters, const uint32_t *__restrict__ sel, uint32_t chunk_cap, uint32_t hist_bins) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint4 *srec = reinterpret_cast<uint4 *>(smem_raw);
    uint32_t *shist = reinterpret_cast<uint32_t *>(smem_raw + (size_t)chunk_cap * sizeof(uint4));
    const uint32_t n_live = tab.n_live;
    const bool single_chunk = n_live <= chunk_cap;
    const uint4 *grec = reinterpret_cast<const uint4 *>(tab.recs);

    for (uint32_t j = threadIdx.x; j < hist_bins; j += blockDim.x) shist[j] = 0;
    if (single_chunk)
        for (uint32_t j = threadIdx.x; j < n_live; j += blockDim.x) srec[j] = __ldg(grec + j);
    __syncthreads();

    const uint64_t tile_objs = (uint64_t)kAssignThreads * OPT;
    const uint64_t n_tiles = (n_work + tile_objs - 1) / tile_objs;
    for (uint64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        uint64_t oi[OPT];
        uint32_t b[OPT], ab[OPT];
        uint64_t best_sc[OPT];
        uint32_t best_u[OPT], best_i[OPT];
        bool valid[OPT];
#pragma unroll
        for (int k = 0; k < OPT; k++) {
            uint64_t t = tile * tile_objs + (uint64_t)k * kAssignThreads + threadIdx.x;
            valid[k] = t < n_work;
            oi[k] = valid[k] ? (sel ? (uint64_t)__ldg(sel + t) : t) : 0;
            uint64_t key = valid[k] ? __ldg(keys + oi[k]) : 0;
            ObjHash o = obj_hash(key);
            b[k] = o.b; ab[k] = o.ab;
            best_sc[k] = ~0ull; best_u[k] = 0; best_i[k] = kNone;
        }
        uint32_t c = 0;                       // current weight class
        uint32_t c_start = 0, c_end = 0, c_invw = 0;
        if (n_live) { ClassRec r0 = tab.classes[0], r1 = tab.classes[1]; c_start = r0.start; c_invw = r0.invw; c_end = r1.start; }
        uint32_t cu[OPT], cj[OPT];
#pragma unroll
        for (int k = 0; k < OPT; k++) { cu[k] = 0; cj[k] = 0; }

        for (uint32_t chunk_lo = 0; chunk_lo < n_live; chunk_lo += chunk_cap) {
            const uint32_t chunk_hi = min(n_live, chunk_lo + chunk_cap);
            if (!single_chunk) {
                __syncthreads();
                for (uint32_t j = chunk_lo + threadIdx.x; j < chunk_hi; j += blockDim.x) srec[j - chunk_lo] = __ldg(grec + j);
                __syncthreads();
            }
            uint32_t q = chunk_lo;
            while (q < chunk_hi) {
                const uint32_t seg_hi = min(c_end, chunk_hi);
                if (q == c_start) {            // first node of the class seeds the running max
                    const uint4 r = srec[q - chunk_lo];
#pragma unroll
                    for (int k = 0; k < OPT; k++) { cu[k] = pair_hash(ObjHash{b[k], ab[k]}, r.x, r.z, r.w); cj[k] = q; }
                    q++;
                }
#pragma unroll 4
                for (; q < seg_hi; q++) {
                    const uint4 r = srec[q - chunk_lo];
#pragma unroll
                    for (int k = 0; k < OPT; k++) {
                        const uint32_t u = pair_hash(ObjHash{b[k], ab[k]}, r.x, r.z, r.w);
                        if (u > cu[k]) { cu[k] = u; cj[k] = q; }
                    }
                }
                if (seg_hi == c_end) {         // class complete: one -log2 and one 64-bit compare per object
#pragma unroll
                    for (int k = 0; k < OPT; k++) {
                        const uint64_t sc = (uint64_t)elog(cu[k]) * c_invw;
                        // cj may live in another chunk by now: fetch its node index from global (rare, cached)
                        const uint32_t nid = __ldg(&tab.recs[cj[k]].nidx);
                        if (cand_better(sc, cu[k], nid, best_sc[k], best_u[k], best_i[k])) { best_sc[k] = sc; best_u[k] = cu[k]; best_i[k] = nid; }
                    }
                    c++;
                    if (c < tab.n_classes) { ClassRec r0 = tab.classes[c], r1 = tab.classes[c + 1]; c_start = r0.start; c_invw = r0.invw; c_end = r1.start; }
                }
            }
        }
#pragma unroll
        for (int k = 0; k < OPT; k++) {
            if (!valid[k]) continue;
            out_idx[oi[k]] = best_i[k];
            if (best_i[k] != kNone) {
                if (hist_bins) atomicAdd(&shist[best_i[k]], 1u);
                else if (counters) atomicAdd(&counters[best_i[k]], 1u);
            }
        }
    }
    if (hist_bins) {
        __syncthreads();
        if (counters)
            for (uint32_t j = threadIdx.x; j < hist_bins; j += blockDim.x) { uint32_t v = shist[j]; if (v) atomicAdd(&counters[j], v); }
    }
}


// ---- v2: grouped 3-input max, index resolved afterwards -------------------------------------------------
// Per pair only the hash (IMAD, IMAD) and half a VIMNMX3 are issued: the running maximum of a
// group of <= 32 consecutive nodes of one weight class is folded with __vimax3_u32, the group that raised the
// class maximum is remembered by its start position, and the node index is recovered at the very end by
// re-hashing the single winning group (<= 32 pairs per object, ~3 % extra at M = 1024).
// Full groups run BLK nodes of straight-line code per loop trip (no bounds inside); the partial group that ends
// a class runs 8-node blocks, then pairs, then a single node.  Positions are 16-bit (the launcher sends larger
// tables to k_assign_hrw): a group is remembered as (class end << 16) | group start, one register per object.
constexpr uint32_t kGroup = 32;
constexpr uint32_t kV2MaxLive = 0xFFFF;
constexpr uint32_t kV2Slack = kGroup;   // records behind the shared-memory table that the index scan may read (never matches)

// The scan against the table in global memory, last position first so the lowest position that reproduces
// u_target wins: tables larger than one shared-memory chunk, and the tie path below.  Out of line: rare, and it
// keeps registers and instruction cache for the kernel body.
__device__ __noinline__ uint32_t resolve_in_group_global(uint32_t b, uint32_t ab, const uint4 *grec, uint32_t pk, uint32_t u_target) {
    const ObjHash o{b, ab};
    const uint32_t gs = pk & 0xFFFFu, cend = pk >> 16;
    uint32_t nid = kNone;
    for (uint32_t q = min(gs + kGroup, cend); q-- > gs;) {
        const uint4 r = __ldg(grec + q);
        if (pair_hash(o, r.x, r.z, r.w) == u_target) nid = r.y;
    }
    return nid;
}

// Two classes with EQUAL 64-bit scores (rare: ~2^-40 per class pair): the larger u wins, and an exact (score, u)
// tie goes to the lower node index (spec 3.4).  Out of line so the common path is two compares and a branch.
__device__ __noinline__ bool equal_score_takes(uint32_t b, uint32_t ab, const uint4 *grec, uint32_t pk_new, uint32_t pk_old, uint32_t u_new, uint32_t u_old) {
    if (u_new != u_old) return u_new > u_old;
    if (pk_old == 0) return false;
    return resolve_in_group_global(b, ab, grec, pk_new, u_new) < resolve_in_group_global(b, ab, grec, pk_old, u_old);
}

template <int OPT, int MINB, int BLK>
__global__ void __launch_bounds__(kAssignThreads, MINB)
k_assign_hrw_v2(const uint64_t *__restrict__ keys, uint64_t n_work, NodeTabDev tab, uint32_t *__restrict__ out_idx,
                uint32_t *__restrict__ counters, const uint32_t *__restrict__ sel, uint32_t chunk_cap, uint32_t hist_bins) {
    static_assert(BLK == 8 || BLK == 16 || BLK == 32, "BLK divides the group");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint4 *srec = reinterpret_cast<uint4 *>(smem_raw);
    uint32_t *shist = reinterpret_cast<uint32_t *>(smem_raw + (size_t)(chunk_cap + kV2Slack) * sizeof(uint4));
    const uint32_t n_live = tab.n_live;
    const bool single_chunk = n_live <= chunk_cap;
    const uint4 *grec = reinterpret_cast<const uint4 *>(tab.recs);

    for (uint32_t j = threadIdx.x; j < hist_bins; j += blockDim.x) shist[j] = 0;
    if (single_chunk)
        for (uint32_t j = threadIdx.x; j < n_live; j += blockDim.x) srec[j] = __ldg(grec + j);
    __syncthreads();

#define RIO_FOLD_PAIR(R0, R1)                                                                                                        \
    _Pragma("unroll") for (int k = 0; k < OPT; k++)                                                                                  \
        gm[k] = __vimax3_u32(gm[k], pair_hash(ObjHash{b[k], ab[k]}, (R0).x, (R0).z, (R0).w), pair_hash(ObjHash{b[k], ab[k]}, (R1).x, (R1).z, (R1).w))
#define RIO_GROUP_DONE(GPK)                                                                                                          \
    _Pragma("unroll") for (int k = 0; k < OPT; k++) if (gm[k] > cu[k]) { cu[k] = gm[k]; cgs[k] = (GPK); }

    const uint64_t tile_objs = (uint64_t)kAssignThreads * OPT;
    const uint64_t n_tiles = (n_work + tile_objs - 1) / tile_objs;
    for (uint64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        uint32_t b[OPT], ab[OPT];
        uint64_t best_sc[OPT];
        uint32_t best_u[OPT], best_pk[OPT];
#pragma unroll
        for (int k = 0; k < OPT; k++) {
            const uint64_t t = tile * tile_objs + (uint64_t)k * kAssignThreads + threadIdx.x;
            const bool valid = t < n_work;
            const uint64_t oi = valid ? (sel ? (uint64_t)__ldg(sel + t) : t) : 0;
            const uint64_t key = valid ? __ldg(keys + oi) : 0;
            const ObjHash o = obj_hash(key);
            b[k] = o.b; ab[k] = o.ab;
            best_sc[k] = ~0ull; best_u[k] = 0; best_pk[k] = 0;
        }
        uint32_t c = 0, c_start = 0, c_end = 0, c_invw = 0;
        if (n_live) { ClassRec r0 = tab.classes[0], r1 = tab.classes[1]; c_start = r0.start; c_invw = r0.invw; c_end = r1.start; }
        uint32_t cu[OPT], cgs[OPT];
#pragma unroll
        for (int k = 0; k < OPT; k++) { cu[k] = 0; cgs[k] = 0; }

        for (uint32_t chunk_lo = 0; chunk_lo < n_live; chunk_lo += chunk_cap) {
            const uint32_t chunk_hi = min(n_live, chunk_lo + chunk_cap);
            if (!single_chunk) {
                __syncthreads();
                for (uint32_t j = chunk_lo + threadIdx.x; j < chunk_hi; j += blockDim.x) srec[j - chunk_lo] = __ldg(grec + j);
                __syncthreads();
            }
            uint32_t q = chunk_lo;
            while (q < chunk_hi) {
                const uint32_t seg_hi = min(c_end, chunk_hi);
                const uint32_t cend_pk = c_end << 16;
                if (q == c_start) {
#pragma unroll
                    for (int k = 0; k < OPT; k++) { cu[k] = 0; cgs[k] = q | cend_pk; }
                }
                uint32_t g = q;
                for (; g + kGroup <= seg_hi; g += kGroup) {       // full groups
                    uint32_t gm[OPT];
#pragma unroll
                    for (int k = 0; k < OPT; k++) gm[k] = 0;
#pragma unroll 1
                    for (uint32_t i0 = 0; i0 < kGroup; i0 += BLK) {
                        const uint4 *s = srec + (g - chunk_lo) + i0;
#pragma unroll
                        for (int i = 0; i < BLK; i += 2) { const uint4 r0 = s[i], r1 = s[i + 1]; RIO_FOLD_PAIR(r0, r1); }
                    }
                    RIO_GROUP_DONE(g | cend_pk);
                }
                if (g < seg_hi) {                                 // the partial group that ends the segment: 16 + 8 + 4 + 2 + 1
                    uint32_t gm[OPT];
#pragma unroll
                    for (int k = 0; k < OPT; k++) gm[k] = 0;
                    const uint32_t rem = seg_hi - g;              // 1..31; each power-of-two piece is straight-line
                    const uint4 *s = srec + (g - chunk_lo);
#pragma unroll
                    for (int piece = 16; piece >= 2; piece >>= 1) {
                        if (rem & piece) {
#pragma unroll
                            for (int i = 0; i < piece; i += 2) { const uint4 r0 = s[i], r1 = s[i + 1]; RIO_FOLD_PAIR(r0, r1); }
                            s += piece;
                        }
                    }
                    if (rem & 1) {
                        const uint4 r0 = s[0];
#pragma unroll
                        for (int k = 0; k < OPT; k++) gm[k] = max(gm[k], pair_hash(ObjHash{b[k], ab[k]}, r0.x, r0.z, r0.w));
                    }
                    RIO_GROUP_DONE(g | cend_pk);
                }
                q = seg_hi;
                if (seg_hi == c_end) {
                    uint64_t sc[OPT];
#pragma unroll
                    for (int k = 0; k < OPT; k++) sc[k] = (uint64_t)elog(cu[k]) * c_invw;    // OPT independent chains
#pragma unroll
                    for (int k = 0; k < OPT; k++) {
                        bool take = sc[k] < best_sc[k];
                        if (sc[k] == best_sc[k]) take = equal_score_takes(b[k], ab[k], grec, cgs[k], best_pk[k], cu[k], best_u[k]);
                        if (take) { best_sc[k] = sc[k]; best_u[k] = cu[k]; best_pk[k] = cgs[k]; }
                    }
                    c++;
                    if (c < tab.n_classes) { ClassRec r0 = tab.classes[c], r1 = tab.classes[c + 1]; c_start = r0.start; c_invw = r0.invw; c_end = r1.start; }
                }
            }
        }
        // recover the node index: re-hash the winning group, last position first so the lowest one wins; no early
        // exit and positions past the class end predicated off, so the OPT scans of a thread interleave
        uint32_t nid[OPT];
#pragma unroll
        for (int k = 0; k < OPT; k++) nid[k] = kNone;       // stays kNone only without live nodes (best_pk == 0)
        if (single_chunk) {
            // Lane L starts at offset L of its group: 32 lanes whose groups are aligned alike (one big class: every
            // group start is a multiple of 32 records = 512 B) would otherwise hit the same 4 banks 32 ways.  The
            // scan order then differs per lane, so the LOWEST matching position is kept with a min, not by order.
            // Positions past the class end may read the kV2Slack records behind the table: never a hit (pos < end).
            const uint32_t lane = threadIdx.x & 31u;
            uint32_t fpos[OPT];
#pragma unroll
            for (int k = 0; k < OPT; k++) fpos[k] = kNone;
#pragma unroll 8
            for (int i = 0; i < (int)kGroup; i++) {
                const uint32_t off = (lane + (uint32_t)i) & (kGroup - 1);
#pragma unroll
                for (int k = 0; k < OPT; k++) {
                    const uint32_t pos = (best_pk[k] & 0xFFFFu) + off;
                    const uint4 r = srec[pos];
                    const bool hit = pair_hash(ObjHash{b[k], ab[k]}, r.x, r.z, r.w) == best_u[k] && pos < (best_pk[k] >> 16);
                    fpos[k] = min(fpos[k], hit ? pos : kNone);
                }
            }
#pragma unroll
            for (int k = 0; k < OPT; k++) nid[k] = fpos[k] != kNone ? srec[fpos[k]].y : kNone;
        } else {
#pragma unroll
            for (int k = 0; k < OPT; k++) nid[k] = resolve_in_group_global(b[k], ab[k], grec, best_pk[k], best_u[k]);
        }
#pragma unroll
        for (int k = 0; k < OPT; k++) {
            const uint64_t t = tile * tile_objs + (uint64_t)k * kAssignThreads + threadIdx.x;
            if (t >= n_work) continue;
            out_idx[sel ? (uint64_t)__ldg(sel + t) : t] = nid[k];
            if (nid[k] != kNone) {
                if (hist_bins) atomicAdd(&shist[nid[k]], 1u);
                else if (counters) atomicAdd(&counters[nid[k]], 1u);
            }
        }
    }
#undef RIO_FOLD_PAIR
#undef RIO_GROUP_DONE
    if (hist_bins) {
        __syncthreads();
        if (counters)
            for (uint32_t j = threadIdx.x; j < hist_bins; j += blockDim.x) { uint32_t v = shist[j]; if (v) atomicAdd(&counters[j], v); }
    }
}

// ---- affinity cost, CUDA-core fp32 path (exact summation order k = 0..K-1 with fmaf) -------------------
// cost_ij = -sum_k Fobj[i,k] * Fnode[j,k]; argmin, ties -> lowest j (DESIGN.md 3.6).
template <int K, int OPT>
__global__ void __launch_bounds__(kAssignThreads, 2)
k_assign_affinity(const float *__restrict__ fobj, uint64_t n, const float *__restrict__ fnode, const uint32_t *__restrict__ live,
                  uint32_t n_total, uint32_t *__restrict__ out_idx, float *__restrict__ out_cost, uint32_t *__restrict__ counters,
                  uint32_t chunk_cap) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *snode = reinterpret_cast<float *>(smem_raw);                               // chunk_cap x K
    uint32_t *slive = reinterpret_cast<uint32_t *>(smem_raw + (size_t)chunk_cap * K * 4);  // chunk_cap
    const uint64_t tile_objs = (uint64_t)kAssignThreads * OPT;
    const uint64_t n_tiles = (n + tile_objs - 1) / tile_objs;
    const bool single_chunk = n_total <= chunk_cap;
    if (single_chunk) {
        for (uint32_t t = threadIdx.x; t < n_total * K; t += blockDim.x) snode[t] = __ldg(fnode + t);
        for (uint32_t t = threadIdx.x; t < n_total; t += blockDim.x) slive[t] = __ldg(live + t);
        __syncthreads();
    }
    for (uint64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        float fo[OPT][K];
        float best[OPT];
        uint32_t bi[OPT];
        uint64_t oi[OPT];
        bool valid[OPT];
#pragma unroll
        for (int o = 0; o < OPT; o++) {
            oi[o] = tile * tile_objs + (uint64_t)o * kAssignThreads + threadIdx.x;
            valid[o] = oi[o] < n;
            const float4 *row = reinterpret_cast<const float4 *>(fobj + (valid[o] ? oi[o] : 0) * K);
#pragma unroll
            for (int k4 = 0; k4 < K / 4; k4++) {
                float4 v = __ldg(row + k4);
                fo[o][4 * k4 + 0] = v.x; fo[o][4 * k4 + 1] = v.y; fo[o][4 * k4 + 2] = v.z; fo[o][4 * k4 + 3] = v.w;
            }
            best[o] = 0.f; bi[o] = kNone;
        }
        for (uint32_t chunk_lo = 0; chunk_lo < n_total; chunk_lo += chunk_cap) {
            const uint32_t chunk_hi = min(n_total, chunk_lo + chunk_cap);
            if (!single_chunk) {
                __syncthreads();
                for (uint32_t t = threadIdx.x; t < (chunk_hi - chunk_lo) * K; t += blockDim.x) snode[t] = __ldg(fnode + (size_t)chunk_lo * K + t);
                for (uint32_t t = threadIdx.x; t < chunk_hi - chunk_lo; t += blockDim.x) slive[t] = __ldg(live + chunk_lo + t);
                __syncthreads();
            }
            for (uint32_t j = chunk_lo; j < chunk_hi; j++) {
                if (!slive[j - chunk_lo]) continue;     // block-uniform
                const float4 *nr = reinterpret_cast<const float4 *>(snode + (size_t)(j - chunk_lo) * K);
                float acc[OPT];
#pragma unroll
                for (int o = 0; o < OPT; o++) acc[o] = 0.f;
#pragma unroll
                for (int k4 = 0; k4 < K / 4; k4++) {
                    const float4 v = nr[k4];
#pragma unroll
                    for (int o = 0; o < OPT; o++) {
                        acc[o] = fmaf(fo[o][4 * k4 + 0], v.x, acc[o]);
                        acc[o] = fmaf(fo[o][4 * k4 + 1], v.y, acc[o]);
                        acc[o] = fmaf(fo[o][4 * k4 + 2], v.z, acc[o]);
                        acc[o] = fmaf(fo[o][4 * k4 + 3], v.w, acc[o]);
                    }
                }
#pragma unroll
                for (int o = 0; o < OPT; o++) {
                    const float cst = -acc[o];
                    if (bi[o] == kNone || cst < best[o]) { best[o] = cst; bi[o] = j; }
                }
            }
        }
#pragma unroll
        for (int o = 0; o < OPT; o++) {
            if (!valid[o]) continue;
            out_idx[oi[o]] = bi[o];
            if (out_cost) out_cost[oi[o]] = best[o];
            if (counters && bi[o] != kNone) atomicAdd(&counters[bi[o]], 1u);
        }
    }
}

// generic K (any K >= 1): one thread per object, node rows streamed through L1/L2
__global__ void __launch_bounds__(kAssignThreads)
k_assign_affinity_generic(const float *__restrict__ fobj, uint64_t n, const float *__restrict__ fnode, const uint32_t *__restrict__ live,
                          uint32_t n_total, uint32_t K, uint32_t *__restrict__ out_idx, float *__restrict__ out_cost,
                          uint32_t *__restrict__ counters) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const float *fo = fobj + i * K;
        float best = 0.f; uint32_t bi = kNone;
        for (uint32_t j = 0; j < n_total; j++) {
            if (!__ldg(live + j)) continue;
            const float *fn = fnode + (size_t)j * K;
            float acc = 0.f;
            for (uint32_t k = 0; k < K; k++) acc = fmaf(__ldg(fo + k), __ldg(fn + k), acc);
            const float cst = -acc;
            if (bi == kNone || cst < best) { best = cst; bi = j; }
        }
        out_idx[i] = bi;
        if (out_cost) out_cost[i] = best;
        if (counters && bi != kNone) atomicAdd(&counters[bi], 1u);
    }
}

// Ranked lists (DESIGN.md 3.9) on the CUDA cores: the node loop and fmaf order of k_assign_affinity / k_assign_affinity_generic,
// one object per thread, and the RT smallest (cost, j) kept sorted in registers.  A node displaces an entry only with a strictly
// smaller cost, so equal costs keep the lower j first and the first entry is the unranked kernels' node.  KC = 16 keeps the object
// row in registers; KC = 0 takes any K at run time.  The first `ranks` (<= RT) entries are written, kNone past the live set.
// SPREAD (DESIGN.md 3.14): the list keeps one entry per failure domain (ndom: dense domain id per interned index).  A node of a
// listed domain replaces that entry only with a strictly smaller cost; any other node enters only by beating the last entry.  The
// list is then the best RT domain representatives, so its first `ranks` entries are the failure-domain list.
template <int KC, int RT, bool SPREAD>
__global__ void __launch_bounds__(kAssignThreads)
k_assign_affinity_ranked(const float *__restrict__ fobj, uint64_t n, const float *__restrict__ fnode, const uint32_t *__restrict__ live,
                         uint32_t n_total, uint32_t K, uint32_t ranks, uint32_t *__restrict__ out_idx, const uint32_t *__restrict__ ndom) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        float fo[KC ? KC : 1];
        if constexpr (KC != 0) {
            const float4 *row = reinterpret_cast<const float4 *>(fobj + i * KC);
#pragma unroll
            for (int k4 = 0; k4 < KC / 4; k4++) {
                const float4 v = __ldg(row + k4);
                fo[4 * k4 + 0] = v.x; fo[4 * k4 + 1] = v.y; fo[4 * k4 + 2] = v.z; fo[4 * k4 + 3] = v.w;
            }
        }
        float lc[RT];
        uint32_t lj[RT], ld[SPREAD ? RT : 1];
#pragma unroll
        for (int s = 0; s < RT; s++) { lc[s] = 0.f; lj[s] = kNone; }
        if constexpr (SPREAD) {
#pragma unroll
            for (int s = 0; s < RT; s++) ld[s] = kNone;
        }
        for (uint32_t j = 0; j < n_total; j++) {
            if (!__ldg(live + j)) continue;
            float acc = 0.f;
            if constexpr (KC != 0) {
                const float4 *nr = reinterpret_cast<const float4 *>(fnode + (size_t)j * KC);
#pragma unroll
                for (int k4 = 0; k4 < KC / 4; k4++) {
                    const float4 v = __ldg(nr + k4);
                    acc = fmaf(fo[4 * k4 + 0], v.x, acc);
                    acc = fmaf(fo[4 * k4 + 1], v.y, acc);
                    acc = fmaf(fo[4 * k4 + 2], v.z, acc);
                    acc = fmaf(fo[4 * k4 + 3], v.w, acc);
                }
            } else {
                const float *fi = fobj + i * K, *fn = fnode + (size_t)j * K;
                for (uint32_t k = 0; k < K; k++) acc = fmaf(__ldg(fi + k), __ldg(fn + k), acc);
            }
            const float cst = -acc;
            if (lj[RT - 1] != kNone && !(cst < lc[RT - 1])) continue;
            if constexpr (SPREAD) {
                // j is larger than every listed index, so "listed before it" is "cost not larger"; the swap chain below carries
                // listed entries, which compare by (cost, index), and stops at the entry of the candidate's own domain
                const uint32_t dc = __ldg(ndom + j);
                bool keep = true;
#pragma unroll
                for (int s = 0; s < RT; s++) keep &= !(ld[s] == dc && !(cst < lc[s]));
                if (!keep) continue;
                float c = cst;
                uint32_t cj = j, cd = dc;
                bool go = true;
#pragma unroll
                for (int s = 0; s < RT; s++) {
                    const bool sw = go && (lj[s] == kNone || c < lc[s] || (c == lc[s] && cj < lj[s]));
                    const float tc = lc[s];
                    const uint32_t tj = lj[s], td = ld[s];
                    lc[s] = sw ? c : tc; lj[s] = sw ? cj : tj; ld[s] = sw ? cd : td;
                    c = sw ? tc : c; cj = sw ? tj : cj; cd = sw ? td : cd;
                    go = go && !(sw && td == dc);
                }
            } else {
#pragma unroll
                for (int s = RT - 1; s > 0; s--) {
                    if (lj[s - 1] == kNone || cst < lc[s - 1]) { lc[s] = lc[s - 1]; lj[s] = lj[s - 1]; }
                    else if (lj[s] == kNone || cst < lc[s]) { lc[s] = cst; lj[s] = j; }
                }
                if (lj[0] == kNone || cst < lc[0]) { lc[0] = cst; lj[0] = j; }
            }
        }
#pragma unroll
        for (int s = 0; s < RT; s++)
            if (s < (int)ranks) out_idx[i * ranks + s] = lj[s];
    }
}


// Register-only replay of the assign inner loop (same IMAD / IMAD / VIMNMX3 mix, no shared or global
// memory in the loop): its pair rate is the integer-ALU roofline the assign kernel is reported against.
__global__ void __launch_bounds__(kAssignThreads, 2)
k_mix_rate(uint32_t iters, uint32_t *sink) {
    uint32_t b[4], ab[4], gm[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {   // opaque per-object constants (read from memory so the compiler cannot relate them)
        b[k] = sink[8 + ((threadIdx.x * 8 + k) & 255)] | 1u; ab[k] = sink[8 + ((threadIdx.x * 8 + 4 + k) & 255)]; gm[k] = 0;
    }
    // per-thread (not warp-uniform) node constants, so that the xor stays ONE 3-input LOP3 like in the real loop
    uint32_t s0a = sink[8 + ((threadIdx.x + 64) & 255)] + blockIdx.x, s0b = s0a ^ 0x7F4A7C15u;
    const uint32_t s1a = sink[8 + ((threadIdx.x + 1) & 255)] | 1u, s1b = sink[8 + ((threadIdx.x + 2) & 255)] | 1u;   // opaque, per thread
    const uint32_t s2a = sink[8 + ((threadIdx.x + 3) & 255)], s2b = sink[8 + ((threadIdx.x + 4) & 255)];
    for (uint32_t it = 0; it < iters; it++) {
#pragma unroll
        for (int r = 0; r < 8; r++) {
#pragma unroll
            for (int k = 0; k < 4; k++)
                gm[k] = __vimax3_u32(gm[k], pair_hash(ObjHash{b[k], ab[k]}, s0a, s1a, s2a), pair_hash(ObjHash{b[k], ab[k]}, s0b, s1b, s2b));
            s0a = s0a * 747796405u + 2891336453u; s0b = s0b * 1664525u + 1013904223u;   // next two "nodes": 2 IMAD per 8 pairs (the real loop has 2 LDS.128 there)
        }
    }
    if ((gm[0] ^ gm[1] ^ gm[2] ^ gm[3]) == 0x12345678u) sink[0] = gm[0];   // keep the loop alive
}

__global__ void k_synth_keys(uint64_t *__restrict__ keys, uint64_t first, uint64_t n, uint64_t seed) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
        keys[i] = synth_key(first + i, seed);
}

// FNV-1a over the joined "{type}.{id}" bytes, then mix64 (== rio_cuda_object_key).  Byte work, HBM bound:
// the block's contiguous byte range is staged into shared memory with coalesced 16-byte loads, then each
// thread walks its own id out of shared memory.
constexpr int kHashThreads = 256;
constexpr uint32_t kHashSmemBytes = 24 * 1024 - 64;   // 8 CTAs per SM: the two barriers of a trip expose a full HBM latency, more CTAs cover it
__global__ void __launch_bounds__(kHashThreads)
k_hash_ids(const char *__restrict__ packed, const uint64_t *__restrict__ offsets, uint64_t n, uint64_t *__restrict__ keys) {
    __shared__ __align__(16) unsigned char sbuf[kHashSmemBytes];
    for (uint64_t base = (uint64_t)blockIdx.x * kHashThreads; base < n; base += (uint64_t)gridDim.x * kHashThreads) {
        const uint64_t last = min(n, base + kHashThreads);
        const uint64_t lo = __ldg(offsets + base), hi = __ldg(offsets + last);
        const uint64_t lo16 = lo & ~15ull;
        const bool staged = (hi - lo16) <= kHashSmemBytes && ((uintptr_t)packed & 15) == 0;
        __syncthreads();
        if (staged) {
            const uint64_t nvec = (hi - lo16 + 15) / 16;   // may over-read up to 15 bytes inside the caller's 16B-padded buffer
            for (uint64_t v = threadIdx.x; v < nvec; v += kHashThreads)
                reinterpret_cast<uint4 *>(sbuf)[v] = __ldg(reinterpret_cast<const uint4 *>(packed + lo16) + v);
        }
        __syncthreads();
        const uint64_t i = base + threadIdx.x;
        if (i < last) {
            const uint64_t a = __ldg(offsets + i), e = __ldg(offsets + i + 1);
            uint64_t h = kFnvBasis;
            if (staged) { for (uint64_t p = a; p < e; p++) { h ^= sbuf[p - lo16]; h *= kFnvPrime; } }
            else        { for (uint64_t p = a; p < e; p++) { h ^= (uint8_t)__ldg(packed + p); h *= kFnvPrime; } }
            keys[i] = mix64(h);
        }
    }
}

__global__ void k_fill_u32(uint32_t *__restrict__ d, uint64_t n, uint32_t v) {
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) d[i] = v;
}

constexpr uint32_t kHistSmemBins = 8192;
__global__ void __launch_bounds__(256)
k_histogram(const uint32_t *__restrict__ idx, uint64_t n, uint32_t *__restrict__ counters, uint32_t n_total, uint32_t bins) {
    extern __shared__ uint32_t sh[];
    for (uint32_t j = threadIdx.x; j < bins; j += blockDim.x) sh[j] = 0;
    __syncthreads();
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t v = __ldg(idx + i);
        if (v < n_total) { if (bins) atomicAdd(&sh[v], 1u); else atomicAdd(&counters[v], 1u); }
    }
    __syncthreads();
    for (uint32_t j = threadIdx.x; j < bins; j += blockDim.x) { uint32_t v = sh[j]; if (v) atomicAdd(&counters[j], v); }
}

__global__ void k_sum_gathered(const uint32_t *__restrict__ g, uint32_t world, uint32_t M, uint32_t *__restrict__ out) {
    for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < M; j += gridDim.x * blockDim.x) {
        uint32_t s = 0;
        for (uint32_t r = 0; r < world; r++) s += g[(size_t)r * M + j];
        out[j] = s;
    }
}

inline int grid_for(uint64_t work_items, int threads, int sm_count, int blocks_per_sm) {
    uint64_t blocks = (work_items + threads - 1) / threads;
    uint64_t cap = (uint64_t)sm_count * blocks_per_sm;
    if (blocks < 1) blocks = 1;
    return (int)(blocks < cap ? blocks : cap);
}

}  // namespace

// RIO_ASSIGN_VARIANT=1 selects the straightforward per-pair compare/select kernel (kept for A/B runs);
// the default (2) is the grouped-max kernel.  Both are the product path and both must match the oracle.
static int assign_variant() {
    const char *e = getenv("RIO_ASSIGN_VARIANT");   // read per launch so tests can flip it
    return (e && e[0] == '1') ? 1 : 2;
}

// Objects one full wave of the default rendezvous launch covers (persistent CTAs x objects per tile): host code that
// pipelines chunks sizes them in whole waves so that no chunk ends on a partially filled wave.
constexpr int kV2DefaultTune = 532;   // 5 objects per thread, 3 CTAs per SM, 32-node straight-line groups
uint64_t assign_wave_objects(int sm_count) { return (uint64_t)sm_count * 3 * kAssignThreads * 5; }

void launch_assign_hrw(const Launch &L, const uint64_t *d_keys, uint64_t n, const NodeTabDev &tab, uint32_t *d_out_idx,
                       uint32_t *d_counters, const uint32_t *d_sel, uint64_t n_sel) {
    const uint64_t n_work = d_sel ? n_sel : n;
    if (!n_work) return;
    // node chunk in shared memory: up to 8192 records (128 KB); histogram bins in smem when they fit beside it
    const uint32_t chunk_cap = tab.n_live < 1 ? 1 : (tab.n_live < 8192 ? tab.n_live : 8192);
    const uint32_t hist_bins = (d_counters && tab.n_total <= 8192) ? tab.n_total : 0;
    const size_t smem = (size_t)chunk_cap * sizeof(uint4) + (size_t)hist_bins * 4;
    if (assign_variant() == 1 || tab.n_live > kV2MaxLive) {
        cudaFuncSetAttribute(k_assign_hrw<kOPT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8192 * 16 + 8192 * 4);
        const uint64_t tiles = (n_work + (uint64_t)kAssignThreads * kOPT - 1) / ((uint64_t)kAssignThreads * kOPT);
        const int bps = smem > 100 * 1024 ? 1 : 2;
        const uint64_t cap = (uint64_t)L.sm_count * bps;
        k_assign_hrw<kOPT><<<(int)(tiles < cap ? tiles : cap), kAssignThreads, smem, L.stream>>>(d_keys, n_work, tab, d_out_idx, d_counters, d_sel, chunk_cap, hist_bins);
    } else {
        // RIO_ASSIGN_TUNE="<objects per thread><min CTAs per SM><a|b|c = 8|16|32 straight-line nodes per trip>" selects a
        // compiled tuning point (A/B runs, tools/tune_assign.py)
        const char *t = getenv("RIO_ASSIGN_TUNE");
        const int tune = (t && t[0] && t[1] && t[2]) ? (t[0] - '0') * 100 + (t[1] - '0') * 10 + (t[2] - 'a') : kV2DefaultTune;
#define RIO_LAUNCH_V2(OPT_, MINB_, BLK_)                                                                                              \
        do {                                                                                                                          \
            cudaFuncSetAttribute(k_assign_hrw_v2<OPT_, MINB_, BLK_>, cudaFuncAttributeMaxDynamicSharedMemorySize, (8192 + kV2Slack) * 16 + 8192 * 4); \
            const uint64_t tiles = (n_work + (uint64_t)kAssignThreads * OPT_ - 1) / ((uint64_t)kAssignThreads * OPT_);                \
            int bps = MINB_;                                                                                                          \
            const size_t smem2 = smem + kV2Slack * sizeof(uint4);                                                                     \
            while (bps > 1 && (size_t)bps * (smem2 + 1024) > 227u * 1024u) bps--;                                                     \
            const uint64_t cap = (uint64_t)L.sm_count * bps;                                                                          \
            k_assign_hrw_v2<OPT_, MINB_, BLK_><<<(int)(tiles < cap ? tiles : cap), kAssignThreads, smem2, L.stream>>>(d_keys, n_work, tab, d_out_idx, \
                                                                                                                  d_counters, d_sel, chunk_cap, hist_bins); \
        } while (0)
        switch (tune) {
#ifdef RIO_ASSIGN_TUNING   // A/B tuning points (RIO_BUILD_TUNING=1): not in the shipped library
            case 430: RIO_LAUNCH_V2(4, 3, 8); break;
            case 431: RIO_LAUNCH_V2(4, 3, 16); break;
            case 432: RIO_LAUNCH_V2(4, 3, 32); break;
            case 420: RIO_LAUNCH_V2(4, 2, 8); break;
            case 422: RIO_LAUNCH_V2(4, 2, 32); break;
            case 820: RIO_LAUNCH_V2(8, 2, 8); break;
            case 822: RIO_LAUNCH_V2(8, 2, 32); break;
            case 240: RIO_LAUNCH_V2(2, 4, 8); break;
            case 342: RIO_LAUNCH_V2(3, 4, 32); break;
            case 332: RIO_LAUNCH_V2(3, 3, 32); break;
            case 622: RIO_LAUNCH_V2(6, 2, 32); break;
            case 522: RIO_LAUNCH_V2(5, 2, 32); break;
#endif
            case 532: default: RIO_LAUNCH_V2(5, 3, 32); break;
        }
#undef RIO_LAUNCH_V2
    }
    RIO_COUNT_LAUNCH(L);
}

void launch_assign_affinity(const Launch &L, const float *d_fobj, uint64_t n, const float *d_fnode, const uint32_t *d_live, uint32_t n_total,
                            uint32_t K, uint32_t *d_out_idx, float *d_out_cost, uint32_t *d_counters) {
    if (!n) return;
    if (K == 16) {
        constexpr int OPT = 2;
        const uint32_t chunk_cap = n_total < 1 ? 1 : (n_total < 2048 ? n_total : 2048);
        const size_t smem = (size_t)chunk_cap * (16 * 4 + 4);
        cudaFuncSetAttribute(k_assign_affinity<16, OPT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 2048 * 68);
        const uint64_t tiles = (n + (uint64_t)kAssignThreads * OPT - 1) / ((uint64_t)kAssignThreads * OPT);
        uint64_t cap = (uint64_t)L.sm_count * (smem > 100 * 1024 ? 1 : 2);
        int grid = (int)(tiles < cap ? tiles : cap);
        k_assign_affinity<16, OPT><<<grid, kAssignThreads, smem, L.stream>>>(d_fobj, n, d_fnode, d_live, n_total, d_out_idx, d_out_cost, d_counters, chunk_cap);
    } else {
        k_assign_affinity_generic<<<grid_for(n, kAssignThreads, L.sm_count, 8), kAssignThreads, 0, L.stream>>>(d_fobj, n, d_fnode, d_live, n_total, K,
                                                                                                       d_out_idx, d_out_cost, d_counters);
    }
    RIO_COUNT_LAUNCH(L);
}

template <int KC, bool SPREAD>
static void launch_affinity_ranked_k(const Launch &L, const float *d_fobj, uint64_t n, const float *d_fnode, const uint32_t *d_live, uint32_t n_total,
                                     uint32_t K, uint32_t ranks, uint32_t *d_out_idx, const uint32_t *d_ndom) {
    const int grid = grid_for(n, kAssignThreads, L.sm_count, 8);
    switch (affinity_ranked_groups(ranks)) {
        case 1: k_assign_affinity_ranked<KC, 1, SPREAD><<<grid, kAssignThreads, 0, L.stream>>>(d_fobj, n, d_fnode, d_live, n_total, K, ranks, d_out_idx, d_ndom); break;
        case 2: k_assign_affinity_ranked<KC, 2, SPREAD><<<grid, kAssignThreads, 0, L.stream>>>(d_fobj, n, d_fnode, d_live, n_total, K, ranks, d_out_idx, d_ndom); break;
        case 4: k_assign_affinity_ranked<KC, 4, SPREAD><<<grid, kAssignThreads, 0, L.stream>>>(d_fobj, n, d_fnode, d_live, n_total, K, ranks, d_out_idx, d_ndom); break;
        default: k_assign_affinity_ranked<KC, 8, SPREAD><<<grid, kAssignThreads, 0, L.stream>>>(d_fobj, n, d_fnode, d_live, n_total, K, ranks, d_out_idx, d_ndom); break;
    }
}

void launch_assign_affinity_ranked(const Launch &L, const float *d_fobj, uint64_t n, const float *d_fnode, const uint32_t *d_live, uint32_t n_total,
                                   uint32_t K, uint32_t ranks, uint32_t *d_out_idx) {
    if (!n) return;
    if (K == 16) launch_affinity_ranked_k<16, false>(L, d_fobj, n, d_fnode, d_live, n_total, K, ranks, d_out_idx, nullptr);
    else launch_affinity_ranked_k<0, false>(L, d_fobj, n, d_fnode, d_live, n_total, K, ranks, d_out_idx, nullptr);
    RIO_COUNT_LAUNCH(L);
}

void launch_assign_affinity_spread(const Launch &L, const float *d_fobj, uint64_t n, const float *d_fnode, const uint32_t *d_live, uint32_t n_total,
                                   uint32_t K, const uint32_t *d_ndom, uint32_t ranks, uint32_t *d_out_idx) {
    if (!n) return;
    if (K == 16) launch_affinity_ranked_k<16, true>(L, d_fobj, n, d_fnode, d_live, n_total, K, ranks, d_out_idx, d_ndom);
    else launch_affinity_ranked_k<0, true>(L, d_fobj, n, d_fnode, d_live, n_total, K, ranks, d_out_idx, d_ndom);
    RIO_COUNT_LAUNCH(L);
}

// returns pairs evaluated by the launch
uint64_t launch_mix_rate(const Launch &L, uint32_t iters, uint32_t *d_sink) {
    const int grid = L.sm_count * 2 * 8;
    k_mix_rate<<<grid, kAssignThreads, 0, L.stream>>>(iters, d_sink);
    RIO_COUNT_LAUNCH(L);
    return (uint64_t)grid * kAssignThreads * (uint64_t)iters * 8 * 4 * 2;
}

void launch_synth_keys(const Launch &L, uint64_t *d_keys, uint64_t first, uint64_t n, uint64_t seed) {
    if (!n) return;
    k_synth_keys<<<grid_for(n, 256, L.sm_count, 8), 256, 0, L.stream>>>(d_keys, first, n, seed);
    RIO_COUNT_LAUNCH(L);
}

void launch_hash_ids(const Launch &L, const char *d_packed, const uint64_t *d_offsets, uint64_t n, uint64_t *d_keys) {
    if (!n) return;
    k_hash_ids<<<grid_for(n, kHashThreads, L.sm_count, 8), kHashThreads, 0, L.stream>>>(d_packed, d_offsets, n, d_keys);
    RIO_COUNT_LAUNCH(L);
}

void launch_fill_u32(const Launch &L, uint32_t *d, uint64_t n, uint32_t v) {
    if (!n) return;
    k_fill_u32<<<grid_for(n, 256, L.sm_count, 8), 256, 0, L.stream>>>(d, n, v);
    RIO_COUNT_LAUNCH(L);
}

void launch_histogram(const Launch &L, const uint32_t *d_idx, uint64_t n, uint32_t *d_counters, uint32_t n_total) {
    if (!n) return;
    const uint32_t bins = n_total <= kHistSmemBins ? n_total : 0;
    k_histogram<<<grid_for(n, 256, L.sm_count, 4), 256, (size_t)bins * 4, L.stream>>>(d_idx, n, d_counters, n_total, bins);
    RIO_COUNT_LAUNCH(L);
}

void launch_sum_gathered(const Launch &L, const uint32_t *d_gathered, uint32_t world, uint32_t M, uint32_t *d_out) {
    if (!M) return;
    k_sum_gathered<<<(M + 255) / 256, 256, 0, L.stream>>>(d_gathered, world, M, d_out);
    RIO_COUNT_LAUNCH(L);
}

void launch_l2_flush(const Launch &L, uint32_t *d_buf, uint64_t n_words, uint32_t v) { launch_fill_u32(L, d_buf, n_words, v); }

}  // namespace rio

// k_affinity_umma.cu -- affinity-cost placement on the Hopper tensor cores (wgmma), K = 16.
//
//   cost_ij = -sum_k Fobj[i,k] * Fnode[j,k]   ->  per-object argmin over the live nodes   (DESIGN.md 3.6 / 5.3)
//
// This is the one dense contraction on the path, so it is the one place tensor cores are used.  fp32 inputs are split
// on the fly into three bf16 pieces (a = a_h + a_m + a_l exactly) and the product is rebuilt from six cross terms
// (hh, hm, mh, mm, hl, lh; the dropped terms are <= 2^-24 relative), each term ONE wgmma (M=64 objects x N=NT nodes x
// K=16) accumulating in fp32 registers.  Nothing is materialised in HBM: the N x M grid lives only in registers.
//
// One CTA per SM, four warpgroups, persistent over 64-object row blocks (each warpgroup walks its own row blocks):
//   - node operands (3 bf16 blocks, 96 B per node, K-major no-swizzle core matrices) are staged once into shared memory
//     and stay resident for the whole kernel; they are the wgmma B operand, read through a shared-memory descriptor;
//   - the object rows are the A operand straight from registers: every thread loads the 8 features its A fragment needs
//     (two rows, k = 2q, 2q+1, 2q+8, 2q+9), splits them and packs the h/m/l fragments; the next row block's features are
//     requested before the current one is scored, so their HBM latency hides behind the tensor-core work;
//   - per node tile a warpgroup issues six wgmma into one register accumulator of NT columns, waits, and reduces it to a
//     running (best value, best group of 8 columns) per row.  The tensor core stays busy during a reduction with the other
//     three warpgroups' tiles.  (Two accumulators in one warpgroup make ptxas serialise every wgmma: reading the finished
//     accumulator while the other one is in flight is not something it proves safe.)  At the end of the row block the four
//     lanes that share a row merge their candidates and only the winning group leaves this kernel.
// k_affinity_resolve (second pass, CUDA cores) re-evaluates the 8 candidates of each winning group in fp32: node index +
// fp32 cost + per-node histogram.
#include "kernels.cuh"
#include "k_affinity_ranked.cuh"
#include "k_affinity_spread.cuh"
#include "spec.cuh"

#include <cuda_bf16.h>
#include <cstdlib>

namespace rio {

namespace {

constexpr int kWarpgroups = 4;
constexpr int kWgThreads = 128 * kWarpgroups;
constexpr int kRows = 64;         // objects per row block == wgmma M

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving reads of an accumulator across the wgmma.wait_group that makes it valid
template <int C>
__device__ __forceinline__ void fence_regs(float (&d)[C]) {
#pragma unroll
    for (int i = 0; i < C; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] (+)= A[64 x 16] (registers, bf16) * B[N x 16]^T (shared memory, bf16, K-major), fp32 accumulate
template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate);
template <> __device__ __forceinline__ void wgmma_bf16<64>(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
                 "{"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
                 "}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}
template <> __device__ __forceinline__ void wgmma_bf16<128>(float (&d)[64], const uint32_t (&a)[4], uint64_t desc_b, uint32_t accumulate) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
                 "{"
                 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
                 "}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(accumulate));
}

// K-major, no-swizzle ("interleave") shared-memory operand descriptor: 8-row x 16-byte core matrices,
// LBO = byte distance between the two 16-byte K chunks, SBO = byte distance between 8-row groups.
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((saddr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32);
    // base offset 0, layout type 0 (no swizzle)
}

// fp32 -> three bf16 pieces with a == h + m + l exactly
__device__ __forceinline__ void split3(float a, __nv_bfloat16 &h, __nv_bfloat16 &m, __nv_bfloat16 &l) {
    h = __float2bfloat16_rn(a);
    const float r1 = a - __bfloat162float(h);
    m = __float2bfloat16_rn(r1);
    l = __float2bfloat16_rn(r1 - __bfloat162float(m));
}
__device__ __forceinline__ uint32_t pack2(__nv_bfloat16 lo, __nv_bfloat16 hi) {
    return (uint32_t)__bfloat16_as_ushort(lo) | ((uint32_t)__bfloat16_as_ushort(hi) << 16);
}

// Split one fp32 row of 16 features and store it as row `r` of the three operand blocks at `base`
// (block x at base + x*block_bytes; inside a block: [k-chunk][row][16 B], chunk stride = chunk_stride bytes).
__device__ __forceinline__ void store_row_split(unsigned char *base, uint32_t block_bytes, uint32_t chunk_stride, uint32_t r, const float (&f)[16]) {
    __nv_bfloat16 h[16], m[16], l[16];
#pragma unroll
    for (int k = 0; k < 16; k++) split3(f[k], h[k], m[k], l[k]);
#pragma unroll
    for (int kc = 0; kc < 2; kc++) {
        uint4 vh = make_uint4(pack2(h[kc * 8 + 0], h[kc * 8 + 1]), pack2(h[kc * 8 + 2], h[kc * 8 + 3]), pack2(h[kc * 8 + 4], h[kc * 8 + 5]), pack2(h[kc * 8 + 6], h[kc * 8 + 7]));
        uint4 vm = make_uint4(pack2(m[kc * 8 + 0], m[kc * 8 + 1]), pack2(m[kc * 8 + 2], m[kc * 8 + 3]), pack2(m[kc * 8 + 4], m[kc * 8 + 5]), pack2(m[kc * 8 + 6], m[kc * 8 + 7]));
        uint4 vl = make_uint4(pack2(l[kc * 8 + 0], l[kc * 8 + 1]), pack2(l[kc * 8 + 2], l[kc * 8 + 3]), pack2(l[kc * 8 + 4], l[kc * 8 + 5]), pack2(l[kc * 8 + 6], l[kc * 8 + 7]));
        const uint32_t off = kc * chunk_stride + r * 16;
        *reinterpret_cast<uint4 *>(base + 0 * block_bytes + off) = vh;
        *reinterpret_cast<uint4 *>(base + 1 * block_bytes + off) = vm;
        *reinterpret_cast<uint4 *>(base + 2 * block_bytes + off) = vl;
    }
}

struct WgmmaParams {
    const float *fobj;        // n x 16
    uint64_t n;
    const float *fnode_c;     // m_pad x 16 fp32, live nodes compacted in node-index order, zero padded
    uint32_t n_live, m_pad;
    uint32_t *out_idx;        // winning group of 8 compacted node positions per object
    unsigned long long *timing;   // optional per-CTA cycle counters (16 per CTA); NULL in production
};

// The 8 features of one thread's A fragment for one row block: rows r and r+8 of the block, k = 2q, 2q+1, 2q+8, 2q+9.
struct AFeat { float2 v[4]; };   // (row r, k 2q) (row r+8, k 2q) (row r, k 2q+8) (row r+8, k 2q+8)

__device__ __forceinline__ AFeat load_afeat(const float *fobj, uint64_t n, uint64_t row, uint32_t q) {
    AFeat f;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const uint64_t r = row + 8 * (i & 1);
        f.v[i] = r < n ? __ldg(reinterpret_cast<const float2 *>(fobj + r * 16 + 2 * q + 8 * (i >> 1))) : make_float2(0.f, 0.f);
    }
    return f;
}

// running (best value, best group) of one row over the two columns per group this thread holds in a tile
template <int NT>
__device__ __forceinline__ void reduce_tile(float (&d)[NT / 2], uint32_t t, uint32_t q, uint32_t n_live, float (&best)[2], uint32_t (&bgroup)[2]) {
    const uint32_t col_base = t * NT;
    if (col_base + NT > n_live) {   // warp-uniform: only the padded tail of the last tile
#pragma unroll
        for (int i = 0; i < NT / 2; i++)
            if (col_base + 8 * (i >> 2) + 2 * q + (i & 1) >= n_live) d[i] = -INFINITY;
    }
#pragma unroll
    for (int gi = 0; gi < NT / 8; gi++) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const float v = fmaxf(d[4 * gi + 2 * h], d[4 * gi + 2 * h + 1]);
            if (v > best[h]) { best[h] = v; bgroup[h] = (col_base >> 3) + gi; }
        }
    }
}

// six bf16 cross terms of one node tile into accumulator d, in increasing magnitude: hl, lh, mm, hm, mh, hh
template <int NT>
__device__ __forceinline__ void issue_tile(float (&d)[NT / 2], const uint32_t (&a)[3][4], uint32_t sb, uint32_t b_block_bytes, uint32_t t, uint32_t m_pad) {
    constexpr int ta[6] = {0, 2, 1, 0, 1, 0}, tb[6] = {2, 0, 1, 1, 0, 0};   // 0 = h, 1 = m, 2 = l
    wgmma_fence();
#pragma unroll
    for (int i = 0; i < 6; i++)
        wgmma_bf16<NT>(d, a[ta[i]], make_desc(sb + tb[i] * b_block_bytes + t * NT * 16, m_pad * 16, 128), i > 0 ? 1u : 0u);
    wgmma_commit();
}

template <int NT>
__global__ void __launch_bounds__(kWgThreads, 1) k_affinity_wgmma(WgmmaParams P) {
    extern __shared__ __align__(128) unsigned char smem[];
    unsigned char *sB = smem;                                      // 3 blocks of m_pad*32 bytes
    const uint32_t b_block_bytes = P.m_pad * 32;
    const long long t_begin = P.timing ? clock64() : 0;

    // ---- one-time setup: node operands, resident for the whole kernel ------------------------------------------
    for (uint32_t p = threadIdx.x; p < P.m_pad; p += blockDim.x) {
        float f[16];
        const float4 *row = reinterpret_cast<const float4 *>(P.fnode_c + (size_t)p * 16);
#pragma unroll
        for (int q = 0; q < 4; q++) { const float4 v = __ldg(row + q); f[4 * q] = v.x; f[4 * q + 1] = v.y; f[4 * q + 2] = v.z; f[4 * q + 3] = v.w; }
        store_row_split(sB, b_block_bytes, P.m_pad * 16, p, f);
    }
    fence_proxy_async();             // generic-proxy stores -> visible to the tensor core (async proxy)
    __syncthreads();
    const long long t_setup = P.timing ? clock64() : 0;

    const uint32_t wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const uint32_t q = lane & 3, r_in = warp * 16 + (lane >> 2);   // row of this thread inside the row block (and r_in + 8)
    const uint32_t n_tiles = P.m_pad / NT;
    const uint64_t n_rb = (P.n + kRows - 1) / kRows, rb_step = (uint64_t)gridDim.x * kWarpgroups;
    const uint32_t sb = smem_u32(sB);

    uint64_t rb = (uint64_t)blockIdx.x * kWarpgroups + wg;
    AFeat next = load_afeat(P.fobj, P.n, rb * kRows + r_in, q);
    for (; rb < n_rb; rb += rb_step) {
        const AFeat cur = next;
        next = load_afeat(P.fobj, P.n, (rb + rb_step) * kRows + r_in, q);   // rows beyond n load nothing
        uint32_t a[3][4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            __nv_bfloat16 h0, m0, l0, h1, m1, l1;
            split3(cur.v[i].x, h0, m0, l0);
            split3(cur.v[i].y, h1, m1, l1);
            a[0][i] = pack2(h0, h1); a[1][i] = pack2(m0, m1); a[2][i] = pack2(l0, l1);
        }
        float best[2] = {-INFINITY, -INFINITY};
        uint32_t bgroup[2] = {0, 0};
        float acc[NT / 2];
        for (uint32_t t = 0; t < n_tiles; t++) {
            issue_tile<NT>(acc, a, sb, b_block_bytes, t, P.m_pad);
            wgmma_wait<0>();
            fence_regs(acc);
            reduce_tile<NT>(acc, t, q, P.n_live, best, bgroup);
        }
        // the four lanes of a row hold disjoint columns of every group: the largest value wins, on equal values the
        // smaller group index (the earlier column), as a single sequential scan over the columns would pick
#pragma unroll
        for (int h = 0; h < 2; h++) {
#pragma unroll
            for (int d = 1; d <= 2; d <<= 1) {
                const float ob = __shfl_xor_sync(0xFFFFFFFFu, best[h], d);
                const uint32_t og = __shfl_xor_sync(0xFFFFFFFFu, bgroup[h], d);
                if (ob > best[h] || (ob == best[h] && og < bgroup[h])) { best[h] = ob; bgroup[h] = og; }
            }
            const uint64_t row = rb * kRows + r_in + 8 * h;
            if (q == 0 && row < P.n) P.out_idx[row] = bgroup[h];
        }
    }
    if (P.timing && threadIdx.x == 0) { P.timing[blockIdx.x * 16 + 8] = t_setup - t_begin; P.timing[blockIdx.x * 16 + 9] = clock64() - t_begin; P.timing[blockIdx.x * 16 + 10] = t_begin; }
}

// Second pass: the 8 candidates of each object's winning group, re-evaluated in fp32 with the summation order of
// k_assign_affinity (fmaf over k = 0..15).  EIGHT lanes per object, four objects per warp trip: lane 8q + r scores
// candidate r of object q.  `fnode_g` is the node features regrouped on the host as [group][16-byte piece k][candidate r],
// so the k-th load of the eight lanes of an object is one 128-byte line (4 lines per object, like the contiguous rows),
// and the object's own row is a broadcast inside the 8 lanes.  Three xor-shuffle steps pick the smallest
// (cost, position).  The earlier one-warp-per-object version issued 50 warp instructions per object and was
// issue-bound; this one issues ~16.
// in/out: idx[row] holds the group on entry, the interned node index on exit.
__global__ void __launch_bounds__(256)
k_affinity_resolve(const float *__restrict__ fobj, uint64_t n, const float *__restrict__ fnode_g, const uint32_t *__restrict__ nidx_map, uint32_t n_live,
                   uint32_t *__restrict__ idx, float *__restrict__ out_cost, uint32_t *__restrict__ counters, uint32_t hist_bins) {
    extern __shared__ uint32_t shist[];
    for (uint32_t j = threadIdx.x; j < hist_bins; j += blockDim.x) shist[j] = 0;
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31, q = lane >> 3, r = lane & 7;
    const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const float4 *fobj4 = reinterpret_cast<const float4 *>(fobj);
    const float4 *fnode4 = reinterpret_cast<const float4 *>(fnode_g) + r;     // piece k of candidate r of group g: + (4*g + k) * 8
    // Software pipeline, one trip ahead: the group index and the object's row of the NEXT trip are in flight (HBM latency)
    // while the current trip reads its candidates (L1/L2 hits) and reduces; without it a warp has one dependent chain
    // idx -> node rows -> dot product in flight and the kernel is latency bound.
    uint64_t base = warp0 * 4;
    bool mine = base + q < n;
    uint64_t row = mine ? base + q : n - 1;                                     // clamp: the tail recomputes the last object
    uint32_t g = 0;
    float4 o[4] = {};
    if (base < n) {
        g = __ldg(idx + row);
#pragma unroll
        for (int k = 0; k < 4; k++) o[k] = __ldg(fobj4 + row * 4 + k);
    }
    for (; base < n; base += nwarps * 4) {
        const uint64_t nbase = base + nwarps * 4;
        const bool nmine = nbase + q < n;
        const uint64_t nrow = nmine ? nbase + q : n - 1;
        uint32_t ng = 0;
        float4 no[4] = {};
        if (nbase < n) {                                                        // warp-uniform
            ng = __ldg(idx + nrow);     // safe to read ahead: idx[nrow] is rewritten only by the trip that owns nrow (this warp, later)
#pragma unroll
            for (int k = 0; k < 4; k++) no[k] = __ldg(fobj4 + nrow * 4 + k);
        }
        const float4 *fn = fnode4 + (size_t)g * 32;
        float a = 0.f;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const float4 x = __ldg(fn + k * 8);                                 // rows beyond n_live are zero padding
            a = fmaf(o[k].x, x.x, a); a = fmaf(o[k].y, x.y, a); a = fmaf(o[k].z, x.z, a); a = fmaf(o[k].w, x.w, a);
        }
        // order-preserving integer image of cost = -dot (+inf for padding); minimum of (key, position) over the 8 lanes
        uint32_t p = g * 8 + r;
        const uint32_t bits = p < n_live ? __float_as_uint(-a) : 0x7F800000u;
        int key = (int)(bits ^ ((uint32_t)((int)bits >> 31) & 0x7FFFFFFFu));
        if (p >= n_live) p = kNone;
#pragma unroll
        for (int d = 4; d >= 1; d >>= 1) {
            const int ok = __shfl_xor_sync(0xFFFFFFFFu, key, d);
            const uint32_t op = __shfl_xor_sync(0xFFFFFFFFu, p, d);
            if (ok < key || (ok == key && op < p)) { key = ok; p = op; }
        }
        if (r == 0 && mine) {
            const uint32_t nid = p == kNone ? kNone : __ldg(nidx_map + p);
            idx[row] = nid;
            if (out_cost) {
                const uint32_t kb = (uint32_t)key;
                out_cost[row] = p == kNone ? 0.f : __uint_as_float(kb ^ ((uint32_t)((int)kb >> 31) & 0x7FFFFFFFu));   // the image is an involution
            }
            if (nid != kNone) {
                if (hist_bins) atomicAdd(&shist[nid], 1u);
                else if (counters) atomicAdd(&counters[nid], 1u);
            }
        }
        mine = nmine; row = nrow; g = ng;
#pragma unroll
        for (int k = 0; k < 4; k++) o[k] = no[k];
    }
    if (hist_bins) {
        __syncthreads();
        if (counters)
            for (uint32_t j = threadIdx.x; j < hist_bins; j += blockDim.x) { const uint32_t v = shist[j]; if (v) atomicAdd(&counters[j], v); }
    }
}

// ---- ranked lists (DESIGN.md 3.9) ------------------------------------------------------------------------------------------------
// A row's list of RT (value, group) pairs, ordered by larger value, then smaller group; empty slots are (-inf, kNone).
__device__ __forceinline__ bool group_before(float v, uint32_t g, float w, uint32_t h) { return v > w || (v == w && g < h); }

// (v, g) into a list it beats at the last slot, behind every entry of equal value: the groups of a scan come in increasing order,
// so this keeps "larger value, then smaller group", and with RT = 1 it is reduce_tile's update
template <int RT>
__device__ __forceinline__ void insert_scan(float (&lv)[RT], uint32_t (&lg)[RT], float v, uint32_t g) {
#pragma unroll
    for (int i = RT - 1; i > 0; i--) {
        if (v > lv[i - 1]) { lv[i] = lv[i - 1]; lg[i] = lg[i - 1]; }
        else if (v > lv[i]) { lv[i] = v; lg[i] = g; }
    }
    if (v > lv[0]) { lv[0] = v; lg[0] = g; }
}

// (v, g) from another lane's list: a group already present keeps the larger of its two values (a lane sees 2 of its 8 columns)
template <int RT>
__device__ __forceinline__ void insert_merge(float (&lv)[RT], uint32_t (&lg)[RT], float v, uint32_t g) {
    bool dup = false;
#pragma unroll
    for (int i = 0; i < RT; i++)
        if (lg[i] == g) { dup = true; lv[i] = fmaxf(lv[i], v); }
    if (!dup && group_before(v, g, lv[RT - 1], lg[RT - 1])) { lv[RT - 1] = v; lg[RT - 1] = g; }
#pragma unroll
    for (int i = RT - 1; i > 0; i--)   // one entry is out of place at most: one bubble pass upwards restores the order
        if (group_before(lv[i], lg[i], lv[i - 1], lg[i - 1])) {
            const float tv = lv[i]; lv[i] = lv[i - 1]; lv[i - 1] = tv;
            const uint32_t tg = lg[i]; lg[i] = lg[i - 1]; lg[i - 1] = tg;
        }
}

// reduce_tile with a list of the best RT groups per row instead of the best one
template <int NT, int RT>
__device__ __forceinline__ void reduce_tile_ranked(float (&d)[NT / 2], uint32_t t, uint32_t q, uint32_t n_live, float (&lv)[2][RT], uint32_t (&lg)[2][RT]) {
    const uint32_t col_base = t * NT;
    if (col_base + NT > n_live) {
#pragma unroll
        for (int i = 0; i < NT / 2; i++)
            if (col_base + 8 * (i >> 2) + 2 * q + (i & 1) >= n_live) d[i] = -INFINITY;
    }
#pragma unroll
    for (int gi = 0; gi < NT / 8; gi++) {
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const float v = fmaxf(d[4 * gi + 2 * h], d[4 * gi + 2 * h + 1]);
            if (v > lv[h][RT - 1]) insert_scan<RT>(lv[h], lg[h], v, (col_base >> 3) + gi);
        }
    }
}

// k_affinity_wgmma keeping each row's best RT distinct groups of 8 columns (a group's value: its largest column) in
// out_groups[row * RT ..], kNone past the groups that hold live nodes.  Node staging, the A fragments and the six-term tiles are
// k_affinity_wgmma's, so the accumulators are bit for bit the same and the first group is the one that kernel writes.  Each lane
// keeps its own best RT over the 2 columns per group it holds; a group of the row's best RT has its value in some lane, and fewer
// than RT groups beat it there, so merging the four lane lists (a butterfly over xor 1 and 2) finds the row's best RT.
// WG warpgroups per CTA: the lists cost 4 RT registers per thread beside the 64 of the accumulator.
template <int NT, int RT, int WG>
__global__ void __launch_bounds__(128 * WG, 1) k_affinity_wgmma_ranked(WgmmaParams P) {
    extern __shared__ __align__(128) unsigned char smem[];
    unsigned char *sB = smem;
    const uint32_t b_block_bytes = P.m_pad * 32;
    for (uint32_t p = threadIdx.x; p < P.m_pad; p += blockDim.x) {
        float f[16];
        const float4 *row = reinterpret_cast<const float4 *>(P.fnode_c + (size_t)p * 16);
#pragma unroll
        for (int q = 0; q < 4; q++) { const float4 v = __ldg(row + q); f[4 * q] = v.x; f[4 * q + 1] = v.y; f[4 * q + 2] = v.z; f[4 * q + 3] = v.w; }
        store_row_split(sB, b_block_bytes, P.m_pad * 16, p, f);
    }
    fence_proxy_async();
    __syncthreads();

    const uint32_t wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const uint32_t q = lane & 3, r_in = warp * 16 + (lane >> 2);
    const uint32_t n_tiles = P.m_pad / NT;
    const uint64_t n_rb = (P.n + kRows - 1) / kRows, rb_step = (uint64_t)gridDim.x * WG;
    const uint32_t sb = smem_u32(sB);

    uint64_t rb = (uint64_t)blockIdx.x * WG + wg;
    AFeat next = load_afeat(P.fobj, P.n, rb * kRows + r_in, q);
    for (; rb < n_rb; rb += rb_step) {
        const AFeat cur = next;
        next = load_afeat(P.fobj, P.n, (rb + rb_step) * kRows + r_in, q);
        uint32_t a[3][4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            __nv_bfloat16 h0, m0, l0, h1, m1, l1;
            split3(cur.v[i].x, h0, m0, l0);
            split3(cur.v[i].y, h1, m1, l1);
            a[0][i] = pack2(h0, h1); a[1][i] = pack2(m0, m1); a[2][i] = pack2(l0, l1);
        }
        float lv[2][RT];
        uint32_t lg[2][RT];
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int i = 0; i < RT; i++) { lv[h][i] = -INFINITY; lg[h][i] = kNone; }
        float acc[NT / 2];
        for (uint32_t t = 0; t < n_tiles; t++) {
            issue_tile<NT>(acc, a, sb, b_block_bytes, t, P.m_pad);
            wgmma_wait<0>();
            fence_regs(acc);
            reduce_tile_ranked<NT, RT>(acc, t, q, P.n_live, lv, lg);
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {
#pragma unroll
            for (int d = 1; d <= 2; d <<= 1) {
                float ov[RT];
                uint32_t og[RT];
#pragma unroll
                for (int i = 0; i < RT; i++) { ov[i] = __shfl_xor_sync(0xFFFFFFFFu, lv[h][i], d); og[i] = __shfl_xor_sync(0xFFFFFFFFu, lg[h][i], d); }
#pragma unroll
                for (int i = 0; i < RT; i++) insert_merge<RT>(lv[h], lg[h], ov[i], og[i]);
            }
            const uint64_t row = rb * kRows + r_in + 8 * h;
            if (q == 0 && row < P.n) {
#pragma unroll
                for (int i = 0; i < RT; i++) P.out_idx[row * RT + i] = lg[h][i];
            }
        }
    }
}

// k_affinity_resolve over the RT groups of each object: lane 8q + r scores candidate r of every group of object q, with the same
// fmaf order.  Rank 1 is the smallest (cost, position) of the first group, exactly as k_affinity_resolve picks it; ranks 2.. are
// the smallest remaining (cost, position) over all 8 RT candidates.  Positions are compacted in node-index order, so this is
// (cost, node index) order.  Each lane of an object holds one group index (lane r: group r), read by the others with a shuffle.
// Launch bounds: without a minimum, ptxas keeps RT = 2 and 4 at 64 registers and spills; a minimum of 2 blocks spills RT = 8, which
// fits in 91 registers without one (ptxas -v).
template <int RT>
__global__ void __launch_bounds__(256, RT <= 4 ? 2 : 0)
k_affinity_resolve_ranked(const float *__restrict__ fobj, uint64_t n, const float *__restrict__ fnode_g, const uint32_t *__restrict__ nidx_map, uint32_t n_live,
                          const uint32_t *__restrict__ groups, uint32_t ranks, uint32_t *__restrict__ out) {
    const uint32_t lane = threadIdx.x & 31, q = lane >> 3, r = lane & 7, seg = lane & ~7u;
    const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const float4 *fobj4 = reinterpret_cast<const float4 *>(fobj);
    const float4 *fnode4 = reinterpret_cast<const float4 *>(fnode_g) + r;
    // one trip ahead, as in k_affinity_resolve: the groups and the row of the next trip are in flight while this trip scores
    uint64_t base = warp0 * 4;
    bool mine = base + q < n;
    uint64_t row = mine ? base + q : n - 1;
    uint32_t g = kNone;
    float4 o[4] = {};
    if (base < n) {
        if (r < RT) g = __ldg(groups + row * RT + r);
#pragma unroll
        for (int k = 0; k < 4; k++) o[k] = __ldg(fobj4 + row * 4 + k);
    }
    for (; base < n; base += nwarps * 4) {
        const uint64_t nbase = base + nwarps * 4;
        const bool nmine = nbase + q < n;
        const uint64_t nrow = nmine ? nbase + q : n - 1;
        uint32_t ng = kNone;
        float4 no[4] = {};
        if (nbase < n) {
            if (r < RT) ng = __ldg(groups + nrow * RT + r);
#pragma unroll
            for (int k = 0; k < 4; k++) no[k] = __ldg(fobj4 + nrow * 4 + k);
        }
        int key[RT];
        uint32_t pos[RT];
#pragma unroll
        for (int j = 0; j < RT; j++) {
            const uint32_t gj = __shfl_sync(0xFFFFFFFFu, g, seg | j);
            const float4 *fn = fnode4 + (size_t)(gj == kNone ? 0u : gj) * 32;
            float a = 0.f;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const float4 x = __ldg(fn + k * 8);
                a = fmaf(o[k].x, x.x, a); a = fmaf(o[k].y, x.y, a); a = fmaf(o[k].z, x.z, a); a = fmaf(o[k].w, x.w, a);
            }
            uint32_t p = gj * 8 + r;
            const bool live = gj != kNone && p < n_live;
            const uint32_t bits = live ? __float_as_uint(-a) : 0x7F800000u;
            key[j] = (int)(bits ^ ((uint32_t)((int)bits >> 31) & 0x7FFFFFFFu));
            pos[j] = live ? p : kNone;
        }
        for (uint32_t rank = 0; rank < ranks; rank++) {   // warp-uniform
            int k = key[0];
            uint32_t p = pos[0];
            if (rank) {
#pragma unroll
                for (int j = 1; j < RT; j++)
                    if (key[j] < k || (key[j] == k && pos[j] < p)) { k = key[j]; p = pos[j]; }
            }
#pragma unroll
            for (int d = 4; d >= 1; d >>= 1) {
                const int ok = __shfl_xor_sync(0xFFFFFFFFu, k, d);
                const uint32_t op = __shfl_xor_sync(0xFFFFFFFFu, p, d);
                if (ok < k || (ok == k && op < p)) { k = ok; p = op; }
            }
            if (r == 0 && mine) out[row * ranks + rank] = p == kNone ? kNone : __ldg(nidx_map + p);
            if (p != kNone) {
#pragma unroll
                for (int j = 0; j < RT; j++)
                    if (pos[j] == p) { key[j] = 0x7F800000; pos[j] = kNone; }
            }
        }
        mine = nmine; row = nrow; g = ng;
#pragma unroll
        for (int k = 0; k < 4; k++) o[k] = no[k];
    }
}

// ---- failure-domain lists (DESIGN.md 3.14) ----------------------------------------------------------------------------------------
// A row's list of RT columns (value, position, domain), one per domain, ordered by larger value, then smaller position; empty slots
// are (-inf, kNone, kNone).
__device__ __forceinline__ bool col_before(float v, uint32_t p, float w, uint32_t q) { return v > w || (v == w && p < q); }

// Domain-aware insert (the rule of spread_insert, DESIGN.md 3.12) of a column the caller found before the last entry: a listed column
// of the same domain that comes before it drops it; otherwise it goes in place and the shift stops at the entry of its own domain.
template <int RT>
__device__ __forceinline__ void insert_dom(float (&lv)[RT], uint32_t (&lp)[RT], uint32_t (&ld)[RT], float v, uint32_t p, uint32_t d) {
    bool keep = true;
#pragma unroll
    for (int i = 0; i < RT; i++) keep &= !(ld[i] == d && col_before(lv[i], lp[i], v, p));
    if (!keep) return;
    const uint32_t dc = d;
    bool go = true;
#pragma unroll
    for (int i = 0; i < RT; i++) {
        const bool sw = go && col_before(v, p, lv[i], lp[i]);
        const float tv = lv[i];
        const uint32_t tp = lp[i], td = ld[i];
        lv[i] = sw ? v : tv; lp[i] = sw ? p : tp; ld[i] = sw ? d : td;
        v = sw ? tv : v; p = sw ? tp : p; d = sw ? td : d;
        go = go && !(sw && td == dc);
    }
}

// k_affinity_wgmma_ranked keeping, per row, the best RT domain representatives among the COLUMNS (not groups) in
// out_idx[row * RT ..], kNone past the live domains.  Node staging, the A fragments and the six-term tiles are k_affinity_wgmma's, so
// the accumulators are the same bits.  A lane scans its columns in increasing position, so `v > last value` is an exact gate, and the
// domain id is read (read-only path) on the insert path only.  The four lane lists of a row merge with the same insert (xor 1, 2).
// The first entry is the row's largest value at its smallest position, so its group is the one k_affinity_wgmma picks.
template <int NT, int RT, int WG>
__global__ void __launch_bounds__(128 * WG, 1) k_affinity_wgmma_spread(WgmmaParams P, const uint32_t *__restrict__ pdom) {
    extern __shared__ __align__(128) unsigned char smem[];
    unsigned char *sB = smem;
    const uint32_t b_block_bytes = P.m_pad * 32;
    for (uint32_t p = threadIdx.x; p < P.m_pad; p += blockDim.x) {
        float f[16];
        const float4 *row = reinterpret_cast<const float4 *>(P.fnode_c + (size_t)p * 16);
#pragma unroll
        for (int q = 0; q < 4; q++) { const float4 v = __ldg(row + q); f[4 * q] = v.x; f[4 * q + 1] = v.y; f[4 * q + 2] = v.z; f[4 * q + 3] = v.w; }
        store_row_split(sB, b_block_bytes, P.m_pad * 16, p, f);
    }
    fence_proxy_async();
    __syncthreads();

    const uint32_t wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const uint32_t q = lane & 3, r_in = warp * 16 + (lane >> 2);
    const uint32_t n_tiles = P.m_pad / NT;
    const uint64_t n_rb = (P.n + kRows - 1) / kRows, rb_step = (uint64_t)gridDim.x * WG;
    const uint32_t sb = smem_u32(sB);

    uint64_t rb = (uint64_t)blockIdx.x * WG + wg;
    AFeat next = load_afeat(P.fobj, P.n, rb * kRows + r_in, q);
    for (; rb < n_rb; rb += rb_step) {
        const AFeat cur = next;
        next = load_afeat(P.fobj, P.n, (rb + rb_step) * kRows + r_in, q);
        uint32_t a[3][4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
            __nv_bfloat16 h0, m0, l0, h1, m1, l1;
            split3(cur.v[i].x, h0, m0, l0);
            split3(cur.v[i].y, h1, m1, l1);
            a[0][i] = pack2(h0, h1); a[1][i] = pack2(m0, m1); a[2][i] = pack2(l0, l1);
        }
        float lv[2][RT];
        uint32_t lp[2][RT], ld[2][RT];
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
            for (int i = 0; i < RT; i++) { lv[h][i] = -INFINITY; lp[h][i] = kNone; ld[h][i] = kNone; }
        float acc[NT / 2];
        for (uint32_t t = 0; t < n_tiles; t++) {
            issue_tile<NT>(acc, a, sb, b_block_bytes, t, P.m_pad);
            wgmma_wait<0>();
            fence_regs(acc);
            const uint32_t col_base = t * NT;
            if (col_base + NT > P.n_live) {   // warp-uniform: only the padded tail of the last tile
#pragma unroll
                for (int i = 0; i < NT / 2; i++)
                    if (col_base + 8 * (i >> 2) + 2 * q + (i & 1) >= P.n_live) acc[i] = -INFINITY;
            }
#pragma unroll
            for (int i = 0; i < NT / 2; i++) {   // increasing column within each row h = (i >> 1) & 1
                const int h = (i >> 1) & 1;
                const uint32_t col = col_base + 8 * (i >> 2) + 2 * q + (i & 1);
                if (acc[i] > lv[h][RT - 1]) insert_dom<RT>(lv[h], lp[h], ld[h], acc[i], col, __ldg(pdom + col));
            }
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {
#pragma unroll
            for (int d = 1; d <= 2; d <<= 1) {
                float ov[RT];
                uint32_t op[RT], od[RT];
#pragma unroll
                for (int i = 0; i < RT; i++) {
                    ov[i] = __shfl_xor_sync(0xFFFFFFFFu, lv[h][i], d);
                    op[i] = __shfl_xor_sync(0xFFFFFFFFu, lp[h][i], d);
                    od[i] = __shfl_xor_sync(0xFFFFFFFFu, ld[h][i], d);
                }
#pragma unroll
                for (int i = 0; i < RT; i++)
                    if (col_before(ov[i], op[i], lv[h][RT - 1], lp[h][RT - 1])) insert_dom<RT>(lv[h], lp[h], ld[h], ov[i], op[i], od[i]);
            }
            const uint64_t row = rb * kRows + r_in + 8 * h;
            if (q == 0 && row < P.n) {
#pragma unroll
                for (int i = 0; i < RT; i++) P.out_idx[row * RT + i] = lp[h][i];
            }
        }
    }
}

// Second pass of the failure-domain lists: eight lanes per object, as in k_affinity_resolve_ranked.  Lane r re-costs column r of the
// first entry's group and candidate r, both with k_affinity_resolve's fmaf order.  Rank 1 is the smallest (cost, position) of that
// group, exactly as k_affinity_resolve picks it; ranks 2.. are the smallest remaining (cost, position) among the candidates whose
// domain is not listed yet, and each pick masks every candidate of its domain (rank 1's included).
template <int RT>
__global__ void __launch_bounds__(256, 2)
k_affinity_resolve_spread(const float *__restrict__ fobj, uint64_t n, const float *__restrict__ fnode_g, const uint32_t *__restrict__ nidx_map,
                          const uint32_t *__restrict__ pdom, uint32_t n_live, const uint32_t *__restrict__ cols, uint32_t ranks, uint32_t *__restrict__ out) {
    const uint32_t lane = threadIdx.x & 31, r = lane & 7, seg = lane & ~7u;
    const uint32_t q = lane >> 3;
    const uint64_t warp0 = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const float4 *fobj4 = reinterpret_cast<const float4 *>(fobj);
    const float4 *fnode4 = reinterpret_cast<const float4 *>(fnode_g);   // piece k of position p: + ((p >> 3) * 4 + k) * 8 + (p & 7)
    auto cost_key = [&](const float4 (&o)[4], uint32_t p) {
        const float4 *fn = fnode4 + (size_t)(p >> 3) * 32 + (p & 7);
        float a = 0.f;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const float4 x = __ldg(fn + k * 8);
            a = fmaf(o[k].x, x.x, a); a = fmaf(o[k].y, x.y, a); a = fmaf(o[k].z, x.z, a); a = fmaf(o[k].w, x.w, a);
        }
        const uint32_t bits = __float_as_uint(-a);
        return (int)(bits ^ ((uint32_t)((int)bits >> 31) & 0x7FFFFFFFu));
    };
    // smallest (key, position) over the 8 lanes of an object, its domain carried along
    auto seg_min = [](int &k, uint32_t &p, uint32_t &dm) {
#pragma unroll
        for (int d = 4; d >= 1; d >>= 1) {
            const int ok = __shfl_xor_sync(0xFFFFFFFFu, k, d);
            const uint32_t op = __shfl_xor_sync(0xFFFFFFFFu, p, d), od = __shfl_xor_sync(0xFFFFFFFFu, dm, d);
            if (ok < k || (ok == k && op < p)) { k = ok; p = op; dm = od; }
        }
    };
    // one trip ahead, as in k_affinity_resolve: the candidates and the row of the next trip are in flight while this trip scores
    uint64_t base = warp0 * 4;
    bool mine = base + q < n;
    uint64_t row = mine ? base + q : n - 1;
    uint32_t c = kNone;
    float4 o[4] = {};
    if (base < n) {
        if (r < RT) c = __ldg(cols + row * RT + r);
#pragma unroll
        for (int k = 0; k < 4; k++) o[k] = __ldg(fobj4 + row * 4 + k);
    }
    for (; base < n; base += nwarps * 4) {
        const uint64_t nbase = base + nwarps * 4;
        const bool nmine = nbase + q < n;
        const uint64_t nrow = nmine ? nbase + q : n - 1;
        uint32_t nc = kNone;
        float4 no[4] = {};
        if (nbase < n) {
            if (r < RT) nc = __ldg(cols + nrow * RT + r);
#pragma unroll
            for (int k = 0; k < 4; k++) no[k] = __ldg(fobj4 + nrow * 4 + k);
        }
        // rank 1: column r of the first entry's group (group 0 when no column was listed, as k_affinity_wgmma's initial group)
        const uint32_t c0 = __shfl_sync(0xFFFFFFFFu, c, seg);
        uint32_t p1 = (c0 == kNone ? 0u : c0 >> 3) * 8 + r;
        int k1 = cost_key(o, p1);
        if (p1 >= n_live) { k1 = 0x7F800000; p1 = kNone; }
        uint32_t d1 = 0;
        seg_min(k1, p1, d1);
        d1 = __ldg(pdom + p1);   // p1 < n_live: the group holds the listed column, or is group 0
        // candidate r: its domain masked out once listed
        int kc = 0x7F800000;
        uint32_t pc = kNone, dc = kNone;
        if (c != kNone) { kc = cost_key(o, c); pc = c; dc = __ldg(pdom + c); }
        if (r == 0 && mine) out[row * ranks] = __ldg(nidx_map + p1);
        uint32_t dl = d1;
        for (uint32_t rank = 1; rank < ranks; rank++) {   // warp-uniform
            if (dc == dl) { kc = 0x7F800000; pc = kNone; dc = kNone; }
            int k = kc;
            uint32_t p = pc, dm = dc;
            seg_min(k, p, dm);
            if (r == 0 && mine) out[row * ranks + rank] = p == kNone ? kNone : __ldg(nidx_map + p);
            dl = dm;   // kNone once nothing is left: it masks only empty slots
        }
        mine = nmine; row = nrow; c = nc;
#pragma unroll
        for (int k = 0; k < 4; k++) o[k] = no[k];
    }
}

}  // namespace

// development hook: device buffer of 16 u64 per CTA that receives the tensor-core kernel's setup and total cycle counts
static unsigned long long *g_umma_timing = nullptr;
void affinity_umma_set_timing_buffer(unsigned long long *d) { g_umma_timing = d; }

// Largest padded live-node count whose operands (96 B per node) fit in the 227 KB of shared memory of a block.
uint32_t affinity_umma_max_nodes() { return ((227u * 1024u) / 96u) / 256u * 256u; }

cudaError_t launch_assign_affinity_umma(const Launch &L, const float *d_fobj, uint64_t n, const float *d_fnode_c, const float *d_fnode_g, const uint32_t *d_nidx_map,
                                        uint32_t n_live, uint32_t m_pad, uint32_t n_total, uint32_t *d_out_idx, float *d_out_cost, uint32_t *d_counters) {
    if (!n) return cudaSuccess;
    const bool small = m_pad <= 64;
    if (!n_live || (small && m_pad != 64) || (!small && (m_pad % 256)) || m_pad > affinity_umma_max_nodes()) return cudaErrorInvalidValue;
    const size_t smem = (size_t)3 * m_pad * 32;
    WgmmaParams P{d_fobj, n, d_fnode_c, n_live, m_pad, d_out_idx, g_umma_timing};
    const uint64_t n_rb = (n + kRows - 1) / kRows, n_cta = (n_rb + kWarpgroups - 1) / kWarpgroups;
    const int grid = (int)(n_cta < (uint64_t)L.sm_count ? n_cta : (uint64_t)L.sm_count);
    cudaError_t err;
    if (small) {
        err = cudaFuncSetAttribute(k_affinity_wgmma<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (err == cudaSuccess) k_affinity_wgmma<64><<<grid, kWgThreads, smem, L.stream>>>(P);
    } else {
        err = cudaFuncSetAttribute(k_affinity_wgmma<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (err == cudaSuccess) k_affinity_wgmma<128><<<grid, kWgThreads, smem, L.stream>>>(P);
    }
    // a tensor-core launch that did not happen is an error for the caller, never a silent switch to the CUDA-core kernel
    if (err == cudaSuccess) err = cudaGetLastError();
    if (err != cudaSuccess) return err;
    RIO_COUNT_LAUNCH(L);
    {
        const uint32_t bins = (d_counters && n_total <= 8192) ? n_total : 0;
        const uint64_t blocks = (n + 31) / 32, cap = (uint64_t)L.sm_count * 8;   // 4 objects per warp trip, 8 warps per CTA
        k_affinity_resolve<<<(int)(blocks < cap ? blocks : cap), 256, (size_t)bins * 4, L.stream>>>(d_fobj, n, d_fnode_g, d_nidx_map, n_live, d_out_idx, d_out_cost, d_counters,
                                                                                          bins);
        RIO_COUNT_LAUNCH(L);
    }
    return cudaGetLastError();
}

namespace {

// warpgroups per CTA of k_affinity_wgmma_ranked<NT, RT>: four where the lists fit in 128 registers without spills (ptxas -v)
constexpr int ranked_warpgroups(int NT, int RT) { return RT <= 4 ? 4 : 2; }

template <int NT, int RT>
cudaError_t launch_wgmma_ranked(const Launch &L, const WgmmaParams &P, size_t smem) {
    constexpr int WG = ranked_warpgroups(NT, RT);
    const uint64_t n_rb = (P.n + kRows - 1) / kRows, n_cta = (n_rb + WG - 1) / WG;
    const int grid = (int)(n_cta < (uint64_t)L.sm_count ? n_cta : (uint64_t)L.sm_count);
    cudaError_t err = cudaFuncSetAttribute(k_affinity_wgmma_ranked<NT, RT, WG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err == cudaSuccess) k_affinity_wgmma_ranked<NT, RT, WG><<<grid, 128 * WG, smem, L.stream>>>(P);
    return err == cudaSuccess ? cudaGetLastError() : err;
}

template <int RT>
cudaError_t launch_ranked_pair(const Launch &L, const WgmmaParams &P, size_t smem, const float *d_fnode_g, const uint32_t *d_nidx_map, uint32_t ranks,
                               uint32_t *d_out_idx) {
    const cudaError_t err = P.m_pad <= 64 ? launch_wgmma_ranked<64, RT>(L, P, smem) : launch_wgmma_ranked<128, RT>(L, P, smem);
    if (err != cudaSuccess) return err;
    RIO_COUNT_LAUNCH(L);
    const uint64_t blocks = (P.n + 31) / 32, cap = (uint64_t)L.sm_count * 8;
    k_affinity_resolve_ranked<RT><<<(int)(blocks < cap ? blocks : cap), 256, 0, L.stream>>>(P.fobj, P.n, d_fnode_g, d_nidx_map, P.n_live, P.out_idx, ranks,
                                                                                           d_out_idx);
    RIO_COUNT_LAUNCH(L);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_assign_affinity_umma_ranked(const Launch &L, const float *d_fobj, uint64_t n, const float *d_fnode_c, const float *d_fnode_g,
                                               const uint32_t *d_nidx_map, uint32_t n_live, uint32_t m_pad, uint32_t ranks, uint32_t *d_groups,
                                               uint32_t *d_out_idx) {
    if (!n) return cudaSuccess;
    const bool small = m_pad <= 64;
    if (!n_live || (small && m_pad != 64) || (!small && (m_pad % 256)) || m_pad > affinity_umma_max_nodes() || ranks < 1 || ranks > kMaxRanks)
        return cudaErrorInvalidValue;
    const size_t smem = (size_t)3 * m_pad * 32;
    const WgmmaParams P{d_fobj, n, d_fnode_c, n_live, m_pad, d_groups, nullptr};
    switch (affinity_ranked_groups(ranks)) {
        case 1: return launch_ranked_pair<1>(L, P, smem, d_fnode_g, d_nidx_map, ranks, d_out_idx);
        case 2: return launch_ranked_pair<2>(L, P, smem, d_fnode_g, d_nidx_map, ranks, d_out_idx);
        case 4: return launch_ranked_pair<4>(L, P, smem, d_fnode_g, d_nidx_map, ranks, d_out_idx);
        default: return launch_ranked_pair<8>(L, P, smem, d_fnode_g, d_nidx_map, ranks, d_out_idx);
    }
}

namespace {

// warpgroups per CTA of k_affinity_wgmma_spread<NT, RT>: the lists cost 6 RT registers per thread; four warpgroups where they fit in
// 128 registers without spills (ptxas -v)
constexpr int spread_warpgroups(int RT) { return RT <= 4 ? 4 : 2; }

template <int NT, int RT>
cudaError_t launch_wgmma_spread(const Launch &L, const WgmmaParams &P, const uint32_t *d_pdom, size_t smem) {
    constexpr int WG = spread_warpgroups(RT);
    const uint64_t n_rb = (P.n + kRows - 1) / kRows, n_cta = (n_rb + WG - 1) / WG;
    const int grid = (int)(n_cta < (uint64_t)L.sm_count ? n_cta : (uint64_t)L.sm_count);
    cudaError_t err = cudaFuncSetAttribute(k_affinity_wgmma_spread<NT, RT, WG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (err == cudaSuccess) k_affinity_wgmma_spread<NT, RT, WG><<<grid, 128 * WG, smem, L.stream>>>(P, d_pdom);
    return err == cudaSuccess ? cudaGetLastError() : err;
}

template <int RT>
cudaError_t launch_spread_pair(const Launch &L, const WgmmaParams &P, const uint32_t *d_pdom, size_t smem, const float *d_fnode_g, const uint32_t *d_nidx_map,
                               uint32_t ranks, uint32_t *d_out_idx) {
    const cudaError_t err = P.m_pad <= 64 ? launch_wgmma_spread<64, RT>(L, P, d_pdom, smem) : launch_wgmma_spread<128, RT>(L, P, d_pdom, smem);
    if (err != cudaSuccess) return err;
    RIO_COUNT_LAUNCH(L);
    const uint64_t blocks = (P.n + 31) / 32, cap = (uint64_t)L.sm_count * 8;
    k_affinity_resolve_spread<RT><<<(int)(blocks < cap ? blocks : cap), 256, 0, L.stream>>>(P.fobj, P.n, d_fnode_g, d_nidx_map, d_pdom, P.n_live, P.out_idx,
                                                                                           ranks, d_out_idx);
    RIO_COUNT_LAUNCH(L);
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_assign_affinity_umma_spread(const Launch &L, const float *d_fobj, uint64_t n, const float *d_fnode_c, const float *d_fnode_g,
                                               const uint32_t *d_nidx_map, const uint32_t *d_pdom, uint32_t n_live, uint32_t m_pad, uint32_t ranks,
                                               uint32_t *d_cols, uint32_t *d_out_idx) {
    if (!n) return cudaSuccess;
    const bool small = m_pad <= 64;
    if (!n_live || (small && m_pad != 64) || (!small && (m_pad % 256)) || m_pad > affinity_umma_max_nodes() || ranks < 1 || ranks > kMaxRanks)
        return cudaErrorInvalidValue;
    const size_t smem = (size_t)3 * m_pad * 32;
    const WgmmaParams P{d_fobj, n, d_fnode_c, n_live, m_pad, d_cols, nullptr};
    switch (affinity_ranked_groups(ranks)) {
        case 1: return launch_spread_pair<1>(L, P, d_pdom, smem, d_fnode_g, d_nidx_map, ranks, d_out_idx);
        case 2: return launch_spread_pair<2>(L, P, d_pdom, smem, d_fnode_g, d_nidx_map, ranks, d_out_idx);
        case 4: return launch_spread_pair<4>(L, P, d_pdom, smem, d_fnode_g, d_nidx_map, ranks, d_out_idx);
        default: return launch_spread_pair<8>(L, P, d_pdom, smem, d_fnode_g, d_nidx_map, ranks, d_out_idx);
    }
}

}  // namespace rio

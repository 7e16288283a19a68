// kernels.cuh -- device data layouts and kernel launchers of librio_cuda (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

#include "buffer_align.cuh"

namespace rio {

// ---- node table as the assign kernels see it -----------------------------------------------------------
// Live nodes sorted by (inv_weight, node index): equal-weight nodes form a "class" in which the spec's
// lexicographic min of (E(u)*r, ~u, j) reduces to "largest u, lowest j" (E is monotone, DESIGN.md 3.4).
struct __align__(16) NodeRec {
    uint32_t s0;    // lo32(seed)
    uint32_t nidx;  // interned node index (what the directory stores)
    uint32_t s1;    // hi32(seed) | 1: the per-node odd multiplier of the second multiply-add
    uint32_t s2;    // lo32(mix64(seed ^ kSaltNode2))
};
struct ClassRec {
    uint32_t start;  // first record of the class in the sorted table
    uint32_t invw;   // floor((2^32-1)/w)
};
struct NodeTabDev {
    const NodeRec *recs;       // n_live records
    const ClassRec *classes;   // n_classes + 1 (sentinel: start = n_live)
    uint32_t n_live;
    uint32_t n_classes;
    uint32_t n_total;          // interned nodes (size of counter / by-index arrays)
    // by-interned-index arrays (n_total entries) for the kernels that gather by node index
    const uint4 *by_idx;       // {s0, invw (0 = not live), hi32(seed)|1, s2}
};

// ---- HRW2 table (DESIGN.md 3.8 / 4.1): one contiguous blob, staged into shared memory by ONE cp.async.bulk ---------
//   [0, 4 << bits)                 thresholds T3 of the trie nodes, heap order (index 1 = root; [0] unused)
//   [4 << bits, 8 << bits)         leaf words, one per bucket: node index | 0x80000000 + byte offset of the chain's first record | kNone (empty)
//   off_crec  (16-byte aligned)    chain records, 32 bytes each, k-1 for a bucket of k nodes: {s0, m2, h2, T3} (the member-keyed
//                                  contest) then {this node's index, next, 0, 0}; next = the last node's index, or 0x80000000 + byte
//                                  offset of the next record
struct TrieDev {
    const void *blob;
    uint32_t blob_bytes;   // multiple of 16
    uint32_t off_crec;     // chain records start here (32 bytes per chain member); leaf words hold byte offsets into the blob
    uint32_t bits;
    uint32_t n_chain;
    uint32_t top[8];       // copy of the thresholds at heap indices 1..7 (levels 0-2): read from the parameter bank by the dense kernel
};

// ---- directory: open addressing, 16-byte AoS slots ------------------------------------------------------
// key == kEmptyKey: free.  val = (seq << 32) | node; seq is non-zero only inside an upsert batch.
struct __align__(16) DirSlot {
    unsigned long long key;
    unsigned long long val;
};
constexpr unsigned long long kEmptyKey = 0xFFFFFFFFFFFFFFFFull;
constexpr unsigned long long kEmptyVal = 0x00000000FFFFFFFFull;  // seq 0, node NONE
struct DirDev {
    DirSlot *slots;
    uint64_t mask;      // capacity - 1
    uint32_t shift;     // 64 - log2(capacity)
};

struct Launch { cudaStream_t stream; int sm_count; uint64_t *launch_counter; int spare_ctas = 0; /* dense walk: leave this many CTA slots of the machine free */ };
// every launcher counts each kernel it launched (rio_cuda_launch_count)
#define RIO_COUNT_LAUNCH(L) do { if ((L).launch_counter) ++*(L).launch_counter; } while (0)

// ---- the tail of a bounded-load pass: counter exchange + capacity check (bounded_tail.cuh) ----------------------------------
struct XchgPeers { uint32_t *win[16]; };
struct BoundedTail {
    uint32_t enabled;          // 0: plain assignment, nothing below is read
    uint32_t M;                // interned nodes (length of every per-node array)
    uint32_t *ticket;          // CTA-done counter of the fused form (left at 0 by the last CTA)
    uint32_t *next_zero;       // nullable: counter buffer of the next pass, cleared by the check
    XchgPeers peers;           // world > 1: every rank's exchange window (CUDA IPC)
    uint32_t rank, world, max_nodes, xchg_epoch;
    uint32_t *glob;            // out: global counters
    const uint32_t *cap;       // capacity per node
    const uint8_t *state;      // kNodeLive per node
    uint32_t *closed_epoch;    // closed[j] <=> closed_epoch[j] == call_epoch (no memset between calls)
    uint32_t call_epoch;
    uint32_t *thr;             // out: spill thresholds
    uint8_t *over;             // out: over-capacity flags
    volatile uint32_t *host_flags;   // mapped pinned: {any over, open nodes, sequence number of this check}
    uint32_t flag_seq;
};

// solver
void launch_assign_hrw(const Launch &L, const uint64_t *d_keys, uint64_t n, const NodeTabDev &tab, uint32_t *d_out_idx,
                       uint32_t *d_counters /*nullable, n_total entries*/, const uint32_t *d_sel /*nullable*/, uint64_t n_sel);
uint64_t assign_wave_objects(int sm_count);
// HRW2 (k_trie.cu)
void trie_upload_level_constants(int device);
uint64_t trie_wave_objects(int sm_count);
void launch_assign_affinity(const Launch &L, const float *d_fobj, uint64_t n, const float *d_fnode /*n_total x K*/,
                            const uint32_t *d_live /*n_total flags*/, uint32_t n_total, uint32_t K, uint32_t *d_out_idx,
                            float *d_out_cost /*nullable*/, uint32_t *d_counters);
// tensor-core (wgmma) path for K == 16 (k_affinity_umma.cu).  The caller picks it when the padded live-node count is at most
// affinity_umma_max_nodes() (the CUDA-core kernel takes larger node sets); a shape it cannot take or a launch that fails is
// returned as an error.
uint32_t affinity_umma_max_nodes();
void affinity_umma_set_timing_buffer(unsigned long long *d);
cudaError_t launch_assign_affinity_umma(const Launch &L, const float *d_fobj, uint64_t n, const float *d_fnode_c, const float *d_fnode_g, const uint32_t *d_nidx_map, uint32_t n_live,
                                 uint32_t m_pad, uint32_t n_total, uint32_t *d_out_idx, float *d_out_cost, uint32_t *d_counters);
uint64_t launch_mix_rate(const Launch &L, uint32_t iters, uint32_t *d_sink);
void launch_synth_keys(const Launch &L, uint64_t *d_keys, uint64_t first, uint64_t n, uint64_t seed);
void launch_hash_ids(const Launch &L, const char *d_packed, const uint64_t *d_offsets, uint64_t n, uint64_t *d_keys);
void launch_fill_u32(const Launch &L, uint32_t *d, uint64_t n, uint32_t v);
void launch_histogram(const Launch &L, const uint32_t *d_idx, uint64_t n, uint32_t *d_counters, uint32_t n_total);

// bounded-load rounds: select spilling objects (idx on an over node, spill_hash < thr) into a compact list
void launch_select_spill(const Launch &L, const uint64_t *d_keys, const uint32_t *d_idx, uint64_t n, const uint32_t *d_thr /*n_total, 0 = not over*/,
                         const uint8_t *d_over, uint32_t round, uint32_t *d_sel, unsigned long long *d_nsel, uint32_t *d_counters);

// rebalance of a dense set
void launch_rebalance_join(const Launch &L, const uint64_t *d_keys, uint32_t *d_idx, uint64_t n, const NodeTabDev &tab, uint32_t new_idx,
                           uint32_t *d_counters, unsigned long long *d_moved);
void launch_select_on_node(const Launch &L, const uint32_t *d_idx, uint64_t n, uint32_t node, uint32_t *d_sel, unsigned long long *d_nsel);

// directory
void launch_dir_init(const Launch &L, DirSlot *slots, uint64_t cap);
void launch_dir_lookup(const Launch &L, const DirDev &dir, const uint64_t *d_keys, uint64_t n, uint32_t *d_out);
void launch_dir_upsert(const Launch &L, const DirDev &dir, const uint64_t *d_keys, const uint32_t *d_idx /*nullable => const_idx*/, uint32_t const_idx,
                       uint64_t n, uint32_t seq_base, unsigned long long *d_new_keys, uint32_t *d_error);
void launch_dir_clear_seq(const Launch &L, const DirDev &dir);
void launch_dir_clean_node(const Launch &L, const DirDev &dir, uint32_t node, unsigned long long *d_removed);
void launch_dir_clean_flagged(const Launch &L, const DirDev &dir, const uint8_t *d_flag, uint32_t n_total, unsigned long long *d_removed);
void launch_dir_rehash(const Launch &L, const DirDev &from, const DirDev &to, unsigned long long *d_new_keys, uint32_t *d_error);
void launch_dir_count(const Launch &L, const DirDev &dir, unsigned long long *d_placed, uint32_t *d_counters /*nullable*/, uint32_t n_total);
// directory-wide rebalance
void launch_dir_rebalance_join(const Launch &L, const DirDev &dir, const NodeTabDev &tab, uint32_t new_idx, unsigned long long *d_moved);
void launch_dir_rebalance_leave(const Launch &L, const DirDev &dir, const NodeTabDev &tab, uint32_t gone_idx, unsigned long long *d_moved);

// HRW2 launchers; DirDev-based one is the directory-wide eager rebalance
// tail (nullable, dense form only): the pass's exchange + capacity check runs in the last CTA of the walk kernel
void launch_assign_trie(const Launch &L, const uint64_t *d_keys, uint64_t n, const TrieDev &t, uint32_t *d_out_idx, uint32_t *d_counters /*nullable*/,
                        const uint32_t *d_sel /*nullable*/, uint64_t n_sel, uint32_t n_total, const BoundedTail *tail = nullptr);
void launch_reassign_trie(const Launch &L, const uint64_t *d_keys, uint64_t n, const TrieDev &t, uint32_t *d_idx, uint32_t *d_counters /*nullable*/,
                          uint32_t n_total, unsigned long long *d_moved);
void launch_dir_reassign_trie(const Launch &L, const DirDev &dir, const TrieDev &t, unsigned long long *d_moved);

// place_batch support: classify looked-up placements against node liveness
// need[i] = 1 if object must be (re)placed; dead_flag[node] = 1 for inactive well-formed nodes that were hit
void launch_classify(const Launch &L, const uint32_t *d_cur, uint64_t n, const uint8_t *d_node_state, uint32_t n_total, uint32_t *d_sel,
                     unsigned long long *d_nsel, uint8_t *d_dead_flag);
// check_address_mismatch for a batch: verdict[i] = verdict_tab[idx[i]] (RIO_ADDR_*; out-of-range index -> MALFORMED); nodes that
// drew DEALLOCATE are flagged for the clean_server scan and counted
void launch_check_address(const Launch &L, const uint32_t *d_idx, uint64_t n, const uint8_t *d_verdict_tab, uint32_t n_total, uint8_t *d_out, uint8_t *d_dead_flag,
                          unsigned long long *d_ndead);
void launch_scatter_const(const Launch &L, uint32_t *d_out, const uint32_t *d_sel, uint64_t n_sel, uint32_t v);
void launch_gather_keys(const Launch &L, const uint64_t *d_keys, const uint32_t *d_sel, uint64_t n_sel, uint64_t *d_out_keys, const uint32_t *d_idx,
                        uint32_t *d_out_idx);
void launch_exchange_p2p(const Launch &L, const uint32_t *d_local, uint32_t *const *peer_windows, uint32_t rank, uint32_t world, uint32_t M, uint32_t max_nodes,
                         uint32_t epoch, uint32_t *d_out_global);
// exchange (world > 1) + bounded-load capacity check as its own single-CTA launch (the flat rendezvous passes and the NCCL path)
void launch_exchange_check(const Launch &L, const uint32_t *d_local, const BoundedTail &b);
void launch_sum_gathered(const Launch &L, const uint32_t *d_gathered, uint32_t world, uint32_t M, uint32_t *d_out);
void launch_l2_flush(const Launch &L, uint32_t *d_buf, uint64_t n_words, uint32_t v);

// node-state bits for d_node_state
constexpr uint8_t kNodeLive = 1;       // active && weight > 0
constexpr uint8_t kNodeMalformed = 2;  // address has no "ip:port" shape (service.rs:213-222)

}  // namespace rio

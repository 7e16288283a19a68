// engine.cu -- host side of librio_cuda: engine state, node-table builds, directory sizing, the bounded-load
// round protocol, the NCCL counter exchange, and every extern "C" entry point declared in include/rio_cuda.h.
//
// Reference interface mirrored: trait ObjectPlacement (rio-rs/src/object_placement/mod.rs:38-56) and the policy
// around it (rio-rs/src/service.rs:193-254).  There is NO CPU fallback anywhere in this file: without a CUDA
// device rio_cuda_create fails with RIO_ERR_UPSTREAM.
#include "../../include/rio_cuda.h"
#include "../../include/rio_cuda_dev.h"
#include "kernels.cuh"
#include "k_ranked.cuh"
#include "k_affinity_ranked.cuh"
#include "k_affinity_spread.cuh"
#include "k_affinity_set.cuh"
#include "k_affinity_bounded.cuh"
#include "k_set_bounded_affinity.cuh"
#include "k_set_churn.cuh"
#include "k_set_commit.cuh"
#include "k_bounded_weighted.cuh"
#include "k_set_weighted_changes.cuh"
#include "k_changes.cuh"
#include "k_ranked_changes.cuh"
#include "k_spread.cuh"
#include "k_spread_changes.cuh"
#include "spec.cuh"
#include "trie_table.hpp"

#include <dlfcn.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

using namespace rio;

namespace {

thread_local std::string g_last_error;

struct RioError {
    rio_status code;
    std::string msg;
};

#define CUDA_TRY(expr)                                                                                         \
    do {                                                                                                       \
        cudaError_t e__ = (expr);                                                                              \
        if (e__ != cudaSuccess)                                                                                \
            throw RioError{RIO_ERR_UPSTREAM, std::string(#expr) + ": " + cudaGetErrorString(e__)};             \
    } while (0)
#define REQUIRE(cond, msg)                                                      \
    do {                                                                        \
        if (!(cond)) throw RioError{RIO_ERR_UNKNOWN, std::string(msg)};         \
    } while (0)

// ---- NCCL through dlopen: no link-time dependency, and inside a torch process we share torch's libnccl ----
struct NcclId { char internal[128]; };
typedef void *NcclComm;
struct NcclApi {
    void *lib = nullptr;
    int (*GetUniqueId)(NcclId *) = nullptr;
    int (*CommInitRank)(NcclComm *, int, NcclId, int) = nullptr;
    int (*AllGather)(const void *, void *, size_t, int, NcclComm, cudaStream_t) = nullptr;
    int (*CommDestroy)(NcclComm) = nullptr;
    const char *(*GetErrorString)(int) = nullptr;
    std::string load_error;
    bool load() {
        if (lib) return true;
        const char *names[] = {getenv("RIO_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
        for (const char *nm : names) {
            if (!nm || !*nm) continue;
            lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
            if (lib) break;
            load_error = dlerror();
        }
        if (!lib) return false;
        GetUniqueId = (decltype(GetUniqueId))dlsym(lib, "ncclGetUniqueId");
        CommInitRank = (decltype(CommInitRank))dlsym(lib, "ncclCommInitRank");
        AllGather = (decltype(AllGather))dlsym(lib, "ncclAllGather");
        CommDestroy = (decltype(CommDestroy))dlsym(lib, "ncclCommDestroy");
        GetErrorString = (decltype(GetErrorString))dlsym(lib, "ncclGetErrorString");
        if (!GetUniqueId || !CommInitRank || !AllGather || !CommDestroy) { load_error = "libnccl lacks required symbols"; lib = nullptr; return false; }
        return true;
    }
};
NcclApi g_nccl;
std::mutex g_nccl_mu;
constexpr int kNcclUint32 = 3;

#define NCCL_TRY(expr)                                                                                              \
    do {                                                                                                            \
        int r__ = (expr);                                                                                           \
        if (r__ != 0)                                                                                               \
            throw RioError{RIO_ERR_UPSTREAM, std::string(#expr) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r__) : "nccl error")}; \
    } while (0)

// ---- growable stream-ordered device buffer ---------------------------------------------------------------
struct DevBuf {
    void *p = nullptr;
    size_t bytes = 0;
    void ensure(size_t need, cudaStream_t st) {
        if (need <= bytes) return;
        size_t nb = std::max(need, bytes + bytes / 2);
        nb = (nb + 255) & ~(size_t)255;
        if (p) CUDA_TRY(cudaFreeAsync(p, st));
        p = nullptr; bytes = 0;
        CUDA_TRY(cudaMallocAsync(&p, nb, st));
        bytes = nb;
    }
    void release(cudaStream_t st) { if (p) cudaFreeAsync(p, st); p = nullptr; bytes = 0; }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};

struct NodeInfo {
    std::string addr;
    uint64_t seed = 0, seed2 = 0;
    uint32_t weight = 0;
    uint32_t domain = RIO_NONE;   // failure-domain label (DESIGN.md 3.12); RIO_NONE = a domain of its own
    bool active = false;
    bool malformed = false;
    std::vector<float> feat;
    bool live() const { return active && weight > 0 && !malformed; }
};

// Every array a table build produces is laid out in ONE pinned staging area and crosses PCIe as ONE copy; the device side is a
// single allocation the kernels' pointers index into.  A membership event therefore costs one host-side build (~0.1 ms at 1024
// nodes), one H2D of ~70 KB and no synchronisation of its own.
struct TabBufs {
    DevBuf dev;
    unsigned char *stage = nullptr;   // pinned
    size_t stage_cap = 0;
    bool upload_pending = false;
    NodeTabDev tab{};
    TrieDev trie{};
    const uint8_t *state = nullptr;   // per interned node: kNodeLive | kNodeMalformed (the policy's view)
    const uint32_t *live = nullptr;   // per interned node: solver eligibility (active, weight > 0)
};

// device scalars (one small allocation): [0]=nsel [1]=moved/removed [2]=new keys (cumulative) [3]=placed ; u32 error at [8]
enum { S_NSEL = 0, S_MOVED = 1, S_NEWKEYS = 2, S_PLACED = 3, S_FLAGS = 4 /* host-only: {any over, open nodes} written by k_exchange_check */, S_CHANGED = 5,
       S_WSUM = 6 /* weight sum of a weighted bounded call (DESIGN.md 3.19) */, S_COUNT = 8 };

// Device + host state of one bounded-load call in flight (DESIGN.md 3.5): capacities, global counters, thresholds, closed set,
// the fused tail's ticket, and three words of mapped pinned memory the capacity check reports into.  Every resident set owns
// one (so several sets can be between _begin and _end at once) and the handle owns one for the host-buffer call.
struct BoundedState {
    DevBuf buf;
    uint32_t *h_flags = nullptr;              // pinned, mapped: {any over, open nodes, sequence number}
    cudaEvent_t ev = nullptr;                 // "pass 0 done" for the check that runs on the auxiliary stream
    uint32_t flag_seq = 0;                    // sequence number of the last check launched into h_flags
    uint32_t epoch = 0;                       // closed-set tag of the current call
    uint64_t cap_key[4] = {~0ull, 0, 0, 0};   // (n_total_objs, num << 32 | den, table version, M) the uploaded capacities belong to
    // the call between _begin and _end
    bool active = false;
    uint64_t n_total_objs = 0;
    uint32_t max_rounds = 0, M = 0;
    uint64_t live_sig = 0;                    // the live node set (indices, weights) pass 0 and the capacities were computed for
    void release(cudaStream_t st) { buf.release(st); if (h_flags) cudaFreeHost(h_flags); h_flags = nullptr; if (ev) cudaEventDestroy(ev); ev = nullptr; }
};

// The kind of a ranked call's or a resident set's lists, from keys: each object's first R nodes under the handle's policy (kHash,
// DESIGN.md 3.9) or its first R nodes in R distinct failure domains (kSpread, 3.12); from feature rows: its R lowest-cost nodes
// (kAffinity, 3.9) or those in R distinct domains (kAffinitySpread, 3.14)
enum class ListKind { kHash, kSpread, kAffinity, kAffinitySpread };
bool is_affinity(ListKind k) { return k == ListKind::kAffinity || k == ListKind::kAffinitySpread; }
bool is_spread(ListKind k) { return k == ListKind::kSpread || k == ListKind::kAffinitySpread; }

}  // namespace

struct rio_placement {
    std::mutex mu;
    int device = 0, sm_count = 0;
    size_t hbm = 0;
    std::string devname;
    cudaStream_t stream = nullptr, h2d_stream = nullptr, d2h_stream = nullptr, aux_stream = nullptr;   // aux: capacity checks of pipelined passes
    uint64_t launches = 0;

    std::vector<NodeInfo> nodes;
    std::unordered_map<std::string, uint32_t> node_index;
    uint32_t K = 0;
    uint32_t dev_table_flags = 0;       // rio_dev_set_table_options
    uint32_t solver = RIO_SOLVER_HRW;   // policy of assign_batch / set_assign / rebalance (rio_cuda_set_solver)
    uint32_t trie_bits = 12;            // HRW2: depth of the binary trie over node positions (DESIGN.md 3.8)
    bool tab_dirty = true;
    TabBufs tabs, tabs_masked;
    DevBuf d_fnode, d_fnode_c, d_fnode_g, d_nidx_map;
    uint32_t aff_live = 0, aff_pad = 0;   // compacted live-node operands of the tensor-core affinity kernel
    // the same operands over live minus closed, rebuilt for every spill round of a bounded affinity call (DESIGN.md 3.16); grow-only
    DevBuf d_fnode_cm, d_fnode_gm, d_nidx_map_m;
    uint32_t aff_live_m = 0, aff_pad_m = 0;

    DirDev dir{};
    uint64_t dir_cap = 0;
    uint64_t dir_keys = 0;      // distinct keys claimed (exact after every host-synchronous call)
    uint64_t dir_keys_pending = 0;  // pessimistic additions from _dev upserts not yet reconciled
    uint32_t dir_seq = 0;           // upsert sequence numbers handed out so far (ordering of duplicate keys, k_dir_upsert)

    DevBuf s_keys, s_idx, s_idx2, s_sel, s_slots, s_keys2, s_feats, s_packed, s_offsets, s_cost, s_misc, s_flush, s_gather;
    DevBuf s_rows;                            // the spilled objects' feature rows of a bounded affinity round
    DevBuf s_churn;                           // set_erase (DESIGN.md 3.18): erase-key hash set, row flags, per-block counts and offsets
    DevBuf s_commit, s_manifest;              // set_commit_changes (DESIGN.md 3.20): per-block counts and offsets, from, row flags; the manifest
    DevBuf s_weights;                         // the object weights of rio_cuda_assign_bounded_weighted_batch (DESIGN.md 3.19)
    // bounded-load state kept on the device between passes (DESIGN.md 3.5): [ticket | cap | global counters | thr | closed epoch | over] x node
    BoundedState bs;                          // for rio_cuda_assign_bounded_batch (host buffers)
    uint64_t tab_version = 0;
    uint64_t live_sig = 0;                    // live_signature() of the node set the current table was built from
    // side table of the ranked HRW2 walk (DESIGN.md 3.9): built on the first ranked call after a table change, never by other calls
    DevBuf rank_dev;
    std::vector<unsigned char> rank_stage;
    TrieRankDev rank_tab{};
    uint64_t rank_version = ~0ull;            // tab_version the side table belongs to
    // side table of the spread walks (DESIGN.md 3.12): built on the first spread call after a table or label change.  Labels never
    // touch tab_version: no other call depends on them.
    uint64_t label_version = 0;
    DevBuf spread_dev;
    std::vector<unsigned char> spread_stage;
    SpreadTabDev spread_tab{};
    uint64_t spread_version[2] = {~0ull, ~0ull};   // (tab_version, label_version) the side table belongs to
    // dense domain ids of the failure-domain affinity lists (DESIGN.md 3.14): n_total per interned index, then aff_pad per compacted
    // affinity position (the order of d_nidx_map), built on the first such call after a table or label change
    DevBuf aff_dom;
    size_t aff_dom_pos = 0;                        // offset of the per-position ids in aff_dom
    uint64_t aff_dom_version[2] = {~0ull, ~0ull};
    // bumped by every call that sets node features (set_nodes with feats, node_upsert with feat): the affinity resident sets compare
    // their feature snapshot only when it moved (DESIGN.md 3.15)
    uint64_t feat_version = 0;
    unsigned long long *d_scalars = nullptr;   // S_COUNT u64 + error u32
    unsigned long long *h_scalars = nullptr;   // pinned mirror

    cudaEvent_t events[RIO_MAX_EVENTS] = {};
    cudaEvent_t ev_pipe[8] = {};
    cudaEvent_t ev_aux = nullptr;   // recorded behind every capacity check on the auxiliary stream
    bool aux_used = false;

    NcclComm comm = nullptr;
    int rank = 0, world = 1;
    // peer-memory exchange window (CUDA IPC): slots[2][world][xchg_nodes] + flags[world]
    uint32_t *xchg_mine = nullptr;
    uint32_t *xchg_peer[16] = {};
    uint32_t xchg_nodes = 0, xchg_epoch = 0;
    bool xchg_ready = false;

    int walk_spare = 0;   // set around a pipelined pass: the walk leaves one CTA slot free for the check kernel of the previous pass
    Launch L() { return Launch{stream, sm_count, &launches, walk_spare}; }
    uint32_t *d_error() { return reinterpret_cast<uint32_t *>(d_scalars + S_COUNT); }
};

struct rio_objset {
    rio_placement *h = nullptr;
    uint64_t capacity = 0, n = 0;
    DevBuf keys, idx, feats, counters, counters_alt, sel;
    uint32_t K = 0;
    uint32_t counters_n = 0;
    bool alt_zero = false;     // counters_alt is known to be all zero (the capacity check of the last bounded pass cleared it)
    BoundedState bs;
    bool assigned = false;
    // ranked lists (DESIGN.md 3.11): n x ranks row-major, column 0 == idx; ranks == 0 = the set holds none.  The buffer is grow-only
    // (capacity x ranks), the lists record their kind (meaningful while ranks != 0) and the policy they were computed under.
    DevBuf lists;
    uint32_t ranks = 0, rank_solver = 0, rank_bits = 0;
    ListKind kind = ListKind::kHash;
    // spread kinds (DESIGN.md 3.13): the lists are failure-domain lists, computed under the labels of label_snap (one per node interned
    // then; a node interned later had RIO_NONE), which were the handle's labels at label_version label_snap_version
    std::vector<uint32_t> label_snap;
    uint64_t label_snap_version = 0;
    // affinity kinds (DESIGN.md 3.15): the lists are affinity lists of the set's features, computed on the tensor cores (aff_tensor) or
    // the CUDA cores under the handle's K aff_K, with the node features of feat_snap (aff_K floats per node interned then; a row that
    // was not K wide is zeros, as the kernels see it), the handle's at feat_version feat_snap_version
    bool aff_tensor = false;
    uint32_t aff_K = 0;
    std::vector<float> feat_snap;
    uint64_t feat_snap_version = 0;
    // bounded-load affinity record (DESIGN.md 3.17): idx is the result of set_assign_bounded_affinity or of the change-set call that
    // keeps it, on the path of aff_tensor under aff_K, with the node features of feat_snap.  Cleared with the lists and by load_feats.
    bool bounded_aff = false;
    // the plain kind (DESIGN.md 3.18): how the last call that rewrote idx without lists placed it, for set_insert -- by the hash
    // policy, or by the affinity argmin on the tensor cores (plain_tensor) or the CUDA cores.  Set by set_assign, the bounded assigns
    // and the set rebalances; left alone by every other call.
    bool plain_aff = false, plain_tensor = false;
    // the weight column (DESIGN.md 3.19): one u32 per row, capacity rows, allocated by the first rio_cuda_set_write_weights; while
    // has_weights is false every weight is 1 (set_load_keys and set_synth_keys clear it).  loads: M u32 of per-node weight sums.
    DevBuf weights, loads;
    bool has_weights = false;
    const uint32_t *weights_or_null() const { return has_weights ? weights.as<uint32_t>() : nullptr; }
    // weighted-bounded record (DESIGN.md 3.21): idx is the result of set_assign_bounded_weighted or of the change-set call that keeps
    // it, by the plain kind -- the hash policy of (bw_solver, bw_bits), or the affinity argmin (plain_aff) on the path of aff_tensor
    // under aff_K with the node features of feat_snap.  Cleared with the lists, and for affinity by load_feats.
    bool bounded_w = false;
    uint32_t bw_solver = 0, bw_bits = 0;
    void drop_lists() { ranks = 0; kind = ListKind::kHash; bounded_aff = false; bounded_w = false; }
};

namespace {

void use_device(rio_placement *h) { CUDA_TRY(cudaSetDevice(h->device)); }

void zero_scalar(rio_placement *h, int which) { CUDA_TRY(cudaMemsetAsync(h->d_scalars + which, 0, 8, h->stream)); }
uint64_t read_scalar(rio_placement *h, int which) {
    CUDA_TRY(cudaMemcpyAsync(h->h_scalars + which, h->d_scalars + which, 8, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(cudaStreamSynchronize(h->stream));
    return h->h_scalars[which];
}
void check_device_error(rio_placement *h) {
    uint32_t e = 0;
    CUDA_TRY(cudaMemcpyAsync(&e, h->d_error(), 4, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(cudaStreamSynchronize(h->stream));
    if (e) { CUDA_TRY(cudaMemsetAsync(h->d_error(), 0, 4, h->stream)); throw RioError{RIO_ERR_UNKNOWN, "directory table overflow (internal sizing error)"}; }
}

bool address_malformed(const std::string &a) {
    // service.rs:205-213: splitn(2, ":") must give a non-empty ip and a non-empty port
    size_t c = a.find(':');
    return c == std::string::npos || c == 0 || c + 1 >= a.size();
}

uint32_t intern_node(rio_placement *h, const std::string &addr) {
    auto it = h->node_index.find(addr);
    if (it != h->node_index.end()) return it->second;
    REQUIRE(h->nodes.size() < 0xFFFFFFF0u, "too many nodes");
    NodeInfo ni;
    ni.addr = addr;
    ni.seed = mix64(fnv1a64(addr.data(), addr.size()));
    ni.seed2 = mix64(ni.seed ^ kSaltNode2);
    ni.malformed = address_malformed(addr);
    uint32_t idx = (uint32_t)h->nodes.size();
    h->nodes.push_back(std::move(ni));
    h->node_index.emplace(addr, idx);
    h->tab_dirty = true;
    return idx;
}

// Build the class-sorted table of live nodes (optionally excluding `closed`) and upload it.
void build_tab(rio_placement *h, TabBufs &tb, const std::vector<uint8_t> *closed) {
    const uint32_t n_total = (uint32_t)h->nodes.size();
    struct Ent { uint32_t invw, idx; };
    std::vector<Ent> live;
    // `closed` was sized when the bounded call began; addresses interned since then (update() may record any address) are not in it
    auto is_closed = [&](uint32_t j) { return closed && j < closed->size() && (*closed)[j]; };
    for (uint32_t j = 0; j < n_total; j++) {
        const NodeInfo &ni = h->nodes[j];
        if (!ni.live()) continue;
        if (is_closed(j)) continue;
        live.push_back(Ent{inv_weight(ni.weight), j});
    }
    // Order by (inverse weight, node index).  `live` is in index order already, so this is a STABLE grouping by inverse weight: with
    // the few weight classes real clusters have (<= 64 distinct values) it is two linear passes instead of a sort; otherwise sort.
    {
        std::vector<uint32_t> classes_seen;
        bool few = true;
        for (const Ent &e : live) {
            if (std::find(classes_seen.begin(), classes_seen.end(), e.invw) != classes_seen.end()) continue;
            if (classes_seen.size() == 64) { few = false; break; }
            classes_seen.push_back(e.invw);
        }
        if (few) {
            std::sort(classes_seen.begin(), classes_seen.end());
            std::vector<uint32_t> start(classes_seen.size() + 1, 0);
            auto cls = [&](uint32_t invw) { return (size_t)(std::lower_bound(classes_seen.begin(), classes_seen.end(), invw) - classes_seen.begin()); };
            for (const Ent &e : live) start[cls(e.invw) + 1]++;
            for (size_t c = 0; c < classes_seen.size(); c++) start[c + 1] += start[c];
            std::vector<Ent> grouped(live.size());
            for (const Ent &e : live) grouped[start[cls(e.invw)]++] = e;
            live.swap(grouped);
        } else {
            std::sort(live.begin(), live.end(), [](const Ent &a, const Ent &b) { return a.invw != b.invw ? a.invw < b.invw : a.idx < b.idx; });
        }
    }
    std::vector<NodeRec> recs(live.size() ? live.size() : 1);
    std::vector<ClassRec> classes;
    for (size_t q = 0; q < live.size(); q++) {
        const NodeInfo &ni = h->nodes[live[q].idx];
        recs[q] = NodeRec{(uint32_t)ni.seed, live[q].idx, (uint32_t)(ni.seed >> 32) | 1u, (uint32_t)ni.seed2};
        if (q == 0 || live[q].invw != live[q - 1].invw || (h->dev_table_flags & RIO_DEV_SPLIT_CLASSES)) classes.push_back(ClassRec{(uint32_t)q, live[q].invw});
    }
    const uint32_t n_classes = (uint32_t)classes.size();
    classes.push_back(ClassRec{(uint32_t)live.size(), 0});
    classes.push_back(ClassRec{(uint32_t)live.size(), 0});   // one spare so classes[c+1] is always readable
    std::vector<uint4> by_idx(n_total ? n_total : 1);
    for (uint32_t j = 0; j < n_total; j++) {
        const NodeInfo &ni = h->nodes[j];
        const bool lv = ni.live() && !is_closed(j);
        by_idx[j] = make_uint4((uint32_t)ni.seed, lv ? inv_weight(ni.weight) : 0u, (uint32_t)(ni.seed >> 32) | 1u, (uint32_t)ni.seed2);
    }
    // ---- HRW2 table (DESIGN.md 3.8): thresholds of the binary trie over node positions, leaf words, chain records: the builder
    // is shared with the client library (trie_table.hpp), so clients and servers walk byte-identical tables ----
    std::vector<TrieMember> members;
    members.reserve(live.size());
    for (const Ent &e : live) members.push_back(TrieMember{h->nodes[e.idx].seed, e.idx, h->nodes[e.idx].weight});
    const TrieBlob blob = build_trie_blob(members, h->trie_bits);
    const uint32_t bits = blob.bits, nb = 1u << bits, blob_bytes = blob.blob_bytes;
    // the policy's view of every interned node (service.rs:226-231 asks is_active only: a draining node -- active, weight 0 --
    // keeps its objects) and the solver's (active and weight > 0)
    std::vector<uint8_t> state(n_total ? n_total : 1, 0);
    std::vector<uint32_t> livef(n_total ? n_total : 1, 0);
    for (uint32_t j = 0; j < n_total; j++) {
        const NodeInfo &ni = h->nodes[j];
        state[j] = ((ni.active && !ni.malformed) ? kNodeLive : 0) | (ni.malformed ? kNodeMalformed : 0);
        livef[j] = (ni.live() && !is_closed(j)) ? 1u : 0u;   // the CUDA-core affinity rounds of 3.16 read the masked flags
    }

    // ---- one staging area, one copy ----
    auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
    const size_t o_recs = 0, o_classes = al(o_recs + recs.size() * sizeof(NodeRec)), o_byidx = al(o_classes + classes.size() * sizeof(ClassRec)),
                 o_trie = al(o_byidx + by_idx.size() * sizeof(uint4)), o_state = al(o_trie + blob_bytes), o_live = al(o_state + state.size()),
                 total = al(o_live + livef.size() * 4);
    cudaStream_t st = h->stream;
    if (tb.upload_pending) { CUDA_TRY(cudaStreamSynchronize(st)); tb.upload_pending = false; }   // the previous copy still reads the staging area
    if (h->aux_stream) CUDA_TRY(cudaStreamSynchronize(h->aux_stream));   // a pipelined capacity check may still be reading the old table's node states
    if (total > tb.stage_cap) {
        if (tb.stage) CUDA_TRY(cudaFreeHost(tb.stage));
        tb.stage = nullptr; tb.stage_cap = 0;
        CUDA_TRY(cudaMallocHost(reinterpret_cast<void **>(&tb.stage), total * 2));
        tb.stage_cap = total * 2;
    }
    memcpy(tb.stage + o_recs, recs.data(), recs.size() * sizeof(NodeRec));
    memcpy(tb.stage + o_classes, classes.data(), classes.size() * sizeof(ClassRec));
    memcpy(tb.stage + o_byidx, by_idx.data(), by_idx.size() * sizeof(uint4));
    memcpy(tb.stage + o_trie, blob.words.data(), blob_bytes);
    memcpy(tb.stage + o_state, state.data(), state.size());
    memcpy(tb.stage + o_live, livef.data(), livef.size() * 4);
    tb.dev.ensure(total, st);
    CUDA_TRY(cudaMemcpyAsync(tb.dev.p, tb.stage, total, cudaMemcpyHostToDevice, st));
    tb.upload_pending = true;
    unsigned char *d = tb.dev.as<unsigned char>();
    tb.trie = TrieDev{d + o_trie, blob_bytes, blob.off_crec, bits, blob.n_chain, {}};
    for (uint32_t i = 1; i < 8 && i < nb; i++) tb.trie.top[i] = blob.words[i];
    tb.tab.recs = reinterpret_cast<const NodeRec *>(d + o_recs);
    tb.tab.classes = reinterpret_cast<const ClassRec *>(d + o_classes);
    tb.tab.by_idx = reinterpret_cast<const uint4 *>(d + o_byidx);
    tb.tab.n_live = (uint32_t)live.size();
    tb.tab.n_classes = n_classes;
    tb.tab.n_total = n_total;
    tb.state = d + o_state;
    tb.live = reinterpret_cast<const uint32_t *>(d + o_live);
}

// One word that changes when the live node set or a live weight changes (interning a never-live address does not change it).
uint64_t live_signature(const rio_placement *h) {
    uint64_t sig = kFnvBasis;
    for (uint32_t j = 0; j < (uint32_t)h->nodes.size(); j++)
        if (h->nodes[j].live()) sig = mix64(sig ^ (((uint64_t)j << 32) | h->nodes[j].weight));
    return sig;
}

// The compacted live nodes (node-index order) of the tensor-core affinity kernel, zero padded to the node tile, without the nodes
// `closed` marks (a spill round of DESIGN.md 3.16), into (fc, fg, map); n_live / n_pad receive the kernel's live and padded counts.
// Synchronises the stream: the host vectors go out of scope.
void build_aff_operands(rio_placement *h, const std::vector<uint8_t> *closed, DevBuf &fc_buf, DevBuf &fg_buf, DevBuf &map_buf, uint32_t &n_live,
                        uint32_t &n_pad) {
    const uint32_t n_total = (uint32_t)h->nodes.size();
    cudaStream_t st = h->stream;
    auto is_closed = [&](uint32_t j) { return closed && j < closed->size() && (*closed)[j]; };
    std::vector<uint32_t> map;
    for (uint32_t j = 0; j < n_total; j++) if (h->nodes[j].live() && !is_closed(j)) map.push_back(j);
    const uint32_t nl = (uint32_t)map.size();
    const uint32_t pad = nl <= 64 ? 64 : (nl + 255) / 256 * 256;
    std::vector<float> fc((size_t)pad * 16, 0.f);
    for (uint32_t q = 0; q < nl; q++) if (h->nodes[map[q]].feat.size() == 16) std::copy(h->nodes[map[q]].feat.begin(), h->nodes[map[q]].feat.end(), fc.begin() + (size_t)q * 16);
    map.resize(pad, kNone);
    // the same rows regrouped as [group of 8 nodes][16-byte piece][node in group] for k_affinity_resolve
    std::vector<float> fg(fc.size());
    for (uint32_t g8 = 0; g8 < pad / 8; g8++)
        for (uint32_t k4 = 0; k4 < 4; k4++)
            for (uint32_t r8 = 0; r8 < 8; r8++)
                std::copy_n(fc.begin() + ((size_t)g8 * 8 + r8) * 16 + k4 * 4, 4, fg.begin() + (((size_t)g8 * 4 + k4) * 8 + r8) * 4);
    fc_buf.ensure(fc.size() * 4, st);
    fg_buf.ensure(fg.size() * 4, st);
    CUDA_TRY(cudaMemcpyAsync(fg_buf.p, fg.data(), fg.size() * 4, cudaMemcpyHostToDevice, st));
    map_buf.ensure(map.size() * 4, st);
    CUDA_TRY(cudaMemcpyAsync(fc_buf.p, fc.data(), fc.size() * 4, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(map_buf.p, map.data(), map.size() * 4, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    n_live = nl; n_pad = pad;
}

void ensure_tab(rio_placement *h) {
    if (!h->tab_dirty) return;
    build_tab(h, h->tabs, nullptr);
    const uint32_t n_total = (uint32_t)h->nodes.size();
    cudaStream_t st = h->stream;
    h->tab_dirty = false;
    h->tab_version++;
    h->live_sig = live_signature(h);
    if (!h->K) return;   // hash path only: nothing else to upload, and no synchronisation
    std::vector<float> fnode((size_t)(n_total ? n_total : 1) * h->K, 0.f);
    for (uint32_t j = 0; j < n_total; j++) {
        const NodeInfo &ni = h->nodes[j];
        if (ni.feat.size() == h->K) std::copy(ni.feat.begin(), ni.feat.end(), fnode.begin() + (size_t)j * h->K);   // others keep zeros
    }
    h->d_fnode.ensure(fnode.size() * 4, st);
    CUDA_TRY(cudaMemcpyAsync(h->d_fnode.p, fnode.data(), fnode.size() * 4, cudaMemcpyHostToDevice, st));
    h->aff_live = h->aff_pad = 0;
    if (h->K == 16) build_aff_operands(h, nullptr, h->d_fnode_c, h->d_fnode_g, h->d_nidx_map, h->aff_live, h->aff_pad);
    CUDA_TRY(cudaStreamSynchronize(st));   // the host vectors above go out of scope
}

// ---- directory sizing ---------------------------------------------------------------------------------------
uint64_t pow2_at_least(uint64_t v) { uint64_t p = 1; while (p < v) p <<= 1; return p; }

void dir_alloc(rio_placement *h, uint64_t cap, DirDev &out) {
    void *p = nullptr;
    CUDA_TRY(cudaMallocAsync(&p, cap * sizeof(DirSlot), h->stream));
    out.slots = reinterpret_cast<DirSlot *>(p);
    out.mask = cap - 1;
    uint32_t lg = 0; while ((1ull << lg) < cap) lg++;
    out.shift = 64 - lg;
    launch_dir_init(h->L(), out.slots, cap);
}

void reconcile_dir_keys(rio_placement *h) {
    h->dir_keys = read_scalar(h, S_NEWKEYS);
    h->dir_keys_pending = 0;
}

// make room for n_more distinct new keys at load factor <= 0.5 after growth, <= 0.7 before
void dir_reserve(rio_placement *h, uint64_t n_more) {
    const uint64_t need = h->dir_keys + h->dir_keys_pending + n_more;
    if (need * 10 <= h->dir_cap * 7) return;
    if (h->dir_keys_pending) { reconcile_dir_keys(h); if ((h->dir_keys + n_more) * 10 <= h->dir_cap * 7) return; }
    // Removed / cleaned keys stay in the table as tombstones (they keep probe chains intact) and are counted in dir_keys; the
    // rehash drops them, so the new table is sized for the keys that are actually placed: under create/remove churn with a
    // constant live count this is a same-size compaction, not a doubling.
    zero_scalar(h, S_PLACED);
    launch_dir_count(h->L(), h->dir, h->d_scalars + S_PLACED, nullptr, 0);
    const uint64_t placed = read_scalar(h, S_PLACED);
    const uint64_t new_cap = pow2_at_least(std::max<uint64_t>((placed + n_more) * 2, 1024));
    DirDev nd{};
    dir_alloc(h, new_cap, nd);
    CUDA_TRY(cudaMemsetAsync(h->d_scalars + S_NEWKEYS, 0, 8, h->stream));
    launch_dir_rehash(h->L(), h->dir, nd, h->d_scalars + S_NEWKEYS, h->d_error());
    CUDA_TRY(cudaFreeAsync(h->dir.slots, h->stream));
    h->dir = nd;
    h->dir_cap = new_cap;
    h->dir_seq = 0;   // the rehash copied node indices only
    check_device_error(h);
    reconcile_dir_keys(h);   // unplaced keys were dropped by the rehash
}

void dir_upsert_dev(rio_placement *h, const uint64_t *d_keys, const uint32_t *d_idx, uint32_t const_idx, uint64_t n) {
    if (!n) return;
    REQUIRE(n < 0xFFFFFFF0ull, "upsert batch too large");
    if ((uint64_t)h->dir_seq + n + 1 > 0xFFFFFFFFull) {   // sequence space exhausted: one streaming pass resets it
        launch_dir_clear_seq(h->L(), h->dir);
        h->dir_seq = 0;
    }
    launch_dir_upsert(h->L(), h->dir, d_keys, d_idx, const_idx, n, h->dir_seq, h->d_scalars + S_NEWKEYS, h->d_error());
    h->dir_seq += (uint32_t)n;
}

// ---- counter exchange: the single collective of the path (all-gather of M u32 per rank, then a sum) -------------
// Exchanges carry consecutive epochs and must reach the device in epoch order on every rank.  Checks of pipelined calls run on
// the auxiliary stream; anything that exchanges on the main stream afterwards waits for them first.
void order_behind_aux_checks(rio_placement *h) {
    if (h->aux_used) CUDA_TRY(cudaStreamWaitEvent(h->stream, h->ev_aux, 0));
}

void exchange_counters(rio_placement *h, const uint32_t *d_local, uint32_t *d_global, uint32_t M) {
    order_behind_aux_checks(h);
    if (h->world > 1 && h->xchg_ready && M <= h->xchg_nodes) {
        // one kernel: P2P stores into every peer's window + flags over NVLink, no NCCL launch on the critical path
        launch_exchange_p2p(h->L(), d_local, h->xchg_peer, (uint32_t)h->rank, (uint32_t)h->world, M, h->xchg_nodes, ++h->xchg_epoch, d_global);
        return;
    }
    if (h->world <= 1 || !h->comm) {
        if (d_local != d_global) CUDA_TRY(cudaMemcpyAsync(d_global, d_local, (size_t)M * 4, cudaMemcpyDeviceToDevice, h->stream));
        return;
    }
    h->s_gather.ensure((size_t)M * 4 * h->world, h->stream);
    NCCL_TRY(g_nccl.AllGather(d_local, h->s_gather.p, M, kNcclUint32, h->comm, h->stream));
    launch_sum_gathered(h->L(), h->s_gather.as<uint32_t>(), (uint32_t)h->world, M, d_global);
}

// the hash-path solver of the handle: flat weighted rendezvous (M pair hashes per object) or HRW2 (~log2 M contests)
void run_assign(rio_placement *h, uint32_t solver, const TabBufs &tb, const uint64_t *d_keys, uint64_t n, uint32_t *d_out_idx, uint32_t *d_counters,
                const uint32_t *d_sel, uint64_t n_sel) {
    if (solver == RIO_SOLVER_HRW2) launch_assign_trie(h->L(), d_keys, n, tb.trie, d_out_idx, d_counters, d_sel, n_sel, tb.tab.n_total);
    else launch_assign_hrw(h->L(), d_keys, n, tb.tab, d_out_idx, d_counters, d_sel, n_sel);
}

// The ranked HRW2 walk needs, beside the blob, the subtree weights the thresholds came from and every live node's bucket and
// weight.  The builder is run again for the current live set (a pure function of it: the same blob, and its weight heap).
void ensure_rank_tab(rio_placement *h) {
    if (h->rank_version == h->tab_version) return;
    const uint32_t n_total = (uint32_t)h->nodes.size();
    std::vector<TrieMember> members;
    for (uint32_t j = 0; j < n_total; j++)
        if (h->nodes[j].live()) members.push_back(TrieMember{h->nodes[j].seed, j, h->nodes[j].weight});
    const TrieBlob blob = build_trie_blob(members, h->trie_bits);
    const uint32_t bits = blob.bits, nb = 1u << bits;
    const size_t o_node = (size_t)nb * 16, total = o_node + ((size_t)n_total * 8 + 15) / 16 * 16;
    h->rank_stage.assign(total, 0);
    memcpy(h->rank_stage.data(), blob.wsum.data(), (size_t)nb * 16);
    uint2 *node = reinterpret_cast<uint2 *>(h->rank_stage.data() + o_node);
    for (const TrieMember &m : members) {
        const uint64_t pos = mix64(m.seed ^ kSaltPos);
        node[m.idx] = make_uint2(bits ? (uint32_t)(pos >> (64 - bits)) : 0u, m.weight);
    }
    cudaStream_t st = h->stream;
    h->rank_dev.ensure(total, st);
    CUDA_TRY(cudaMemcpyAsync(h->rank_dev.p, h->rank_stage.data(), total, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    unsigned char *d = h->rank_dev.as<unsigned char>();
    h->rank_tab = TrieRankDev{reinterpret_cast<const unsigned long long *>(d), reinterpret_cast<const uint2 *>(d + o_node), n_total,
                              (uint32_t)members.size(), (uint32_t)total};
    h->rank_version = h->tab_version;
}

void check_ranked_args(size_t n, uint32_t ranks) {
    REQUIRE(ranks >= 1 && ranks <= RIO_MAX_RANKS, "ranks must be in [1, RIO_MAX_RANKS]");
    REQUIRE(n <= SIZE_MAX / 4 / ranks, "n x ranks overflows");
}

// Dense domain ids of the live nodes per interned index (kNone for the others): one per label shared by live nodes, one per live
// node labelled RIO_NONE, numbered in node-index order.  Returns the number of domains.
uint32_t dense_domains(const rio_placement *h, std::vector<uint32_t> &ndom) {
    ndom.assign(h->nodes.size(), kNone);
    std::unordered_map<uint32_t, uint32_t> dense;
    uint32_t n_dom = 0;
    for (uint32_t j = 0; j < (uint32_t)h->nodes.size(); j++) {
        const NodeInfo &ni = h->nodes[j];
        if (!ni.live()) continue;
        if (ni.domain == RIO_NONE) ndom[j] = n_dom++;
        else ndom[j] = dense.emplace(ni.domain, n_dom).second ? n_dom++ : dense[ni.domain];
    }
    return n_dom;
}

// The spread walks need the ranked side table plus the live members grouped by domain: dense domain ids (one per label shared by
// live nodes, one per live node labelled RIO_NONE), the members sorted by (domain, bucket, index) with a running weight, and for the
// flat kernel the domain of every record in the class-sorted order build_tab gives the table, (inverse weight, node index).
void ensure_spread_tab(rio_placement *h) {
    if (h->spread_version[0] == h->tab_version && h->spread_version[1] == h->label_version) return;
    const uint32_t n_total = (uint32_t)h->nodes.size();
    std::vector<TrieMember> members;
    std::vector<uint32_t> live, ndom;
    const uint32_t n_dom = dense_domains(h, ndom);
    for (uint32_t j = 0; j < n_total; j++) {
        const NodeInfo &ni = h->nodes[j];
        if (!ni.live()) continue;
        members.push_back(TrieMember{ni.seed, j, ni.weight});
        live.push_back(j);
    }
    const TrieBlob blob = build_trie_blob(members, h->trie_bits);
    const uint32_t bits = blob.bits, nb = 1u << bits, n_live = (uint32_t)live.size();
    std::vector<uint32_t> bucket(n_total, 0);
    for (uint32_t j : live) bucket[j] = bits ? (uint32_t)(mix64(h->nodes[j].seed ^ kSaltPos) >> (64 - bits)) : 0u;
    std::vector<uint32_t> by_dom(live), by_class(live);
    std::sort(by_dom.begin(), by_dom.end(), [&](uint32_t a, uint32_t b) {
        return ndom[a] != ndom[b] ? ndom[a] < ndom[b] : bucket[a] != bucket[b] ? bucket[a] < bucket[b] : a < b;
    });
    std::stable_sort(by_class.begin(), by_class.end(), [&](uint32_t a, uint32_t b) { return inv_weight(h->nodes[a].weight) < inv_weight(h->nodes[b].weight); });
    auto al = [](size_t v) { return (v + 15) / 16 * 16; };
    SpreadTabDev sp{};
    sp.o_node = nb * 16u;
    sp.o_ndom = (uint32_t)(sp.o_node + al((size_t)n_total * 8));
    sp.o_pre = (uint32_t)(sp.o_ndom + al((size_t)n_total * 4));
    sp.o_mb = (uint32_t)(sp.o_pre + al(((size_t)n_live + 1) * 8));
    sp.o_dstart = (uint32_t)(sp.o_mb + al((size_t)n_live * 4));
    sp.trie_bytes = (uint32_t)(sp.o_dstart + al(((size_t)n_dom + 1) * 4));
    sp.n_members = n_live;
    sp.n_domains = n_dom;
    const size_t total = sp.trie_bytes + al((size_t)n_live * 4);
    h->spread_stage.assign(total, 0);
    unsigned char *st8 = h->spread_stage.data();
    memcpy(st8, blob.wsum.data(), (size_t)nb * 16);
    uint2 *node = reinterpret_cast<uint2 *>(st8 + sp.o_node);
    for (uint32_t j : live) node[j] = make_uint2(bucket[j], h->nodes[j].weight);
    memcpy(st8 + sp.o_ndom, ndom.data(), (size_t)n_total * 4);
    uint64_t *pre = reinterpret_cast<uint64_t *>(st8 + sp.o_pre);
    uint32_t *mb = reinterpret_cast<uint32_t *>(st8 + sp.o_mb), *dstart = reinterpret_cast<uint32_t *>(st8 + sp.o_dstart);
    uint32_t *pos_dom = reinterpret_cast<uint32_t *>(st8 + sp.trie_bytes);
    for (uint32_t q = 0; q < n_live; q++) {
        const uint32_t j = by_dom[q];
        pre[q + 1] = pre[q] + h->nodes[j].weight;
        mb[q] = bucket[j];
        dstart[ndom[j] + 1] = q + 1;
        pos_dom[q] = ndom[by_class[q]];
    }
    cudaStream_t st = h->stream;
    h->spread_dev.ensure(total, st);
    CUDA_TRY(cudaMemcpyAsync(h->spread_dev.p, st8, total, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    sp.base = h->spread_dev.as<unsigned char>();
    h->spread_tab = sp;
    h->spread_version[0] = h->tab_version;
    h->spread_version[1] = h->label_version;
}

// affinity dispatch: no live node fills the output with NONE; the tensor-core (wgmma) kernel for K == 16 (unless
// RIO_AFFINITY_VARIANT=ffma or the node set does not fit); else the CUDA cores
enum class AffinityPath { kNoLiveNode, kTensorCores, kCudaCores };
bool affinity_umma_wanted() {
    const char *v = getenv("RIO_AFFINITY_VARIANT");
    return !(v && v[0] == 'f');
}
// want_umma = false keeps K == 16 on the CUDA cores (an affinity resident set recorded there, DESIGN.md 3.15)
AffinityPath affinity_path(const rio_placement *h, bool want_umma = affinity_umma_wanted()) {
    if (!h->aff_live && h->K == 16 && h->tabs.tab.n_live == 0) return AffinityPath::kNoLiveNode;
    if (want_umma && h->K == 16 && h->aff_live && h->aff_pad <= affinity_umma_max_nodes()) return AffinityPath::kTensorCores;
    return AffinityPath::kCudaCores;
}

void run_affinity(rio_placement *h, const float *d_fobj, uint64_t n, uint32_t *d_out_idx, float *d_out_cost, uint32_t *d_counters, AffinityPath path) {
    if (!n) return;
    switch (path) {
        case AffinityPath::kNoLiveNode: launch_fill_u32(h->L(), d_out_idx, n, kNone); break;
        case AffinityPath::kTensorCores:
            CUDA_TRY(launch_assign_affinity_umma(h->L(), d_fobj, n, h->d_fnode_c.as<float>(), h->d_fnode_g.as<float>(), h->d_nidx_map.as<uint32_t>(), h->aff_live,
                                                 h->aff_pad, h->tabs.tab.n_total, d_out_idx, d_out_cost, d_counters));
            break;
        case AffinityPath::kCudaCores:
            launch_assign_affinity(h->L(), d_fobj, n, h->d_fnode.as<float>(), h->tabs.live, h->tabs.tab.n_total, h->K, d_out_idx, d_out_cost, d_counters);
            break;
    }
}

// The domain ids of the failure-domain affinity lists: without the HRW2 blob ensure_spread_tab builds, so the first call after a
// relabel costs one pass over the nodes and one small copy
void ensure_aff_dom(rio_placement *h) {
    if (h->aff_dom_version[0] == h->tab_version && h->aff_dom_version[1] == h->label_version) return;
    std::vector<uint32_t> ids;
    dense_domains(h, ids);
    const size_t n_total = ids.size();
    if (h->aff_pad) {   // the live nodes in node-index order, padded with kNone: the compacted positions of ensure_tab
        ids.reserve(n_total + h->aff_pad);
        for (size_t j = 0; j < n_total; j++)
            if (ids[j] != kNone) ids.push_back(ids[j]);
        ids.resize(n_total + h->aff_pad, kNone);
    }
    if (ids.empty()) ids.push_back(kNone);
    h->aff_dom.ensure(ids.size() * 4, h->stream);
    CUDA_TRY(cudaMemcpyAsync(h->aff_dom.p, ids.data(), ids.size() * 4, cudaMemcpyHostToDevice, h->stream));
    CUDA_TRY(cudaStreamSynchronize(h->stream));   // ids goes out of scope
    h->aff_dom_pos = n_total;
    h->aff_dom_version[0] = h->tab_version;
    h->aff_dom_version[1] = h->label_version;
}

// The n x ranks lists of `kind` (see ListKind) for the n keys or feature rows at `in` into d_out_idx, under the handle's policy.  The
// affinity kinds run on `path` (the batch calls pass affinity_path(h), so that rank 1 is run_affinity's answer; a resident set passes
// its recorded path), and their tensor-core pairs keep each object's groups or listed column positions in s_idx2 between the two
// passes.  A build without the kind's kernels refuses before anything is launched.
void run_lists(rio_placement *h, ListKind kind, const void *in, uint64_t n, uint32_t ranks, uint32_t *d_out_idx, AffinityPath path) {
    const uint64_t *d_keys = static_cast<const uint64_t *>(in);
    switch (kind) {
        case ListKind::kHash:
            if (!launch_assign_hrw_ranked || !launch_assign_trie_ranked)
                throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no ranked kernels (k_ranked.cu is not linked)"};
            ensure_tab(h);
            if (h->solver == RIO_SOLVER_HRW2) {
                ensure_rank_tab(h);
                launch_assign_trie_ranked(h->L(), d_keys, n, h->tabs.trie, h->rank_tab, ranks, d_out_idx);
            } else {
                launch_assign_hrw_ranked(h->L(), d_keys, n, h->tabs.tab, ranks, d_out_idx);
            }
            return;
        case ListKind::kSpread:
            if (!launch_assign_hrw_spread || !launch_assign_trie_spread)
                throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no spread kernels (k_spread.cu is not linked)"};
            ensure_tab(h);
            ensure_spread_tab(h);
            if (h->solver == RIO_SOLVER_HRW2) launch_assign_trie_spread(h->L(), d_keys, n, h->tabs.trie, h->spread_tab, ranks, d_out_idx);
            else launch_assign_hrw_spread(h->L(), d_keys, n, h->tabs.tab, h->spread_tab, ranks, d_out_idx);
            return;
        case ListKind::kAffinity:
            if (!launch_assign_affinity_ranked || !launch_assign_affinity_umma_ranked)
                throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no ranked affinity kernels (k_affinity_umma.cu / k_assign.cu are not linked)"};
            break;
        case ListKind::kAffinitySpread:
            if (!launch_assign_affinity_spread || !launch_assign_affinity_umma_spread)
                throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no failure-domain affinity kernels (k_affinity_spread.cuh launchers are not linked)"};
            break;
    }
    if (!n) return;   // an empty resident set: no list to compute, no domain table needed
    const float *d_fobj = static_cast<const float *>(in);
    const bool spread = kind == ListKind::kAffinitySpread;
    if (path == AffinityPath::kNoLiveNode) { launch_fill_u32(h->L(), d_out_idx, n * ranks, kNone); return; }
    if (spread) ensure_aff_dom(h);
    const uint32_t *ndom = h->aff_dom.as<uint32_t>();
    if (path == AffinityPath::kTensorCores) {
        h->s_idx2.ensure(n * affinity_ranked_groups(ranks) * 4, h->stream);
        if (spread)
            CUDA_TRY(launch_assign_affinity_umma_spread(h->L(), d_fobj, n, h->d_fnode_c.as<float>(), h->d_fnode_g.as<float>(), h->d_nidx_map.as<uint32_t>(),
                                                        ndom + h->aff_dom_pos, h->aff_live, h->aff_pad, ranks, h->s_idx2.as<uint32_t>(), d_out_idx));
        else
            CUDA_TRY(launch_assign_affinity_umma_ranked(h->L(), d_fobj, n, h->d_fnode_c.as<float>(), h->d_fnode_g.as<float>(), h->d_nidx_map.as<uint32_t>(),
                                                        h->aff_live, h->aff_pad, ranks, h->s_idx2.as<uint32_t>(), d_out_idx));
    } else if (spread) {
        launch_assign_affinity_spread(h->L(), d_fobj, n, h->d_fnode.as<float>(), h->tabs.live, h->tabs.tab.n_total, h->K, ndom, ranks, d_out_idx);
    } else {
        launch_assign_affinity_ranked(h->L(), d_fobj, n, h->d_fnode.as<float>(), h->tabs.live, h->tabs.tab.n_total, h->K, ranks, d_out_idx);
    }
}

// ---- caller buffers of the _dev calls (the alignment rules of buffer_align.cuh) ----------------------------------------------------------
bool aligned_to(const void *p, uint32_t align) { return ((uintptr_t)p & (align - 1)) == 0; }

// A _dev call refuses a buffer that is not naturally aligned for its element type, before it enqueues anything.
void require_natural(const void *p, uint32_t align, const char *name) {
    if (p) REQUIRE(aligned_to(p, align), std::string(name) + " is not aligned to its element size (" + std::to_string(align) + " bytes)");
}

// A caller's input the launcher reads in place if it starts at `align`; otherwise a copy of it in the handle's staging buffer `buf`,
// made on the stream.
template <class T>
const T *input_at(rio_placement *h, DevBuf &buf, const T *p, size_t count, uint32_t align) {
    if (aligned_to(p, align)) return p;
    buf.ensure(count * sizeof(T), h->stream);
    CUDA_TRY(cudaMemcpyAsync(buf.p, p, count * sizeof(T), cudaMemcpyDeviceToDevice, h->stream));
    return buf.as<const T>();
}

// Where the launcher writes a caller's output of `count` indices: the buffer itself if it starts at `align`, else the handle's staging
// buffer `buf`, which output_done then copies into the caller's buffer on the stream.  Staging buffers are reused by the next call
// only behind that copy, in stream order.
uint32_t *output_at(rio_placement *h, DevBuf &buf, uint32_t *p, size_t count, uint32_t align) {
    if (aligned_to(p, align)) return p;
    buf.ensure(count * 4, h->stream);
    return buf.as<uint32_t>();
}
void output_done(rio_placement *h, const uint32_t *written, uint32_t *p, size_t count) {
    if (written != p) CUDA_TRY(cudaMemcpyAsync(p, written, count * 4, cudaMemcpyDeviceToDevice, h->stream));
}

// The feature rows of an affinity _dev call where the launchers of `path` read them; the no-live-node fill reads none.  Every affinity
// kernel writes its indices one at a time, so the caller's output is used in place.
const float *affinity_input(rio_placement *h, const float *d_feats, uint64_t n, AffinityPath path) {
    return path == AffinityPath::kNoLiveNode ? d_feats : input_at(h, h->s_feats, d_feats, n * h->K, affinity_feats_align(h->K));
}

// The path of an affinity list batch of n rows, once the handle's K admits it, with the table current; the hash kinds take none
AffinityPath list_batch_path(rio_placement *h, ListKind kind, size_t n) {
    if (!is_affinity(kind)) return AffinityPath::kCudaCores;
    REQUIRE(h->K > 0, "assign with object features needs node features");
    REQUIRE(n <= SIZE_MAX / 4 / h->K, "n x K overflows");
    ensure_tab(h);
    return affinity_path(h);
}

// The host-buffer form of a list call: keys staged through s_keys or feature rows through s_feats, the n x ranks lists through s_idx
// back into out_idx, and the stream synchronised
void lists_from_host(rio_placement *h, ListKind kind, const void *in, size_t n, uint32_t ranks, uint32_t *out_idx) {
    check_ranked_args(n, ranks);
    if (!n) return;
    REQUIRE(in && out_idx, "null buffer");
    const AffinityPath path = list_batch_path(h, kind, n);
    DevBuf &d_in = is_affinity(kind) ? h->s_feats : h->s_keys;
    const size_t in_bytes = is_affinity(kind) ? n * h->K * 4 : n * 8;
    cudaStream_t st = h->stream;
    d_in.ensure(in_bytes, st);
    h->s_idx.ensure(n * ranks * 4, st);
    CUDA_TRY(cudaMemcpyAsync(d_in.p, in, in_bytes, cudaMemcpyHostToDevice, st));
    run_lists(h, kind, d_in.p, n, ranks, h->s_idx.as<uint32_t>(), path);
    CUDA_TRY(cudaMemcpyAsync(out_idx, h->s_idx.p, n * ranks * 4, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
}

// The device-buffer form: every list kernel reads keys and writes list entries one at a time, so those buffers are used in place;
// feature rows are read where affinity_input puts them
void lists_from_device(rio_placement *h, ListKind kind, const void *d_in, size_t n, uint32_t ranks, uint32_t *d_out_idx) {
    check_ranked_args(n, ranks);
    if (!n) return;
    REQUIRE(d_in && d_out_idx, "null buffer");
    if (is_affinity(kind)) require_natural(d_in, 4, "d_obj_feats");
    else require_natural(d_in, 8, "d_keys");
    require_natural(d_out_idx, 4, "d_out_idx");
    const AffinityPath path = list_batch_path(h, kind, n);
    if (is_affinity(kind)) d_in = affinity_input(h, static_cast<const float *>(d_in), n, path);
    run_lists(h, kind, d_in, n, ranks, d_out_idx, path);
}

uint32_t capacity_of(uint64_t n_total, uint32_t w, uint64_t w_sum, uint32_t num, uint32_t den) {
    if (!w || !w_sum || !den) return 0;
    unsigned __int128 a = (unsigned __int128)num * n_total * w, b = (unsigned __int128)den * w_sum;
    unsigned __int128 q = (a + b - 1) / b;
    return q > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)q;
}

// host keys -> device, chunk-pipelined on three streams so H2D, the score grid and D2H overlap (e2e path)
void assign_host_pipelined(rio_placement *h, const uint64_t *keys, const float *feats, size_t n, uint32_t *out, uint32_t *d_counters = nullptr,
                           bool final_sync = true) {
    ensure_tab(h);
    if (feats) REQUIRE(h->K > 0, "assign with object features needs node features (set_nodes feats)");
    // chunks of two full kernel waves (sm_count x 3 CTAs x threads x 5 objects each): whole waves leave no tail, small chunks keep the
    // pipeline fill/drain (first H2D, last D2H) short
    // HRW2 walks a chunk in microseconds, so PCIe is the only clock: small chunks (512 Ki objects = 4 MiB in, 2 MiB out) keep the
    // pipeline's fill (first H2D) and drain (last D2H) at ~0.1 ms of an 80 MB transfer
    const size_t chunk = feats ? (size_t)(1u << 20)
                               : (h->solver == RIO_SOLVER_HRW2 ? (size_t)(1u << 19) : (size_t)(2 * assign_wave_objects(h->sm_count)));
    if (!feats) h->s_keys.ensure(n * 8, h->stream);
    h->s_idx.ensure(n * 4, h->stream);
    if (feats) h->s_feats.ensure(n * (size_t)h->K * 4, h->stream);
    CUDA_TRY(cudaEventRecord(h->ev_pipe[0], h->stream));          // buffers (re)allocated on the main stream
    CUDA_TRY(cudaStreamWaitEvent(h->h2d_stream, h->ev_pipe[0], 0));
    CUDA_TRY(cudaStreamWaitEvent(h->d2h_stream, h->ev_pipe[0], 0));
    for (size_t lo = 0; lo < n; lo += chunk) {
        const size_t m = std::min(chunk, n - lo);
        if (!feats) CUDA_TRY(cudaMemcpyAsync(h->s_keys.as<uint64_t>() + lo, keys + lo, m * 8, cudaMemcpyHostToDevice, h->h2d_stream));   // keys may be NULL with feats
        if (feats) CUDA_TRY(cudaMemcpyAsync(h->s_feats.as<float>() + lo * h->K, feats + lo * h->K, m * (size_t)h->K * 4, cudaMemcpyHostToDevice, h->h2d_stream));
        CUDA_TRY(cudaEventRecord(h->ev_pipe[1], h->h2d_stream));
        CUDA_TRY(cudaStreamWaitEvent(h->stream, h->ev_pipe[1], 0));
        if (feats)
            run_affinity(h, h->s_feats.as<float>() + lo * h->K, m, h->s_idx.as<uint32_t>() + lo, nullptr, nullptr, affinity_path(h));
        else
            run_assign(h, h->solver, h->tabs, h->s_keys.as<uint64_t>() + lo, m, h->s_idx.as<uint32_t>() + lo, d_counters, nullptr, 0);
        CUDA_TRY(cudaEventRecord(h->ev_pipe[2], h->stream));
        CUDA_TRY(cudaStreamWaitEvent(h->d2h_stream, h->ev_pipe[2], 0));
        CUDA_TRY(cudaMemcpyAsync(out + lo, h->s_idx.as<uint32_t>() + lo, m * 4, cudaMemcpyDeviceToHost, h->d2h_stream));
    }
    if (!final_sync) return;   // the caller still has work for the main stream (capacity check) while the last D2H is in flight
    CUDA_TRY(cudaEventRecord(h->ev_pipe[3], h->d2h_stream));
    CUDA_TRY(cudaStreamWaitEvent(h->stream, h->ev_pipe[3], 0));
    CUDA_TRY(cudaStreamSynchronize(h->stream));
}

// ---- bounded-load rounds (DESIGN.md 3.5) over a device-resident (keys, idx, counters) triple ------------------------------------
// Pass 0 = plain assignment with the fused histogram.  The counter exchange (peer memory, world > 1) and the capacity check run on
// the device -- under HRW2 in the last CTA of the walk kernel itself, otherwise as one small kernel behind it -- and leave two
// words in mapped pinned memory; the host reads those after the stream synchronises.  Only when a node is over capacity (rare at
// the default factor 1.25) do the thresholds get used by the spill selection and the closed set come back to the host for the
// masked table of the next pass.
struct BoundedDev { uint32_t *cap, *glob, *thr, *closed_epoch, *ticket; uint8_t *over; };
BoundedDev bounded_layout(rio_placement *h, BoundedState &bs, uint32_t M) {
    const size_t m = std::max(M, 1u);
    const size_t need = m * 17 + 64;
    if (need > bs.buf.bytes) {
        bs.buf.ensure(need, h->stream);
        CUDA_TRY(cudaMemsetAsync(bs.buf.p, 0, bs.buf.bytes, h->stream));   // closed epochs and the ticket start at 0
        bs.epoch = 0;
        bs.cap_key[0] = ~0ull;
    }
    if (!bs.h_flags) {
        CUDA_TRY(cudaHostAlloc(reinterpret_cast<void **>(&bs.h_flags), 16, cudaHostAllocMapped));
        memset(bs.h_flags, 0, 16);
        CUDA_TRY(cudaEventCreateWithFlags(&bs.ev, cudaEventDisableTiming));
    }
    BoundedDev b;
    b.ticket = bs.buf.as<uint32_t>();          // 16 words reserved
    b.cap = b.ticket + 16;
    b.glob = b.cap + m;
    b.thr = b.glob + m;
    b.closed_epoch = b.thr + m;
    b.over = reinterpret_cast<uint8_t *>(b.closed_epoch + m);
    return b;
}

BoundedTail make_tail(rio_placement *h, BoundedState &bs, const BoundedDev &b, uint32_t M, uint32_t *next_zero, bool peer_exchange) {
    BoundedTail t{};
    t.enabled = 1;
    t.M = M;
    t.ticket = b.ticket;
    t.next_zero = next_zero;
    t.world = 1;
    if (peer_exchange) {
        for (int p = 0; p < h->world && p < 16; p++) t.peers.win[p] = h->xchg_peer[p];
        t.rank = (uint32_t)h->rank; t.world = (uint32_t)h->world; t.max_nodes = h->xchg_nodes; t.xchg_epoch = ++h->xchg_epoch;
    }
    t.glob = b.glob; t.cap = b.cap; t.state = h->tabs.state; t.closed_epoch = b.closed_epoch; t.call_epoch = bs.epoch;
    t.thr = b.thr; t.over = b.over;
    uint32_t *flags_dev = nullptr;
    CUDA_TRY(cudaHostGetDevicePointer(reinterpret_cast<void **>(&flags_dev), bs.h_flags, 0));
    t.host_flags = flags_dev;
    t.flag_seq = ++bs.flag_seq;
    return t;
}

// The check's two words arrive in mapped pinned memory followed by a sequence number.  Polling that number costs ~1 us after the
// write lands; a stream synchronise costs a driver wake-up (5-8 us) on top of a 60 us pass.  Everything the pass wrote to HBM is
// ordered before the flag, later work on the stream is ordered behind the kernel as usual.  Falls back to a synchronise (which
// also surfaces a failed kernel) if the number does not show up.
std::pair<uint32_t, uint32_t> read_flags(rio_placement *h, BoundedState &bs) {
    const volatile uint32_t *flags = bs.h_flags;
    const auto t_end = std::chrono::steady_clock::now() + std::chrono::milliseconds(20);
    while (flags[2] != bs.flag_seq) {
        if (std::chrono::steady_clock::now() > t_end) {
            // slow path (a peer rank is late, first use of the peer mappings, ...): block on both streams the check may be on;
            // this also surfaces a failed kernel as a CUDA error instead of a missing report
            CUDA_TRY(cudaStreamSynchronize(h->stream));
            if (h->aux_stream) CUDA_TRY(cudaStreamSynchronize(h->aux_stream));
            REQUIRE(flags[2] == bs.flag_seq, "capacity check did not report (internal error)");
            break;
        }
#if defined(__x86_64__)
        __builtin_ia32_pause();
#endif
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    return {flags[0], flags[1]};
}

// enqueue one exchange + check as its own launch (the result is picked up later with read_flags)
void launch_check(rio_placement *h, BoundedState &bs, const uint32_t *d_local, const BoundedDev &b, uint32_t M, uint32_t *next_zero, cudaStream_t st) {
    const bool p2p = h->world > 1 && h->xchg_ready && M <= h->xchg_nodes;
    const uint32_t *src = d_local;
    Launch L = h->L();
    L.stream = st;
    if (!p2p && h->world > 1 && h->comm) {   // portable path: NCCL all-gather + sum, then the check alone
        h->s_gather.ensure((size_t)M * 4 * h->world, h->stream);
        if (st != h->stream) { CUDA_TRY(cudaEventRecord(h->ev_pipe[4], h->stream)); CUDA_TRY(cudaStreamWaitEvent(st, h->ev_pipe[4], 0)); }   // the gather buffer may just have been allocated
        NCCL_TRY(g_nccl.AllGather(d_local, h->s_gather.p, M, kNcclUint32, h->comm, st));
        launch_sum_gathered(L, h->s_gather.as<uint32_t>(), (uint32_t)h->world, M, b.glob);
        src = b.glob;
    }
    launch_exchange_check(L, src, make_tail(h, bs, b, M, next_zero, p2p));
}

// First half of a bounded call: capacities, pass 0 and its check are enqueued; nothing is waited for (except the one-off
// capacity upload when the table or the factor changed).
// pipelined: the caller keeps several calls in flight (rio_cuda_set_assign_bounded_begin): the check then runs as its own one-CTA
// kernel on the auxiliary stream behind an event, so the next set's walk starts the moment this one ends instead of waiting for the
// ~8 us the last CTA needs for fence + ticket + check + the PCIe write.  One call at a time: the check rides in the walk kernel's
// last CTA (one launch, lowest latency).
void bounded_begin(rio_placement *h, BoundedState &bs, const uint64_t *d_keys, uint64_t n, uint32_t *d_idx, uint32_t *d_counters, uint32_t M,
                   uint64_t n_total_objs, uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds, bool first_pass_done, bool counters_zeroed, uint32_t *next_zero,
                   bool pipelined = false) {
    cudaStream_t st = h->stream;
    REQUIRE(!bs.active, "a bounded call is already in flight on this set (call _end first)");
    const BoundedDev b = bounded_layout(h, bs, M);
    const uint64_t key[4] = {n_total_objs, ((uint64_t)cap_num << 32) | cap_den, h->tab_version, M};
    if (memcmp(key, bs.cap_key, sizeof key) != 0) {   // capacities depend only on (N, factor, live weights): upload once per table
        uint64_t W = 0;
        for (auto &ni : h->nodes) if (ni.live()) W += ni.weight;
        std::vector<uint32_t> cap(std::max(M, 1u), 0);
        for (uint32_t j = 0; j < M && j < h->nodes.size(); j++) if (h->nodes[j].live()) cap[j] = capacity_of(n_total_objs, h->nodes[j].weight, W, cap_num, cap_den);
        CUDA_TRY(cudaMemcpyAsync(b.cap, cap.data(), (size_t)std::max(M, 1u) * 4, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        memcpy(bs.cap_key, key, sizeof key);
    }
    if (++bs.epoch == 0) {   // the closed set of a call is "closed_epoch[j] == this call's epoch": no memset per call
        CUDA_TRY(cudaMemsetAsync(b.closed_epoch, 0, (size_t)std::max(M, 1u) * 4, st));
        bs.epoch = 1;
    }
    bool fused = false;
    if (!first_pass_done) {
        if (!counters_zeroed) CUDA_TRY(cudaMemsetAsync(d_counters, 0, (size_t)std::max(M, 1u) * 4, st));
        const bool p2p = h->world > 1 && h->xchg_ready && M <= h->xchg_nodes;
        if (!pipelined && max_rounds > 1 && h->solver == RIO_SOLVER_HRW2 && (h->world == 1 || p2p)) {
            order_behind_aux_checks(h);
            const BoundedTail t = make_tail(h, bs, b, M, next_zero, p2p);   // walk + histogram + exchange + check: ONE launch
            launch_assign_trie(h->L(), d_keys, n, h->tabs.trie, d_idx, d_counters, nullptr, 0, h->tabs.tab.n_total, &t);
            fused = true;
        } else {
            // pipelined: five walk CTAs per SM leave no room for the 256-thread check kernel of the previous pass, which then takes
            // the slot of one of THIS pass's CTAs at the kernel boundary and delays it; one spare slot on the machine avoids that
            static const int spare = [] { const char *e = getenv("RIO_TRIE_SPARE"); return e ? atoi(e) : 1; }();
            struct SpareScope { int &v; ~SpareScope() { v = 0; } } scope{h->walk_spare};   // also reset when the launch throws
            h->walk_spare = (pipelined && max_rounds > 1) ? spare : 0;
            run_assign(h, h->solver, h->tabs, d_keys, n, d_idx, d_counters, nullptr, 0);
        }
    }
    if (!fused && max_rounds > 1) {
        if (pipelined) {
            CUDA_TRY(cudaEventRecord(bs.ev, st));
            CUDA_TRY(cudaStreamWaitEvent(h->aux_stream, bs.ev, 0));
            launch_check(h, bs, d_counters, b, M, next_zero, h->aux_stream);
            CUDA_TRY(cudaEventRecord(h->ev_aux, h->aux_stream));
            h->aux_used = true;
        } else {
            order_behind_aux_checks(h);
            launch_check(h, bs, d_counters, b, M, next_zero, st);
        }
    }
    bs.active = true;
    bs.n_total_objs = n_total_objs; bs.max_rounds = max_rounds; bs.M = M;
    bs.live_sig = h->live_sig;   // of the table pass 0 ran on (every caller went through ensure_tab)
}

// Second half: wait for the check (two words in mapped memory), run the spill rounds it asks for.  Returns the passes run.
// select(b, round) appends the spilling objects to d_sel (counted at S_NSEL) and takes them off d_counters: launch_select_spill for the
// object counts of 3.5, the weighted selection of 3.19 for loads.  replace(closed, nsel) re-places the nsel objects of d_sel over live
// minus closed and adds them back: hash_replace for the hash policy, the affinity launch of the call's path for 3.16.
template <class Select, class Replace>
uint32_t bounded_end(rio_placement *h, BoundedState &bs, uint32_t *d_counters, Select &&select, Replace &&replace) {
    REQUIRE(bs.active, "no bounded call in flight on this set");
    bs.active = false;
    cudaStream_t st = h->stream;
    const uint32_t M = bs.M;
    const BoundedDev b = bounded_layout(h, bs, M);
    uint32_t passes = 1;
    for (uint32_t r = 1; r < bs.max_rounds; r++) {
        const auto [any, open] = read_flags(h, bs);                  // the one collective of the pass has happened on the device
        if (!any || !open) break;
        // A spill round re-places objects over "live minus closed" with the capacities, counters and closed set of the table pass 0
        // ran on.  If the live set changed between _begin and _end (a join / leave / weight change by another call) those no
        // longer describe the same cluster -- and a node that joined since has no counter slot: refuse, the caller runs the call again.
        REQUIRE(live_signature(h) == bs.live_sig, "the live node set changed between the two halves of a bounded call: run it again");
        zero_scalar(h, S_NSEL);
        select(b, r);
        std::vector<uint32_t> ce(M, 0);
        CUDA_TRY(cudaMemcpyAsync(ce.data(), b.closed_epoch, (size_t)M * 4, cudaMemcpyDeviceToHost, st));
        const uint64_t nsel = read_scalar(h, S_NSEL);
        std::vector<uint8_t> closed(M, 0);
        for (uint32_t j = 0; j < M; j++) closed[j] = ce[j] == bs.epoch;
        replace(closed, nsel);
        passes++;
        if (r + 1 < bs.max_rounds) { order_behind_aux_checks(h); launch_check(h, bs, d_counters, b, M, nullptr, st); }
    }
    return passes;
}

// the rounds over object counts (3.5, 3.16, 3.17)
template <class Replace>
uint32_t bounded_end(rio_placement *h, BoundedState &bs, const uint64_t *d_keys, uint64_t n, uint32_t *d_idx, uint32_t *d_counters, uint32_t *d_sel,
                     Replace &&replace) {
    return bounded_end(h, bs, d_counters, [&](const BoundedDev &b, uint32_t r) {
        launch_select_spill(h->L(), d_keys, d_idx, n, b.thr, b.over, r, d_sel, h->d_scalars + S_NSEL, d_counters);
    }, replace);
}

// the spill rounds of 3.5: the handle's policy over the masked table
auto hash_replace(rio_placement *h, const uint64_t *d_keys, uint64_t n, uint32_t *d_idx, uint32_t *d_counters, uint32_t *d_sel) {
    return [=](const std::vector<uint8_t> &closed, uint64_t nsel) {
        build_tab(h, h->tabs_masked, &closed);
        if (nsel) run_assign(h, h->solver, h->tabs_masked, d_keys, n, d_idx, d_counters, d_sel, nsel);
    };
}

// ---- bounded-load rounds under the affinity cost (DESIGN.md 3.16) ----------------------------------------------------------------
void require_bounded_affinity_kernels() {
    if (!launch_scatter_idx || !launch_gather_rows)
        throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no bounded affinity kernels (k_affinity_bounded.cuh launchers are not linked)"};
}

// Re-places the nsel objects of d_sel on `path`, adding them to d_counters: with closed (a bounded round) over live minus closed -- the
// CUDA-core kernel with the masked table's live flags, or the tensor-core kernel over operands compacted without the closed nodes --,
// without (the S1 objects of 3.17) over the live set, as run_affinity places them.  The rows go through s_rows, the new nodes through
// s_idx2, and k_scatter_idx writes them into d_idx.
void affinity_replace(rio_placement *h, AffinityPath path, const std::vector<uint8_t> *closed, const float *d_feats, const uint32_t *d_sel, uint64_t nsel,
                      uint32_t *d_idx, uint32_t *d_counters) {
    const uint32_t K = h->K, n_total = h->tabs.tab.n_total;
    if (closed) {
        if (path == AffinityPath::kTensorCores) build_aff_operands(h, closed, h->d_fnode_cm, h->d_fnode_gm, h->d_nidx_map_m, h->aff_live_m, h->aff_pad_m);
        else build_tab(h, h->tabs_masked, closed);
    }
    if (!nsel) return;
    h->s_rows.ensure(nsel * K * 4, h->stream);
    h->s_idx2.ensure(nsel * 4, h->stream);
    uint32_t *d_new = h->s_idx2.as<uint32_t>();
    launch_gather_rows(h->L(), d_feats, K, d_sel, nsel, h->s_rows.as<float>());
    if (!closed)
        run_affinity(h, h->s_rows.as<float>(), nsel, d_new, nullptr, d_counters, path);
    else if (path == AffinityPath::kCudaCores)
        launch_assign_affinity(h->L(), h->s_rows.as<float>(), nsel, h->d_fnode.as<float>(), h->tabs_masked.live, n_total, K, d_new, nullptr, d_counters);
    else if (path == AffinityPath::kTensorCores && h->aff_live_m)
        CUDA_TRY(launch_assign_affinity_umma(h->L(), h->s_rows.as<float>(), nsel, h->d_fnode_cm.as<float>(), h->d_fnode_gm.as<float>(),
                                             h->d_nidx_map_m.as<uint32_t>(), h->aff_live_m, h->aff_pad_m, n_total, d_new, nullptr, d_counters));
    else   // no live node is open (only an active node of weight 0 kept the round going)
        launch_fill_u32(h->L(), d_new, nsel, kNone);
    launch_scatter_idx(h->L(), d_new, d_sel, nsel, d_idx);
}

// Pass 0 is run_affinity with the counters on `path` (affinity_path() now), then the rounds of 3.5, whose spilled objects
// affinity_replace puts back on the same path over live minus closed.
uint32_t bounded_affinity(rio_placement *h, BoundedState &bs, const uint64_t *d_keys, const float *d_feats, uint64_t n, uint32_t *d_idx, uint32_t *d_counters,
                          uint32_t M, uint32_t *d_sel, uint64_t n_total_objs, uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds, AffinityPath path) {
    CUDA_TRY(cudaMemsetAsync(d_counters, 0, (size_t)std::max(M, 1u) * 4, h->stream));
    run_affinity(h, d_feats, n, d_idx, nullptr, d_counters, path);
    bounded_begin(h, bs, d_keys, n, d_idx, d_counters, M, n_total_objs, cap_num, cap_den, max_rounds, true, true, nullptr);
    return bounded_end(h, bs, d_keys, n, d_idx, d_counters, d_sel, [&](const std::vector<uint8_t> &closed, uint64_t nsel) {
        affinity_replace(h, path, &closed, d_feats, d_sel, nsel, d_idx, d_counters);
    });
}

// ---- bounded-load rounds over object weights (DESIGN.md 3.19) -------------------------------------------------------------------
void require_weighted_kernels() {
    if (!launch_weight_sum || !launch_load_histogram || !launch_select_spill_weighted || !launch_add_loads_sel)
        throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no weighted bounded kernels (k_bounded_weighted.cuh launchers are not linked)"};
}

constexpr uint64_t kMaxLoad = 0xFFFFFFFFull;   // loads are u32 sums

// the local weight sum of d_w[0..n) (nullptr: n); a device column costs one 8-byte readback
uint64_t local_weight_sum(rio_placement *h, const uint32_t *d_w, uint64_t n) {
    if (!d_w || !n) return n;
    zero_scalar(h, S_WSUM);
    launch_weight_sum(h->L(), d_w, n, h->d_scalars + S_WSUM);
    return read_scalar(h, S_WSUM);
}

// The weight sum of every rank's shard: with world > 1 one exchange of the counter path (collective; every rank calls it in the same
// order), the u64 sums cut into four 16-bit pieces so that the u32 sum of each piece over any world size up to 2^16 cannot wrap
uint64_t global_weight_sum(rio_placement *h, uint64_t local) {
    if (h->world <= 1) return local;
    uint32_t piece[8] = {};
    for (int k = 0; k < 4; k++) piece[k] = (uint32_t)(local >> (16 * k)) & 0xFFFFu;
    h->s_misc.ensure(sizeof piece, h->stream);
    uint32_t *d = h->s_misc.as<uint32_t>();
    CUDA_TRY(cudaMemcpyAsync(d, piece, 16, cudaMemcpyHostToDevice, h->stream));
    exchange_counters(h, d, d + 4, 4);
    CUDA_TRY(cudaMemcpyAsync(piece + 4, d + 4, 16, cudaMemcpyDeviceToHost, h->stream));
    CUDA_TRY(cudaStreamSynchronize(h->stream));
    uint64_t sum = 0;
    for (int k = 0; k < 4; k++) sum += (uint64_t)piece[4 + k] << (16 * k);
    return sum;
}

// The load total L of a weighted call from the global weight sum: load_total, or that sum when it is 0, refused where a u32 load could
// overflow.  Every rank decides from the same numbers, so a refusal here is collective.
uint64_t weighted_load_total(uint64_t global, uint64_t load_total) {
    REQUIRE(global <= kMaxLoad, "the object weights of all ranks sum past 2^32-1 (loads are u32)");
    REQUIRE(load_total <= kMaxLoad, "load_total past 2^32-1 (loads are u32)");
    if (!load_total) return global;
    REQUIRE(load_total >= global, "load_total is below the weight sum of all ranks");
    return load_total;
}

// The loads of the assignment in d_idx, then the rounds of 3.5 on d_loads from it: a spill takes its weight off its node, a re-placed
// object (counters = nullptr) adds it to its new one -- by the hash policy, or by affinity on `path`.  d_w == nullptr: every weight is 1.
uint32_t weighted_rounds(rio_placement *h, BoundedState &bs, const uint64_t *d_keys, const float *d_feats, const uint32_t *d_w, uint64_t n, uint32_t *d_idx,
                         uint32_t *d_loads, uint32_t M, uint32_t *d_sel, uint64_t load_total, uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds,
                         bool affinity, AffinityPath path) {
    CUDA_TRY(cudaMemsetAsync(d_loads, 0, (size_t)std::max(M, 1u) * 4, h->stream));
    launch_load_histogram(h->L(), d_idx, d_w, n, d_loads, M);
    bounded_begin(h, bs, d_keys, n, d_idx, d_loads, M, load_total, cap_num, cap_den, max_rounds, true, true, nullptr);
    const auto hash = hash_replace(h, d_keys, n, d_idx, nullptr, d_sel);
    return bounded_end(h, bs, d_loads,
                       [&](const BoundedDev &b, uint32_t r) {
                           launch_select_spill_weighted(h->L(), d_keys, d_idx, d_w, n, b.thr, b.over, r, d_sel, h->d_scalars + S_NSEL, d_loads);
                       },
                       [&](const std::vector<uint8_t> &closed, uint64_t nsel) {
                           if (affinity) affinity_replace(h, path, &closed, d_feats, d_sel, nsel, d_idx, nullptr);
                           else hash(closed, nsel);
                           launch_add_loads_sel(h->L(), d_sel, nsel, d_idx, d_w, d_loads, M);
                       });
}

// Pass 0 is the plain assignment (run_assign, or run_affinity on `path`) without counters, then the weighted rounds from its result.
// The set call and the host-buffer call both come here.
uint32_t bounded_weighted(rio_placement *h, BoundedState &bs, const uint64_t *d_keys, const float *d_feats, const uint32_t *d_w, uint64_t n, uint32_t *d_idx,
                          uint32_t *d_loads, uint32_t M, uint32_t *d_sel, uint64_t load_total, uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds,
                          bool affinity, AffinityPath path) {
    if (affinity) run_affinity(h, d_feats, n, d_idx, nullptr, nullptr, path);
    else run_assign(h, h->solver, h->tabs, d_keys, n, d_idx, nullptr, nullptr, 0);
    return weighted_rounds(h, bs, d_keys, d_feats, d_w, n, d_idx, d_loads, M, d_sel, load_total, cap_num, cap_den, max_rounds, affinity, path);
}

template <class F>
rio_status guarded(rio_placement *h, F &&f) {
    try {
        if (h) {
            std::lock_guard<std::mutex> g(h->mu);
            use_device(h);
            f();
            // a failed launch (bad configuration, wrong architecture) is not reported by the later synchronize/memcpy calls
            const cudaError_t le = cudaGetLastError();
            if (le != cudaSuccess) throw RioError{RIO_ERR_UPSTREAM, std::string("kernel launch failed: ") + cudaGetErrorString(le)};
        } else {
            f();
        }
        return RIO_OK;
    } catch (const RioError &e) {
        g_last_error = e.msg;
        return e.code;
    } catch (const std::exception &e) {
        g_last_error = e.what();
        return RIO_ERR_UNKNOWN;
    } catch (...) {
        g_last_error = "unknown C++ exception";
        return RIO_ERR_UNKNOWN;
    }
}

void set_ensure_counters(rio_objset *s) {
    rio_placement *h = s->h;
    const uint32_t n_total = (uint32_t)h->nodes.size();
    if (s->counters_n != n_total || !s->counters.p) {
        DevBuf nb;
        nb.ensure((size_t)(n_total ? n_total : 1) * 4, h->stream);
        CUDA_TRY(cudaMemsetAsync(nb.p, 0, nb.bytes, h->stream));
        if (s->counters.p && s->counters_n)
            CUDA_TRY(cudaMemcpyAsync(nb.p, s->counters.p, (size_t)std::min(s->counters_n, n_total) * 4, cudaMemcpyDeviceToDevice, h->stream));
        s->counters.release(h->stream);
        s->counters = nb;
        s->counters_n = n_total;
        s->counters_alt.release(h->stream);
        s->counters_alt.ensure(nb.bytes, h->stream);
        s->alt_zero = false;
    }
}

// every per-node counter of the set to 0, on the handle's stream, before a pass rebuilds them
void set_zero_counters(rio_objset *s) {
    rio_placement *h = s->h;
    CUDA_TRY(cudaMemsetAsync(s->counters.p, 0, (size_t)std::max(s->counters_n, 1u) * 4, h->stream));
}

// the plain kind after an affinity argmin on `path` (DESIGN.md 3.18); with no live node, the path the handle would take for K == 16,
// as record_affinity decides it
void record_plain_affinity(rio_objset *s, AffinityPath path) {
    s->plain_aff = true;
    s->plain_tensor = path == AffinityPath::kTensorCores || (path == AffinityPath::kNoLiveNode && affinity_umma_wanted());
}

}  // namespace

// =====================================================================================================================
extern "C" {

uint32_t rio_cuda_abi_version(void) { return RIO_ABI_VERSION; }

const char *rio_cuda_last_error(rio_placement *) { return g_last_error.c_str(); }

rio_status rio_cuda_create(const rio_config *cfg, rio_placement **out) {
    if (!out) { g_last_error = "out is NULL"; return RIO_ERR_UNKNOWN; }
    *out = nullptr;
    rio_placement *h = nullptr;
    try {
        int ndev = 0;
        cudaError_t e = cudaGetDeviceCount(&ndev);
        if (e != cudaSuccess || ndev == 0)
            throw RioError{RIO_ERR_UPSTREAM, std::string("no CUDA device available (") + cudaGetErrorString(e) + "); librio_cuda has no CPU fallback"};
        h = new rio_placement();
        int dev = cfg && cfg->struct_size >= sizeof(rio_config) ? cfg->device : -1;
        if (dev < 0) CUDA_TRY(cudaGetDevice(&dev));
        REQUIRE(dev < ndev, "device ordinal out of range");
        h->device = dev;
        CUDA_TRY(cudaSetDevice(dev));
        cudaDeviceProp prop;
        CUDA_TRY(cudaGetDeviceProperties(&prop, dev));
        h->sm_count = prop.multiProcessorCount;
        h->hbm = prop.totalGlobalMem;
        h->devname = prop.name;
        trie_upload_level_constants(dev);
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        CUDA_TRY(cudaStreamCreateWithFlags(&h->h2d_stream, cudaStreamNonBlocking));
        CUDA_TRY(cudaStreamCreateWithFlags(&h->d2h_stream, cudaStreamNonBlocking));
        {   // highest priority: its one-CTA kernels must not queue behind the next set's walk
            int lo_prio = 0, hi_prio = 0;
            CUDA_TRY(cudaDeviceGetStreamPriorityRange(&lo_prio, &hi_prio));
            CUDA_TRY(cudaStreamCreateWithPriority(&h->aux_stream, cudaStreamNonBlocking, hi_prio));
        }
        for (auto &ev : h->events) CUDA_TRY(cudaEventCreate(&ev));
        for (auto &ev : h->ev_pipe) CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        CUDA_TRY(cudaEventCreateWithFlags(&h->ev_aux, cudaEventDisableTiming));
        // keep freed blocks in the pool: the scratch buffers are re-used every call
        cudaMemPool_t pool;
        CUDA_TRY(cudaDeviceGetDefaultMemPool(&pool, dev));
        uint64_t thresh = ~0ull;
        CUDA_TRY(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh));
        void *sc = nullptr;
        CUDA_TRY(cudaMalloc(&sc, (S_COUNT + 1) * 8));
        CUDA_TRY(cudaMemset(sc, 0, (S_COUNT + 1) * 8));
        h->d_scalars = reinterpret_cast<unsigned long long *>(sc);
        CUDA_TRY(cudaHostAlloc(reinterpret_cast<void **>(&h->h_scalars), (S_COUNT + 1) * 8, cudaHostAllocMapped));   // S_FLAGS is written by the device
        memset(h->h_scalars, 0, (S_COUNT + 1) * 8);
        uint64_t cap = cfg && cfg->struct_size >= sizeof(rio_config) && cfg->directory_capacity ? cfg->directory_capacity : (1ull << 16);
        cap = pow2_at_least(std::max<uint64_t>(cap, 1024));
        dir_alloc(h, cap, h->dir);
        h->dir_cap = cap;
        CUDA_TRY(cudaStreamSynchronize(h->stream));
        *out = h;
        return RIO_OK;
    } catch (const RioError &e) {
        g_last_error = e.msg;
        delete h;
        return e.code;
    } catch (...) {
        g_last_error = "unknown error in rio_cuda_create";
        delete h;
        return RIO_ERR_UNKNOWN;
    }
}

void rio_cuda_destroy(rio_placement *h) {
    if (!h) return;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    if (h->aux_stream) cudaStreamSynchronize(h->aux_stream);
    if (h->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(h->comm);
    if (h->xchg_mine) {
        for (int p = 0; p < h->world && p < 16; p++)
            if (h->xchg_ready && p != h->rank && h->xchg_peer[p]) cudaIpcCloseMemHandle(h->xchg_peer[p]);
        cudaFree(h->xchg_mine);
    }
    for (TabBufs *tb : {&h->tabs, &h->tabs_masked}) if (tb->stage) cudaFreeHost(tb->stage);
    DevBuf *bufs[] = {&h->tabs.dev, &h->tabs_masked.dev, &h->d_fnode, &h->d_fnode_c, &h->d_fnode_g, &h->d_nidx_map, &h->d_fnode_cm, &h->d_fnode_gm, &h->d_nidx_map_m, &h->s_keys, &h->s_idx, &h->s_idx2, &h->s_sel, &h->s_slots, &h->s_keys2, &h->s_feats,
                      &h->s_packed, &h->s_offsets, &h->s_cost, &h->s_misc, &h->s_flush, &h->s_gather, &h->s_rows, &h->s_churn, &h->s_commit, &h->s_manifest, &h->s_weights, &h->rank_dev, &h->spread_dev, &h->aff_dom};
    h->bs.release(h->stream);
    for (DevBuf *b : bufs) b->release(h->stream);
    if (h->dir.slots) cudaFreeAsync(h->dir.slots, h->stream);
    cudaStreamSynchronize(h->stream);
    if (h->d_scalars) cudaFree(h->d_scalars);
    if (h->h_scalars) cudaFreeHost(h->h_scalars);
    for (auto &ev : h->events) if (ev) cudaEventDestroy(ev);
    for (auto &ev : h->ev_pipe) if (ev) cudaEventDestroy(ev);
    if (h->ev_aux) cudaEventDestroy(h->ev_aux);
    cudaStreamDestroy(h->stream);
    cudaStreamDestroy(h->h2d_stream);
    cudaStreamDestroy(h->d2h_stream);
    if (h->aux_stream) cudaStreamDestroy(h->aux_stream);
    delete h;
}

rio_status rio_cuda_sync(rio_placement *h) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { CUDA_TRY(cudaStreamSynchronize(h->stream)); if (h->dir_keys_pending) reconcile_dir_keys(h); check_device_error(h); });
}

rio_status rio_cuda_device_info(rio_placement *h, int32_t *device, int32_t *sm_count, uint64_t *hbm_bytes, char *name_buf, size_t name_cap) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (device) *device = h->device;
        if (sm_count) *sm_count = h->sm_count;
        if (hbm_bytes) *hbm_bytes = h->hbm;
        if (name_buf && name_cap) { size_t n = std::min(name_cap - 1, h->devname.size()); memcpy(name_buf, h->devname.data(), n); name_buf[n] = 0; }
    });
}

uint64_t rio_cuda_object_key(const char *type, size_t type_len, const char *id, size_t id_len) {
    uint64_t hsh = fnv1a64(type, type_len);
    const char dot = '.';
    hsh = fnv1a64(&dot, 1, hsh);
    hsh = fnv1a64(id, id_len, hsh);
    return mix64(hsh);
}

uint64_t rio_cuda_node_seed(const char *address, size_t len) { return mix64(fnv1a64(address, len)); }

rio_status rio_cuda_hash_ids(rio_placement *h, const char *packed, const uint64_t *offsets, size_t n, uint64_t *out_keys) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (!n) return;
        REQUIRE(packed && offsets && out_keys, "null buffer");
        const uint64_t total = offsets[n];
        h->s_packed.ensure(total + 64, h->stream);
        h->s_offsets.ensure((n + 1) * 8, h->stream);
        h->s_keys.ensure(n * 8, h->stream);
        CUDA_TRY(cudaMemcpyAsync(h->s_packed.p, packed, total, cudaMemcpyHostToDevice, h->stream));
        CUDA_TRY(cudaMemcpyAsync(h->s_offsets.p, offsets, (n + 1) * 8, cudaMemcpyHostToDevice, h->stream));
        launch_hash_ids(h->L(), h->s_packed.as<char>(), h->s_offsets.as<uint64_t>(), n, h->s_keys.as<uint64_t>());
        CUDA_TRY(cudaMemcpyAsync(out_keys, h->s_keys.p, n * 8, cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(cudaStreamSynchronize(h->stream));
    });
}

// ---- node table ----------------------------------------------------------------------------------------------------
rio_status rio_cuda_set_nodes(rio_placement *h, const char *const *addrs, const uint32_t *weights, const float *feats, uint32_t M, uint32_t K,
                              uint32_t *out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(M == 0 || addrs, "addrs is NULL");
        REQUIRE(!feats || K > 0, "feats given with K == 0");
        if (feats) { h->K = K; for (auto &ni : h->nodes) ni.feat.clear(); h->feat_version++; }
        for (auto &ni : h->nodes) ni.active = false;
        for (uint32_t j = 0; j < M; j++) {
            REQUIRE(addrs[j], "null address");
            const uint32_t idx = intern_node(h, addrs[j]);
            NodeInfo &ni = h->nodes[idx];
            ni.weight = weights ? weights[j] : 1u;
            ni.active = true;
            if (feats) ni.feat.assign(feats + (size_t)j * K, feats + (size_t)(j + 1) * K);
            if (out_idx) out_idx[j] = idx;
        }
        h->tab_dirty = true;
    });
}

rio_status rio_cuda_node_upsert(rio_placement *h, const char *address, uint32_t weight, const float *feat, uint32_t K, uint32_t *out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(address, "address is NULL");
        const uint32_t idx = intern_node(h, address);
        NodeInfo &ni = h->nodes[idx];
        ni.weight = weight;
        ni.active = true;
        if (feat) { REQUIRE(K > 0 && (h->K == 0 || h->K == K), "feature dimension mismatch"); h->K = K; ni.feat.assign(feat, feat + K); h->feat_version++; }
        h->tab_dirty = true;
        if (out_idx) *out_idx = idx;
    });
}

rio_status rio_cuda_node_set_active(rio_placement *h, uint32_t idx, int32_t active) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(idx < h->nodes.size(), "node index out of range");
        h->nodes[idx].active = active != 0;
        h->tab_dirty = true;
    });
}

rio_status rio_cuda_node_index(rio_placement *h, const char *address, uint32_t *out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(address && out_idx, "null argument");
        auto it = h->node_index.find(address);
        *out_idx = it == h->node_index.end() ? RIO_NONE : it->second;
    });
}

rio_status rio_cuda_node_intern(rio_placement *h, const char *address, uint32_t *out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(address && out_idx, "null argument");
        *out_idx = intern_node(h, address);
    });
}

rio_status rio_cuda_node_set_domains(rio_placement *h, const uint32_t *idx, const uint32_t *domain, size_t k) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (!k) return;
        REQUIRE(idx && domain, "null domain arrays");
        std::vector<uint8_t> seen(h->nodes.size(), 0);
        for (size_t i = 0; i < k; i++) {
            REQUIRE(idx[i] < h->nodes.size(), "node index out of range");
            REQUIRE(!seen[idx[i]], "duplicate node index");
            seen[idx[i]] = 1;
        }
        for (size_t i = 0; i < k; i++) h->nodes[idx[i]].domain = domain[i];
        h->label_version++;
    });
}

rio_status rio_cuda_node_domain(rio_placement *h, uint32_t idx, uint32_t *out_domain) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(out_domain, "null argument");
        REQUIRE(idx < h->nodes.size(), "node index out of range");
        *out_domain = h->nodes[idx].domain;
    });
}

rio_status rio_cuda_node_address(rio_placement *h, uint32_t idx, char *buf, size_t cap, size_t *out_len) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(idx < h->nodes.size(), "node index out of range");
        const std::string &a = h->nodes[idx].addr;
        if (out_len) *out_len = a.size();
        if (buf && cap) memcpy(buf, a.data(), std::min(cap, a.size()));
    });
}

rio_status rio_cuda_node_count(rio_placement *h, uint32_t *out_total, uint32_t *out_live) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (out_total) *out_total = (uint32_t)h->nodes.size();
        if (out_live) { uint32_t c = 0; for (auto &ni : h->nodes) c += ni.live(); *out_live = c; }
    });
}

rio_status rio_cuda_node_state(rio_placement *h, uint32_t idx, int32_t *active, uint32_t *weight, int32_t *malformed) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(idx < h->nodes.size(), "node index out of range");
        if (active) *active = h->nodes[idx].active ? 1 : 0;
        if (weight) *weight = h->nodes[idx].weight;
        if (malformed) *malformed = h->nodes[idx].malformed ? 1 : 0;
    });
}

rio_status rio_cuda_set_solver(rio_placement *h, uint32_t solver, uint32_t trie_bits) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(solver == RIO_SOLVER_HRW || solver == RIO_SOLVER_HRW2, "unknown solver");
        REQUIRE(trie_bits <= 14, "trie_bits must be in [0, 14] (0 = keep the current depth)");
        h->solver = solver;
        if (trie_bits && trie_bits != h->trie_bits) { h->trie_bits = trie_bits; h->tab_dirty = true; }
    });
}

rio_status rio_cuda_get_solver(rio_placement *h, uint32_t *solver, uint32_t *trie_bits) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { if (solver) *solver = h->solver; if (trie_bits) *trie_bits = h->trie_bits; });
}

// ---- directory -----------------------------------------------------------------------------------------------------
rio_status rio_cuda_lookup_batch(rio_placement *h, const uint64_t *keys, size_t n, uint32_t *out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (!n) return;
        REQUIRE(keys && out_idx, "null buffer");
        h->s_keys.ensure(n * 8, h->stream);
        h->s_idx.ensure(n * 4, h->stream);
        CUDA_TRY(cudaMemcpyAsync(h->s_keys.p, keys, n * 8, cudaMemcpyHostToDevice, h->stream));
        launch_dir_lookup(h->L(), h->dir, h->s_keys.as<uint64_t>(), n, h->s_idx.as<uint32_t>());
        CUDA_TRY(cudaMemcpyAsync(out_idx, h->s_idx.p, n * 4, cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(cudaStreamSynchronize(h->stream));
    });
}

rio_status rio_cuda_upsert_batch(rio_placement *h, const uint64_t *keys, const uint32_t *idx, size_t n) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (!n) return;
        REQUIRE(keys && idx, "null buffer");
        dir_reserve(h, n);
        h->s_keys.ensure(n * 8, h->stream);
        h->s_idx.ensure(n * 4, h->stream);
        CUDA_TRY(cudaMemcpyAsync(h->s_keys.p, keys, n * 8, cudaMemcpyHostToDevice, h->stream));
        CUDA_TRY(cudaMemcpyAsync(h->s_idx.p, idx, n * 4, cudaMemcpyHostToDevice, h->stream));
        dir_upsert_dev(h, h->s_keys.as<uint64_t>(), h->s_idx.as<uint32_t>(), 0, n);
        reconcile_dir_keys(h);
        check_device_error(h);
    });
}

rio_status rio_cuda_remove_batch(rio_placement *h, const uint64_t *keys, size_t n) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (!n) return;
        REQUIRE(keys, "null buffer");
        dir_reserve(h, n);
        h->s_keys.ensure(n * 8, h->stream);
        CUDA_TRY(cudaMemcpyAsync(h->s_keys.p, keys, n * 8, cudaMemcpyHostToDevice, h->stream));
        dir_upsert_dev(h, h->s_keys.as<uint64_t>(), nullptr, kNone, n);
        reconcile_dir_keys(h);
        check_device_error(h);
    });
}

rio_status rio_cuda_clean_node(rio_placement *h, uint32_t idx, uint64_t *out_removed) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (idx == RIO_NONE || idx >= h->nodes.size()) { if (out_removed) *out_removed = 0; return; }   // unknown address: nothing recorded on it
        zero_scalar(h, S_MOVED);
        launch_dir_clean_node(h->L(), h->dir, idx, h->d_scalars + S_MOVED);
        const uint64_t r = read_scalar(h, S_MOVED);
        if (out_removed) *out_removed = r;
    });
}

rio_status rio_cuda_directory_len(rio_placement *h, uint64_t *out_placed, uint64_t *out_slots) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        zero_scalar(h, S_PLACED);
        launch_dir_count(h->L(), h->dir, h->d_scalars + S_PLACED, nullptr, 0);
        const uint64_t p = read_scalar(h, S_PLACED);
        if (out_placed) *out_placed = p;
        if (out_slots) *out_slots = h->dir_cap;
    });
}

rio_status rio_cuda_directory_reserve(rio_placement *h, uint64_t n_more) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { dir_reserve(h, n_more); CUDA_TRY(cudaStreamSynchronize(h->stream)); });
}

rio_status rio_cuda_load_counters(rio_placement *h, uint32_t *out, uint32_t cap) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        const uint32_t n_total = (uint32_t)h->nodes.size();
        REQUIRE(out && cap >= n_total, "counter buffer too small");
        if (!n_total) return;
        h->s_misc.ensure((size_t)n_total * 4, h->stream);
        CUDA_TRY(cudaMemsetAsync(h->s_misc.p, 0, (size_t)n_total * 4, h->stream));
        zero_scalar(h, S_PLACED);
        launch_dir_count(h->L(), h->dir, h->d_scalars + S_PLACED, h->s_misc.as<uint32_t>(), n_total);
        CUDA_TRY(cudaMemcpyAsync(out, h->s_misc.p, (size_t)n_total * 4, cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(cudaStreamSynchronize(h->stream));
    });
}

// ---- solver --------------------------------------------------------------------------------------------------------
rio_status rio_cuda_assign_batch(rio_placement *h, const uint64_t *keys, const float *obj_feats, size_t n, uint32_t *out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (!n) return;
        REQUIRE((keys || obj_feats) && out_idx, "null buffer");
        if (!obj_feats) REQUIRE(keys, "keys is NULL");
        assign_host_pipelined(h, keys, obj_feats, n, out_idx);
    });
}

rio_status rio_cuda_assign_bounded_batch(rio_placement *h, const uint64_t *keys, size_t n, uint64_t n_total_objs, uint32_t cap_num, uint32_t cap_den,
                                         uint32_t max_rounds, uint32_t *out_idx, uint32_t *out_passes) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (out_passes) *out_passes = 0;
        if (!n) return;
        REQUIRE(keys && out_idx, "null buffer");
        REQUIRE(cap_den > 0 && max_rounds > 0, "bad capacity factor / rounds");
        REQUIRE(n < 0xFFFFFFFFull, "batch too large");
        ensure_tab(h);
        const uint32_t M = h->tabs.tab.n_total;
        if (!n_total_objs) n_total_objs = (uint64_t)n * (uint64_t)h->world;
        h->s_misc.ensure((size_t)std::max(M, 1u) * 4, h->stream);
        h->s_sel.ensure(n * 4, h->stream);
        uint32_t *d_cnt = h->s_misc.as<uint32_t>();
        CUDA_TRY(cudaMemsetAsync(d_cnt, 0, (size_t)std::max(M, 1u) * 4, h->stream));
        // pass 0: chunk-pipelined H2D / score+histogram / D2H; the exchange + capacity check runs behind the last chunk while its
        // indices are still crossing PCIe
        assign_host_pipelined(h, keys, nullptr, n, out_idx, d_cnt, false);
        bounded_begin(h, h->bs, h->s_keys.as<uint64_t>(), n, h->s_idx.as<uint32_t>(), d_cnt, M, n_total_objs, cap_num, cap_den, max_rounds, true, true, nullptr);
        const uint32_t passes = bounded_end(h, h->bs, h->s_keys.as<uint64_t>(), n, h->s_idx.as<uint32_t>(), d_cnt, h->s_sel.as<uint32_t>(),
                                            hash_replace(h, h->s_keys.as<uint64_t>(), n, h->s_idx.as<uint32_t>(), d_cnt, h->s_sel.as<uint32_t>()));
        CUDA_TRY(cudaStreamSynchronize(h->d2h_stream));
        if (passes > 1) {   // a spill round rewrote some indices after their chunk had left: send the final state again
            CUDA_TRY(cudaMemcpyAsync(out_idx, h->s_idx.p, n * 4, cudaMemcpyDeviceToHost, h->stream));
            CUDA_TRY(cudaStreamSynchronize(h->stream));
        }
        if (out_passes) *out_passes = passes;
    });
}

rio_status rio_cuda_assign_bounded_affinity_batch(rio_placement *h, const uint64_t *keys, const float *obj_feats, size_t n, uint64_t n_total_objs,
                                                  uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds, uint32_t *out_idx, uint32_t *out_passes) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (out_passes) *out_passes = 0;
        if (!n) return;
        REQUIRE(keys && obj_feats && out_idx, "null buffer");
        REQUIRE(cap_den > 0 && max_rounds > 0, "bad capacity factor / rounds");
        REQUIRE(n < 0xFFFFFFFFull, "batch too large");
        REQUIRE(h->K > 0, "assign with object features needs node features");
        require_bounded_affinity_kernels();
        ensure_tab(h);
        const uint32_t M = h->tabs.tab.n_total, K = h->K;
        if (!n_total_objs) n_total_objs = (uint64_t)n * (uint64_t)h->world;
        cudaStream_t st = h->stream;
        h->s_keys.ensure(n * 8, st);
        h->s_feats.ensure(n * (size_t)K * 4, st);
        h->s_idx.ensure(n * 4, st);
        h->s_sel.ensure(n * 4, st);
        h->s_misc.ensure((size_t)std::max(M, 1u) * 4, st);
        CUDA_TRY(cudaMemcpyAsync(h->s_keys.p, keys, n * 8, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(h->s_feats.p, obj_feats, n * (size_t)K * 4, cudaMemcpyHostToDevice, st));
        const uint32_t passes = bounded_affinity(h, h->bs, h->s_keys.as<uint64_t>(), h->s_feats.as<float>(), n, h->s_idx.as<uint32_t>(), h->s_misc.as<uint32_t>(), M,
                                                 h->s_sel.as<uint32_t>(), n_total_objs, cap_num, cap_den, max_rounds, affinity_path(h));
        CUDA_TRY(cudaMemcpyAsync(out_idx, h->s_idx.p, n * 4, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        if (out_passes) *out_passes = passes;
    });
}

rio_status rio_cuda_assign_bounded_weighted_batch(rio_placement *h, const uint64_t *keys, const float *obj_feats, const uint32_t *weights, size_t n,
                                                  uint64_t load_total, uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds, uint32_t *out_idx,
                                                  uint32_t *out_passes) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (out_passes) *out_passes = 0;
        if (!n) return;
        REQUIRE(keys && out_idx, "null buffer");
        REQUIRE(cap_den > 0 && max_rounds > 0, "bad capacity factor / rounds");
        REQUIRE(n < 0xFFFFFFFFull, "batch too large");
        if (obj_feats) {
            REQUIRE(h->K > 0, "assign with object features needs node features");
            require_bounded_affinity_kernels();
        }
        require_weighted_kernels();
        uint64_t local = n;
        if (weights) { local = 0; for (size_t i = 0; i < n; i++) local += weights[i]; }
        const uint64_t L = weighted_load_total(global_weight_sum(h, local), load_total);
        ensure_tab(h);
        const uint32_t M = h->tabs.tab.n_total, K = h->K;
        cudaStream_t st = h->stream;
        h->s_keys.ensure(n * 8, st);
        h->s_idx.ensure(n * 4, st);
        h->s_sel.ensure(n * 4, st);
        h->s_misc.ensure((size_t)std::max(M, 1u) * 4, st);
        CUDA_TRY(cudaMemcpyAsync(h->s_keys.p, keys, n * 8, cudaMemcpyHostToDevice, st));
        if (obj_feats) {
            h->s_feats.ensure(n * (size_t)K * 4, st);
            CUDA_TRY(cudaMemcpyAsync(h->s_feats.p, obj_feats, n * (size_t)K * 4, cudaMemcpyHostToDevice, st));
        }
        if (weights) {
            h->s_weights.ensure(n * 4, st);
            CUDA_TRY(cudaMemcpyAsync(h->s_weights.p, weights, n * 4, cudaMemcpyHostToDevice, st));
        }
        const uint32_t passes = bounded_weighted(h, h->bs, h->s_keys.as<uint64_t>(), obj_feats ? h->s_feats.as<float>() : nullptr,
                                                 weights ? h->s_weights.as<uint32_t>() : nullptr, n, h->s_idx.as<uint32_t>(), h->s_misc.as<uint32_t>(), M,
                                                 h->s_sel.as<uint32_t>(), L, cap_num, cap_den, max_rounds, obj_feats != nullptr, affinity_path(h));
        CUDA_TRY(cudaMemcpyAsync(out_idx, h->s_idx.p, n * 4, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        if (out_passes) *out_passes = passes;
    });
}

rio_status rio_cuda_assign_batch_dev(rio_placement *h, const uint64_t *d_keys, const float *d_obj_feats, size_t n, uint32_t *d_out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (!n) return;
        REQUIRE(d_out_idx && (d_keys || d_obj_feats), "null buffer");
        require_natural(d_keys, 8, "d_keys");
        require_natural(d_obj_feats, 4, "d_obj_feats");
        require_natural(d_out_idx, 4, "d_out_idx");
        if (d_obj_feats) {
            REQUIRE(h->K > 0, "assign with object features needs node features");
            REQUIRE(n <= SIZE_MAX / 4 / h->K, "n x K overflows");
            ensure_tab(h);
            const AffinityPath path = affinity_path(h);
            run_affinity(h, affinity_input(h, d_obj_feats, n, path), n, d_out_idx, nullptr, nullptr, path);
        } else {
            ensure_tab(h);
            // the flat kernels read keys and write indices one at a time; the HRW2 walk two at a time
            const bool trie = h->solver == RIO_SOLVER_HRW2;
            const uint64_t *keys = input_at(h, h->s_keys, d_keys, n, trie ? kAlignTrieKeys : 8u);
            uint32_t *out = output_at(h, h->s_idx, d_out_idx, n, trie ? kAlignTrieOut : 4u);
            run_assign(h, h->solver, h->tabs, keys, n, out, nullptr, nullptr, 0);
            output_done(h, out, d_out_idx, n);
        }
    });
}

rio_status rio_cuda_assign_ranked_batch(rio_placement *h, const uint64_t *keys, size_t n, uint32_t ranks, uint32_t *out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { lists_from_host(h, ListKind::kHash, keys, n, ranks, out_idx); });
}

rio_status rio_cuda_assign_ranked_batch_dev(rio_placement *h, const uint64_t *d_keys, size_t n, uint32_t ranks, uint32_t *d_out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { lists_from_device(h, ListKind::kHash, d_keys, n, ranks, d_out_idx); });
}

rio_status rio_cuda_assign_ranked_spread_batch(rio_placement *h, const uint64_t *keys, size_t n, uint32_t ranks, uint32_t *out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { lists_from_host(h, ListKind::kSpread, keys, n, ranks, out_idx); });
}

rio_status rio_cuda_assign_ranked_spread_batch_dev(rio_placement *h, const uint64_t *d_keys, size_t n, uint32_t ranks, uint32_t *d_out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { lists_from_device(h, ListKind::kSpread, d_keys, n, ranks, d_out_idx); });
}

rio_status rio_cuda_assign_ranked_affinity_batch(rio_placement *h, const float *obj_feats, size_t n, uint32_t ranks, uint32_t *out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { lists_from_host(h, ListKind::kAffinity, obj_feats, n, ranks, out_idx); });
}

rio_status rio_cuda_assign_ranked_affinity_batch_dev(rio_placement *h, const float *d_obj_feats, size_t n, uint32_t ranks, uint32_t *d_out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { lists_from_device(h, ListKind::kAffinity, d_obj_feats, n, ranks, d_out_idx); });
}

rio_status rio_cuda_assign_ranked_affinity_spread_batch(rio_placement *h, const float *obj_feats, size_t n, uint32_t ranks, uint32_t *out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { lists_from_host(h, ListKind::kAffinitySpread, obj_feats, n, ranks, out_idx); });
}

rio_status rio_cuda_assign_ranked_affinity_spread_batch_dev(rio_placement *h, const float *d_obj_feats, size_t n, uint32_t ranks, uint32_t *d_out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { lists_from_device(h, ListKind::kAffinitySpread, d_obj_feats, n, ranks, d_out_idx); });
}

rio_status rio_cuda_lookup_batch_dev(rio_placement *h, const uint64_t *d_keys, size_t n, uint32_t *d_out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (!n) return;
        REQUIRE(d_keys && d_out_idx, "null buffer");
        require_natural(d_keys, 8, "d_keys");
        require_natural(d_out_idx, 4, "d_out_idx");
        launch_dir_lookup(h->L(), h->dir, d_keys, n, d_out_idx);   // one key read and one index written at a time: used in place
    });
}

rio_status rio_cuda_upsert_batch_dev(rio_placement *h, const uint64_t *d_keys, const uint32_t *d_idx, size_t n) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (!n) return;
        REQUIRE(d_keys && d_idx, "null buffer");
        require_natural(d_keys, 8, "d_keys");
        require_natural(d_idx, 4, "d_idx");
        // k_dir_upsert reads one key and one index at a time: the caller's buffers are used in place
        REQUIRE((h->dir_keys + h->dir_keys_pending + n) * 10 <= h->dir_cap * 9, "directory too small for an asynchronous upsert: call rio_cuda_directory_reserve first");
        dir_upsert_dev(h, d_keys, d_idx, 0, n);
        h->dir_keys_pending += n;
    });
}

rio_status rio_cuda_place_batch(rio_placement *h, const uint64_t *keys, size_t n, uint32_t policy, uint32_t self_idx, uint32_t *out_idx) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (!n) return;
        REQUIRE(keys && out_idx, "null buffer");
        REQUIRE(policy == RIO_PLACE_SELF || policy == RIO_PLACE_HRW || policy == RIO_PLACE_HRW2, "unknown policy");
        REQUIRE(n < 0xFFFFFFFFull, "batch too large");
        if (policy == RIO_PLACE_SELF) REQUIRE(self_idx < h->nodes.size(), "self_idx is not a known node");
        ensure_tab(h);
        const uint32_t n_total = h->tabs.tab.n_total;
        cudaStream_t st = h->stream;
        h->s_keys.ensure(n * 8, st);
        h->s_idx.ensure(n * 4, st);
        h->s_sel.ensure(n * 4, st);
        h->s_misc.ensure(std::max<size_t>(n_total, 1), st);
        CUDA_TRY(cudaMemcpyAsync(h->s_keys.p, keys, n * 8, cudaMemcpyHostToDevice, st));
        launch_dir_lookup(h->L(), h->dir, h->s_keys.as<uint64_t>(), n, h->s_idx.as<uint32_t>());                          // service.rs:199-201
        zero_scalar(h, S_NSEL);
        CUDA_TRY(cudaMemsetAsync(h->s_misc.p, 0, std::max<size_t>(n_total, 1), st));
        launch_classify(h->L(), h->s_idx.as<uint32_t>(), n, h->tabs.state, n_total, h->s_sel.as<uint32_t>(), h->d_scalars + S_NSEL,
                        h->s_misc.as<uint8_t>());
        const uint64_t nsel = read_scalar(h, S_NSEL);
        if (nsel) {
            // clean_server for every inactive node that was met (service.rs:233-237): one pass over the table for all of them
            zero_scalar(h, S_MOVED);
            launch_dir_clean_flagged(h->L(), h->dir, h->s_misc.as<uint8_t>(), n_total, h->d_scalars + S_MOVED);
            if (policy == RIO_PLACE_SELF) launch_scatter_const(h->L(), h->s_idx.as<uint32_t>(), h->s_sel.as<uint32_t>(), nsel, self_idx);   // :244-252
            else run_assign(h, policy == RIO_PLACE_HRW2 ? RIO_SOLVER_HRW2 : RIO_SOLVER_HRW, h->tabs, h->s_keys.as<uint64_t>(), n, h->s_idx.as<uint32_t>(), nullptr, h->s_sel.as<uint32_t>(), nsel);
            h->s_keys2.ensure(nsel * 8, st);
            h->s_idx2.ensure(nsel * 4, st);
            launch_gather_keys(h->L(), h->s_keys.as<uint64_t>(), h->s_sel.as<uint32_t>(), nsel, h->s_keys2.as<uint64_t>(), h->s_idx.as<uint32_t>(),
                               h->s_idx2.as<uint32_t>());
            dir_reserve(h, nsel);
            dir_upsert_dev(h, h->s_keys2.as<uint64_t>(), h->s_idx2.as<uint32_t>(), 0, nsel);
        }
        CUDA_TRY(cudaMemcpyAsync(out_idx, h->s_idx.p, n * 4, cudaMemcpyDeviceToHost, st));
        if (nsel) { reconcile_dir_keys(h); check_device_error(h); } else CUDA_TRY(cudaStreamSynchronize(st));
    });
}

rio_status rio_cuda_check_address_batch(rio_placement *h, const uint32_t *addr_idx, size_t n, uint32_t self_idx, uint8_t *out_verdict, uint64_t *out_cleaned) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (out_cleaned) *out_cleaned = 0;
        if (!n) return;
        REQUIRE(addr_idx && out_verdict, "null buffer");
        REQUIRE(self_idx < h->nodes.size(), "self_idx is not a known node");
        const uint32_t n_total = (uint32_t)h->nodes.size();
        // verdict of every interned address against this server (service.rs:261-298): a table of n_total bytes, built on the host
        // from the membership view, applied to the batch on the device together with the clean_server scan
        std::vector<uint8_t> verdict(n_total, RIO_ADDR_DEALLOCATE);
        for (uint32_t j = 0; j < n_total; j++) {
            const std::string &a = h->nodes[j].addr;
            if (j == self_idx) { verdict[j] = RIO_ADDR_LOCAL; continue; }                          // :262-264 (before any format check)
            const size_t c = a.find(':');
            if (c == std::string::npos) { verdict[j] = RIO_ADDR_MALFORMED; continue; }              // :272-278 "Missing PORT"
            const size_t c2 = a.find(':', c + 1);                                                    // split(':'): ip = piece 0, port = piece 1
            bool active = h->nodes[j].active;
            if (c2 != std::string::npos) {   // a third piece: is_active is asked about "ip:port" of the first two
                auto it = h->node_index.find(a.substr(0, c2));
                active = it != h->node_index.end() && h->nodes[it->second].active;
            }
            verdict[j] = active ? RIO_ADDR_REDIRECT : RIO_ADDR_DEALLOCATE;                          // :280-297
        }
        cudaStream_t st = h->stream;
        h->s_idx.ensure(n * 4, st);
        h->s_idx2.ensure(n, st);
        h->s_misc.ensure((size_t)n_total * 2, st);
        uint8_t *d_verdict_tab = h->s_misc.as<uint8_t>(), *d_dead = d_verdict_tab + n_total;
        CUDA_TRY(cudaMemcpyAsync(h->s_idx.p, addr_idx, n * 4, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(d_verdict_tab, verdict.data(), n_total, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemsetAsync(d_dead, 0, n_total, st));
        zero_scalar(h, S_NSEL);
        zero_scalar(h, S_MOVED);
        launch_check_address(h->L(), h->s_idx.as<uint32_t>(), n, d_verdict_tab, n_total, h->s_idx2.as<uint8_t>(), d_dead, h->d_scalars + S_NSEL);
        CUDA_TRY(cudaMemcpyAsync(out_verdict, h->s_idx2.p, n, cudaMemcpyDeviceToHost, st));
        const uint64_t n_dead = read_scalar(h, S_NSEL);
        if (n_dead) {   // clean_server for every non-active address that was met (service.rs:291-296): one scan for all of them
            launch_dir_clean_flagged(h->L(), h->dir, d_dead, n_total, h->d_scalars + S_MOVED);
            const uint64_t cleaned = read_scalar(h, S_MOVED);
            if (out_cleaned) *out_cleaned = cleaned;
        }
    });
}

rio_status rio_dev_set_node_seed(rio_placement *h, uint32_t idx, uint64_t seed) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(idx < h->nodes.size(), "node index out of range");
        h->nodes[idx].seed = seed;
        h->nodes[idx].seed2 = mix64(seed ^ kSaltNode2);
        h->tab_dirty = true;
    });
}

rio_status rio_dev_set_table_options(rio_placement *h, uint32_t flags) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { h->dev_table_flags = flags; h->tab_dirty = true; });
}

rio_status rio_cuda_rebalance(rio_placement *h, uint32_t event, uint32_t idx, uint64_t *out_moved) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(event == RIO_EV_JOIN || event == RIO_EV_LEAVE, "unknown event");
        REQUIRE(idx < h->nodes.size(), "node index out of range");
        ensure_tab(h);
        zero_scalar(h, S_MOVED);
        if (event == RIO_EV_JOIN) REQUIRE(h->nodes[idx].live(), "JOIN of a node that is not live");
        else REQUIRE(!h->nodes[idx].live(), "LEAVE of a node that is still live (deactivate it first)");
        if (h->solver == RIO_SOLVER_HRW2)   // thresholds changed on the whole root path of the node: every placed key is walked again (16 B/slot stream)
            launch_dir_reassign_trie(h->L(), h->dir, h->tabs.trie, h->d_scalars + S_MOVED);
        else if (event == RIO_EV_JOIN) launch_dir_rebalance_join(h->L(), h->dir, h->tabs.tab, idx, h->d_scalars + S_MOVED);
        else launch_dir_rebalance_leave(h->L(), h->dir, h->tabs.tab, idx, h->d_scalars + S_MOVED);
        const uint64_t m = read_scalar(h, S_MOVED);
        if (out_moved) *out_moved = m;
    });
}

namespace {

// A change set (DESIGN.md 3.10) as the flat-policy kernels see it: one byte per interned node (REPLACE / CANDIDATE / neither) and
// the list of candidates, uploaded into h->s_misc.  The arguments were checked by check_change_set.
struct ChangeSetHost {
    std::vector<uint8_t> bytes;   // n_total flag bytes, padded to 4, then the candidate indices
    uint32_t n_cand = 0;
    // every interned node not live now is REPLACE; the caller's rule classifies the changed live nodes with mark()
    explicit ChangeSetHost(const rio_placement *h) {
        const uint32_t n_total = (uint32_t)h->nodes.size();
        bytes.assign(std::max<size_t>((n_total + 3) & ~(size_t)3, 4), 0);
        for (uint32_t j = 0; j < n_total; j++) if (!h->nodes[j].live()) bytes[j] = kChgReplace;
    }
    // node j's flags become `flags`; a CANDIDATE goes onto the candidate list once
    void mark(uint32_t j, uint8_t flags) {
        if ((flags & kChgCandidate) && !(bytes[j] & kChgCandidate)) {
            const size_t o = bytes.size();
            bytes.resize(o + 4);
            memcpy(bytes.data() + o, &j, 4);
            n_cand++;
        }
        bytes[j] = flags;
    }
};

void check_change_set(const rio_placement *h, const uint32_t *idx, const uint32_t *prev_weight, size_t k) {
    REQUIRE(!k || (idx && prev_weight), "null change-set arrays");
    const size_t n_total = h->nodes.size();
    std::vector<uint8_t> seen(n_total, 0);
    for (size_t i = 0; i < k; i++) {
        REQUIRE(idx[i] < n_total, "change-set node index out of range");
        REQUIRE(!seen[idx[i]], "duplicate node index in the change set");
        seen[idx[i]] = 1;
    }
}

ChangeSetHost build_change_set(const rio_placement *h, const uint32_t *idx, const uint32_t *prev_weight, size_t k) {
    ChangeSetHost cs(h);
    for (size_t i = 0; i < k; i++) {
        const NodeInfo &ni = h->nodes[idx[i]];
        if (!ni.live()) continue;   // REPLACE already
        const uint32_t r_prev = prev_weight[i] ? inv_weight(prev_weight[i]) : 0u, r_now = inv_weight(ni.weight);
        if (r_prev && r_now > r_prev) cs.mark(idx[i], kChgReplace);                  // lost weight
        else if (!r_prev || r_now < r_prev) cs.mark(idx[i], kChgCandidate);          // joined or gained weight
    }
    return cs;
}

// Spread lists (DESIGN.md 3.13): a relabelled live node is REPLACE | CANDIDATE.  Lists holding it are recomputed; every other list
// considers it under its new label.
void add_relabels(ChangeSetHost &cs, const std::vector<uint32_t> &relabelled) {
    for (uint32_t j : relabelled) cs.mark(j, kChgReplace | kChgCandidate);
}

ChangeSetDev upload_change_set(rio_placement *h, const ChangeSetHost &cs) {
    h->s_misc.ensure(cs.bytes.size(), h->stream);
    CUDA_TRY(cudaMemcpyAsync(h->s_misc.p, cs.bytes.data(), cs.bytes.size(), cudaMemcpyHostToDevice, h->stream));
    const uint8_t *d = h->s_misc.as<uint8_t>();
    return ChangeSetDev{d, reinterpret_cast<const uint32_t *>(d + cs.bytes.size() - (size_t)cs.n_cand * 4), cs.n_cand};
}

void require_change_kernels() {
    if (!launch_dir_rebalance_changes || !launch_dir_scatter_changes || !launch_rebalance_changes || !launch_count_changed)
        throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no change-set kernels (k_directory.cu without them is linked)"};
}

}  // namespace

rio_status rio_cuda_rebalance_changes(rio_placement *h, const uint32_t *idx, const uint32_t *prev_weight, size_t k, uint64_t *out_moved) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        check_change_set(h, idx, prev_weight, k);
        uint64_t moved = 0;
        if (k) {
            ensure_tab(h);
            zero_scalar(h, S_MOVED);
            if (h->solver == RIO_SOLVER_HRW2) {   // one re-walk of every placed key, whatever the change set holds
                launch_dir_reassign_trie(h->L(), h->dir, h->tabs.trie, h->d_scalars + S_MOVED);
            } else {
                require_change_kernels();
                const ChangeSetHost cs = build_change_set(h, idx, prev_weight, k);
                const ChangeSetDev dcs = upload_change_set(h, cs);
                // every claimed key could be an R1 entry (all nodes left): the lists are sized for that, grow-only
                const uint64_t max_r1 = std::max<uint64_t>(h->dir_keys + h->dir_keys_pending, 1);
                h->s_slots.ensure(max_r1 * 8, h->stream);
                h->s_keys2.ensure(max_r1 * 8, h->stream);
                zero_scalar(h, S_NSEL);
                launch_dir_rebalance_changes(h->L(), h->dir, h->tabs.tab, dcs, h->s_slots.as<uint64_t>(), h->s_keys2.as<uint64_t>(), h->d_scalars + S_NSEL,
                                             h->d_scalars + S_MOVED);
                const uint64_t n_r1 = read_scalar(h, S_NSEL);
                if (n_r1) {
                    h->s_idx2.ensure(n_r1 * 4, h->stream);
                    launch_assign_hrw(h->L(), h->s_keys2.as<uint64_t>(), n_r1, h->tabs.tab, h->s_idx2.as<uint32_t>(), nullptr, nullptr, 0);
                    launch_dir_scatter_changes(h->L(), h->dir, h->s_slots.as<uint64_t>(), h->s_idx2.as<uint32_t>(), n_r1, h->d_scalars + S_MOVED);
                }
            }
            moved = read_scalar(h, S_MOVED);
        }
        if (out_moved) *out_moved = moved;
    });
}

// ---- resident object sets --------------------------------------------------------------------------------------------
rio_status rio_cuda_set_create(rio_placement *h, uint64_t capacity, rio_objset **out) {
    if (!h || !out) { g_last_error = "null argument"; return RIO_ERR_UNKNOWN; }
    *out = nullptr;
    rio_objset *s = new rio_objset();
    rio_status st = guarded(h, [&] {
        REQUIRE(capacity > 0 && capacity < 0xFFFFFFFFull, "set capacity must be in [1, 2^32-2]");
        s->h = h;
        s->capacity = capacity;
        s->keys.ensure(capacity * 8, h->stream);
        s->idx.ensure(capacity * 4, h->stream);
        s->sel.ensure(capacity * 4, h->stream);
        launch_fill_u32(h->L(), s->idx.as<uint32_t>(), capacity, kNone);
        CUDA_TRY(cudaStreamSynchronize(h->stream));
    });
    if (st != RIO_OK) { delete s; return st; }
    *out = s;
    return RIO_OK;
}

void rio_cuda_set_destroy(rio_objset *s) {
    if (!s) return;
    rio_placement *h = s->h;
    {
        std::lock_guard<std::mutex> g(h->mu);
        cudaSetDevice(h->device);
        if (h->aux_stream) cudaStreamSynchronize(h->aux_stream);   // a check of this set may still be in flight
        s->keys.release(h->stream); s->idx.release(h->stream); s->feats.release(h->stream); s->counters.release(h->stream); s->counters_alt.release(h->stream); s->sel.release(h->stream); s->bs.release(h->stream); s->lists.release(h->stream);
        s->weights.release(h->stream); s->loads.release(h->stream);
        cudaStreamSynchronize(h->stream);
    }
    delete s;
}

rio_status rio_cuda_set_load_keys(rio_objset *s, const uint64_t *keys, uint64_t n) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(n <= s->capacity && (keys || !n), "too many keys for this set");
        CUDA_TRY(cudaMemcpyAsync(s->keys.p, keys, n * 8, cudaMemcpyHostToDevice, h->stream));
        s->n = n; s->assigned = false; s->drop_lists(); s->has_weights = false;
        CUDA_TRY(cudaStreamSynchronize(h->stream));
    });
}

rio_status rio_cuda_set_synth_keys(rio_objset *s, uint64_t first, uint64_t n, uint64_t seed) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(n <= s->capacity, "too many keys for this set");
        launch_synth_keys(h->L(), s->keys.as<uint64_t>(), first, n, seed);
        s->n = n; s->assigned = false; s->drop_lists(); s->has_weights = false;
    });
}

rio_status rio_cuda_set_load_feats(rio_objset *s, const float *feats, uint32_t K) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(feats && K > 0, "null features");
        s->feats.ensure(s->n * (size_t)K * 4, h->stream);
        CUDA_TRY(cudaMemcpyAsync(s->feats.p, feats, s->n * (size_t)K * 4, cudaMemcpyHostToDevice, h->stream));
        s->K = K;
        if (is_affinity(s->kind)) s->drop_lists();   // affinity lists are lists of the features just replaced; hash lists stay
        s->bounded_aff = false;
        if (s->plain_aff) s->bounded_w = false;
        CUDA_TRY(cudaStreamSynchronize(h->stream));
    });
}

rio_status rio_cuda_set_assign(rio_objset *s, uint32_t use_affinity) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        s->drop_lists();
        ensure_tab(h);
        set_ensure_counters(s);
        set_zero_counters(s);
        if (use_affinity) {
            REQUIRE(s->K > 0 && s->K == h->K, "set features / node features missing or of different K");
            const AffinityPath path = affinity_path(h);
            run_affinity(h, s->feats.as<float>(), s->n, s->idx.as<uint32_t>(), nullptr, s->counters.as<uint32_t>(), path);
            record_plain_affinity(s, path);
        } else {
            run_assign(h, h->solver, h->tabs, s->keys.as<uint64_t>(), s->n, s->idx.as<uint32_t>(), s->counters.as<uint32_t>(), nullptr, 0);
            s->plain_aff = false;
        }
        s->assigned = true;
    });
}

static void set_bounded_begin(rio_objset *s, uint64_t n_total_objs, uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds, bool pipelined) {
    rio_placement *h = s->h;
    REQUIRE(cap_den > 0 && max_rounds > 0, "bad capacity factor / rounds");
    s->drop_lists();
    ensure_tab(h);
    set_ensure_counters(s);
    if (!n_total_objs) n_total_objs = s->n * (uint64_t)h->world;
    // two counter buffers take turns: the check of this pass clears the other one, so the next pass starts without a memset
    const bool zeroed = s->alt_zero;
    if (zeroed) std::swap(s->counters, s->counters_alt);
    bounded_begin(h, s->bs, s->keys.as<uint64_t>(), s->n, s->idx.as<uint32_t>(), s->counters.as<uint32_t>(), s->counters_n, n_total_objs, cap_num, cap_den, max_rounds,
                  false, zeroed, s->counters_alt.as<uint32_t>(), pipelined);
    s->alt_zero = max_rounds > 1;
    s->plain_aff = false;
}
static uint32_t set_bounded_end(rio_objset *s) {
    rio_placement *h = s->h;
    const uint32_t passes = bounded_end(h, s->bs, s->keys.as<uint64_t>(), s->n, s->idx.as<uint32_t>(), s->counters.as<uint32_t>(), s->sel.as<uint32_t>(),
                                        hash_replace(h, s->keys.as<uint64_t>(), s->n, s->idx.as<uint32_t>(), s->counters.as<uint32_t>(), s->sel.as<uint32_t>()));
    s->assigned = true;
    if (s->bs.max_rounds == 1) CUDA_TRY(cudaStreamSynchronize(h->stream));   // otherwise the check's report already ordered the pass before this return
    return passes;
}

rio_status rio_cuda_set_assign_bounded(rio_objset *s, uint64_t n_total_objs, uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds, uint32_t *out_passes) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    return guarded(s->h, [&] {
        set_bounded_begin(s, n_total_objs, cap_num, cap_den, max_rounds, false);
        const uint32_t passes = set_bounded_end(s);
        if (out_passes) *out_passes = passes;
    });
}

rio_status rio_cuda_set_assign_bounded_begin(rio_objset *s, uint64_t n_total_objs, uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    return guarded(s->h, [&] { set_bounded_begin(s, n_total_objs, cap_num, cap_den, max_rounds, true); });
}

rio_status rio_cuda_set_assign_bounded_end(rio_objset *s, uint32_t *out_passes) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    return guarded(s->h, [&] {
        const uint32_t passes = set_bounded_end(s);
        if (out_passes) *out_passes = passes;
    });
}

namespace {
void record_affinity(rio_objset *s, AffinityPath path);
}  // namespace

rio_status rio_cuda_set_assign_bounded_affinity(rio_objset *s, uint64_t n_total_objs, uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds,
                                                uint32_t *out_passes) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(cap_den > 0 && max_rounds > 0, "bad capacity factor / rounds");
        REQUIRE(h->K > 0, "assign with object features needs node features");
        REQUIRE(s->K > 0 && s->K == h->K && s->feats.bytes >= s->n * (size_t)s->K * 4, "set features / node features missing or of different K");
        REQUIRE(!s->bs.active, "a bounded call is already in flight on this set (call _end first)");
        require_bounded_affinity_kernels();
        s->drop_lists();
        ensure_tab(h);
        set_ensure_counters(s);
        if (!n_total_objs) n_total_objs = s->n * (uint64_t)h->world;
        const AffinityPath path = affinity_path(h);
        const uint32_t passes = bounded_affinity(h, s->bs, s->keys.as<uint64_t>(), s->feats.as<float>(), s->n, s->idx.as<uint32_t>(), s->counters.as<uint32_t>(),
                                                 s->counters_n, s->sel.as<uint32_t>(), n_total_objs, cap_num, cap_den, max_rounds, path);
        s->assigned = true;
        if (max_rounds == 1) CUDA_TRY(cudaStreamSynchronize(h->stream));   // otherwise the check's report already ordered the pass before this return
        record_affinity(s, path);
        record_plain_affinity(s, path);
        s->bounded_aff = true;
        if (out_passes) *out_passes = passes;
    });
}

// ---- weighted objects (DESIGN.md 3.19) --------------------------------------------------------------------------------------------
rio_status rio_cuda_set_write_weights(rio_objset *s, uint64_t first, uint64_t n, const uint32_t *w) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(w || !n, "null weights");
        REQUIRE(first <= s->n && n <= s->n - first, "range outside the set");
        if (!n) return;
        if (!s->has_weights) {   // first write: the column, every row 1
            s->weights.ensure(s->capacity * 4, h->stream);
            launch_fill_u32(h->L(), s->weights.as<uint32_t>(), s->n, 1u);
            s->has_weights = true;
        }
        CUDA_TRY(cudaMemcpyAsync(s->weights.as<uint32_t>() + first, w, n * 4, cudaMemcpyHostToDevice, h->stream));
        CUDA_TRY(cudaStreamSynchronize(h->stream));
    });
}

rio_status rio_cuda_set_read_weights(rio_objset *s, uint64_t first, uint64_t n, uint32_t *out) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(out || !n, "null buffer");
        REQUIRE(first <= s->n && n <= s->n - first, "range outside the set");
        if (!n) return;
        if (!s->has_weights) { std::fill(out, out + n, 1u); return; }
        CUDA_TRY(cudaMemcpyAsync(out, s->weights.as<uint32_t>() + first, n * 4, cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(cudaStreamSynchronize(h->stream));
    });
}

rio_status rio_cuda_set_assign_bounded_weighted(rio_objset *s, uint32_t use_affinity, uint64_t load_total, uint32_t cap_num, uint32_t cap_den,
                                                uint32_t max_rounds, uint32_t *out_passes) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(cap_den > 0 && max_rounds > 0, "bad capacity factor / rounds");
        REQUIRE(use_affinity <= 1, "use_affinity must be 0 or 1");
        REQUIRE(!s->bs.active, "a bounded call is already in flight on this set (call _end first)");
        if (use_affinity) {
            REQUIRE(h->K > 0, "assign with object features needs node features");
            REQUIRE(s->K > 0 && s->K == h->K && s->feats.bytes >= s->n * (size_t)s->K * 4, "set features / node features missing or of different K");
            require_bounded_affinity_kernels();
        }
        require_weighted_kernels();
        const uint32_t *d_w = s->weights_or_null();
        const uint64_t L = weighted_load_total(global_weight_sum(h, local_weight_sum(h, d_w, s->n)), load_total);
        s->drop_lists();
        ensure_tab(h);
        set_ensure_counters(s);
        const uint32_t M = s->counters_n;
        s->loads.ensure((size_t)std::max(M, 1u) * 4, h->stream);
        const AffinityPath path = affinity_path(h);
        const uint32_t passes = bounded_weighted(h, s->bs, s->keys.as<uint64_t>(), s->feats.as<float>(), d_w, s->n, s->idx.as<uint32_t>(), s->loads.as<uint32_t>(), M,
                                                 s->sel.as<uint32_t>(), L, cap_num, cap_den, max_rounds, use_affinity != 0, path);
        // the counters stay object counts, whatever the rounds balanced
        set_zero_counters(s);
        launch_histogram(h->L(), s->idx.as<uint32_t>(), s->n, s->counters.as<uint32_t>(), M);
        if (use_affinity) record_plain_affinity(s, path);
        else s->plain_aff = false;
        s->assigned = true;
        CUDA_TRY(cudaStreamSynchronize(h->stream));
        if (use_affinity) record_affinity(s, path);
        s->bounded_w = true;
        s->bw_solver = h->solver;
        s->bw_bits = h->trie_bits;
        if (out_passes) *out_passes = passes;
    });
}

rio_status rio_cuda_set_loads(rio_objset *s, uint32_t *out, uint32_t cap) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        require_weighted_kernels();
        set_ensure_counters(s);
        const uint32_t M = s->counters_n;
        REQUIRE(out && cap >= M, "load buffer too small");
        if (!M) return;
        const uint32_t *d_w = s->weights_or_null();
        REQUIRE(global_weight_sum(h, local_weight_sum(h, d_w, s->n)) <= kMaxLoad, "the object weights of all ranks sum past 2^32-1 (loads are u32)");
        s->loads.ensure((size_t)M * 4, h->stream);
        CUDA_TRY(cudaMemsetAsync(s->loads.p, 0, (size_t)M * 4, h->stream));
        if (s->assigned) launch_load_histogram(h->L(), s->idx.as<uint32_t>(), d_w, s->n, s->loads.as<uint32_t>(), M);
        h->s_misc.ensure((size_t)M * 4, h->stream);
        exchange_counters(h, s->loads.as<uint32_t>(), h->s_misc.as<uint32_t>(), M);
        CUDA_TRY(cudaMemcpyAsync(out, h->s_misc.p, (size_t)M * 4, cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(cudaStreamSynchronize(h->stream));
    });
}

rio_status rio_cuda_set_rebalance(rio_objset *s, uint32_t event, uint32_t idx, uint64_t *out_moved) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(event == RIO_EV_JOIN || event == RIO_EV_LEAVE, "unknown event");
        REQUIRE(idx < h->nodes.size(), "node index out of range");
        REQUIRE(s->assigned, "set has no assignment yet");
        s->drop_lists();
        s->plain_aff = false;
        ensure_tab(h);
        set_ensure_counters(s);
        zero_scalar(h, S_MOVED);
        uint64_t moved = 0;
        if (h->solver == RIO_SOLVER_HRW2) {
            if (event == RIO_EV_JOIN) REQUIRE(h->nodes[idx].live(), "JOIN of a node that is not live");
            else REQUIRE(!h->nodes[idx].live(), "LEAVE of a node that is still live (deactivate it first)");
            // one streaming pass: walk every key again, write only the indices that changed, rebuild the counters
            set_zero_counters(s);
            launch_reassign_trie(h->L(), s->keys.as<uint64_t>(), s->n, h->tabs.trie, s->idx.as<uint32_t>(), s->counters.as<uint32_t>(), h->tabs.tab.n_total, h->d_scalars + S_MOVED);
            moved = read_scalar(h, S_MOVED);
        } else if (event == RIO_EV_JOIN) {
            REQUIRE(h->nodes[idx].live(), "JOIN of a node that is not live");
            launch_rebalance_join(h->L(), s->keys.as<uint64_t>(), s->idx.as<uint32_t>(), s->n, h->tabs.tab, idx, s->counters.as<uint32_t>(), h->d_scalars + S_MOVED);
            moved = read_scalar(h, S_MOVED);
        } else {
            REQUIRE(!h->nodes[idx].live(), "LEAVE of a node that is still live (deactivate it first)");
            zero_scalar(h, S_NSEL);
            launch_select_on_node(h->L(), s->idx.as<uint32_t>(), s->n, idx, s->sel.as<uint32_t>(), h->d_scalars + S_NSEL);
            moved = read_scalar(h, S_NSEL);
            CUDA_TRY(cudaMemsetAsync(s->counters.as<uint32_t>() + idx, 0, 4, h->stream));
            if (moved) run_assign(h, RIO_SOLVER_HRW, h->tabs, s->keys.as<uint64_t>(), s->n, s->idx.as<uint32_t>(), s->counters.as<uint32_t>(), s->sel.as<uint32_t>(), moved);
        }
        if (out_moved) *out_moved = moved;
    });
}

rio_status rio_cuda_set_rebalance_changes(rio_objset *s, const uint32_t *idx, const uint32_t *prev_weight, size_t k, uint64_t *out_moved) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        check_change_set(h, idx, prev_weight, k);
        REQUIRE(s->assigned, "set has no assignment yet");
        s->drop_lists();
        s->plain_aff = false;
        uint64_t moved = 0;
        if (k) {
            ensure_tab(h);
            set_ensure_counters(s);
            zero_scalar(h, S_MOVED);
            if (h->solver == RIO_SOLVER_HRW2) {   // one re-walk of every key, counters rebuilt, as rio_cuda_set_rebalance does
                set_zero_counters(s);
                launch_reassign_trie(h->L(), s->keys.as<uint64_t>(), s->n, h->tabs.trie, s->idx.as<uint32_t>(), s->counters.as<uint32_t>(), h->tabs.tab.n_total,
                                     h->d_scalars + S_MOVED);
            } else {
                require_change_kernels();
                const ChangeSetHost cs = build_change_set(h, idx, prev_weight, k);
                const ChangeSetDev dcs = upload_change_set(h, cs);
                h->s_idx2.ensure(std::max<uint64_t>(s->n, 1) * 4, h->stream);   // old node of each selected object
                zero_scalar(h, S_NSEL);
                launch_rebalance_changes(h->L(), s->keys.as<uint64_t>(), s->idx.as<uint32_t>(), s->n, h->tabs.tab, dcs, s->counters.as<uint32_t>(),
                                         s->sel.as<uint32_t>(), h->s_idx2.as<uint32_t>(), h->d_scalars + S_NSEL, h->d_scalars + S_MOVED);
                const uint64_t n_sel = read_scalar(h, S_NSEL);
                if (n_sel) {
                    run_assign(h, RIO_SOLVER_HRW, h->tabs, s->keys.as<uint64_t>(), s->n, s->idx.as<uint32_t>(), s->counters.as<uint32_t>(), s->sel.as<uint32_t>(), n_sel);
                    launch_count_changed(h->L(), s->idx.as<uint32_t>(), s->sel.as<uint32_t>(), h->s_idx2.as<uint32_t>(), n_sel, h->d_scalars + S_MOVED);
                }
            }
            moved = read_scalar(h, S_MOVED);
        }
        if (out_moved) *out_moved = moved;
    });
}

// ---- ranked resident sets (DESIGN.md 3.11) ----------------------------------------------------------------------------------
namespace {

void require_ranked_set_kernels(uint32_t solver) {
    const bool have = launch_ranked_primary && launch_assign_hrw_ranked && launch_assign_trie_ranked &&
                      (solver == RIO_SOLVER_HRW2 ? launch_reassign_trie_ranked != nullptr : launch_rebalance_changes_ranked && launch_scatter_ranked);
    if (!have) throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no ranked-set kernels (k_ranked_changes.cuh launchers are not linked)"};
}

void require_spread_set_kernels(uint32_t solver) {
    const bool have = launch_ranked_primary && launch_assign_hrw_spread && launch_assign_trie_spread &&
                      (solver == RIO_SOLVER_HRW2 ? launch_reassign_trie_spread != nullptr : launch_rebalance_changes_spread && launch_scatter_ranked);
    if (!have) throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no spread-set kernels (k_spread_changes.cuh launchers are not linked)"};
}

// the handle's labels become the set's snapshot (DESIGN.md 3.13)
void snapshot_labels(rio_objset *s) {
    const rio_placement *h = s->h;
    s->label_snap.resize(h->nodes.size());
    for (size_t j = 0; j < h->nodes.size(); j++) s->label_snap[j] = h->nodes[j].domain;
    s->label_snap_version = h->label_version;
}

// live nodes whose label differs from the set's snapshot; a node interned after the snapshot had RIO_NONE there
std::vector<uint32_t> relabelled_live(const rio_objset *s) {
    const rio_placement *h = s->h;
    std::vector<uint32_t> out;
    if (s->label_snap_version == h->label_version) return out;
    for (uint32_t j = 0; j < (uint32_t)h->nodes.size(); j++) {
        const uint32_t was = j < s->label_snap.size() ? s->label_snap[j] : RIO_NONE;
        if (h->nodes[j].domain != was && h->nodes[j].live()) out.push_back(j);
    }
    return out;
}

// ---- affinity resident sets (DESIGN.md 3.15) ------------------------------------------------------------------------------------
void require_affinity_set_kernels(bool spread) {
    const bool have = launch_ranked_primary && launch_scatter_ranked && launch_rebalance_changes_affinity && launch_gather_rows &&
                      (spread ? launch_assign_affinity_spread && launch_assign_affinity_umma_spread
                              : launch_assign_affinity_ranked && launch_assign_affinity_umma_ranked);
    if (!have) throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no affinity-set kernels (k_affinity_set.cuh launchers are not linked)"};
}

// the handle's node features, as the kernels see them (K floats per interned node, zeros for a row that is not K wide), become the
// set's snapshot
void snapshot_feats(rio_objset *s) {
    const rio_placement *h = s->h;
    const uint32_t K = h->K;
    s->feat_snap.assign(h->nodes.size() * K, 0.f);
    for (size_t j = 0; j < h->nodes.size(); j++)
        if (h->nodes[j].feat.size() == K) std::copy(h->nodes[j].feat.begin(), h->nodes[j].feat.end(), s->feat_snap.begin() + j * K);
    s->feat_snap_version = h->feat_version;
}

// the path, the handle's K and the node features a set's affinity result was computed under (the lists of 3.15, the bounded record of
// 3.17); with no live node the path is decided by what the handle would take for K == 16
void record_affinity(rio_objset *s, AffinityPath path) {
    s->aff_tensor = path == AffinityPath::kTensorCores || (path == AffinityPath::kNoLiveNode && affinity_umma_wanted());
    s->aff_K = s->h->K;
    snapshot_feats(s);
}

// live nodes whose feature row differs bitwise from the set's snapshot; a node interned after the snapshot counts as refeatured
std::vector<uint32_t> refeatured_live(const rio_objset *s) {
    const rio_placement *h = s->h;
    std::vector<uint32_t> out;
    if (s->feat_snap_version == h->feat_version) return out;
    const uint32_t K = s->aff_K;
    const size_t snap_n = s->feat_snap.size() / K;
    const std::vector<float> zeros(K, 0.f);
    for (uint32_t j = 0; j < (uint32_t)h->nodes.size(); j++) {
        const NodeInfo &ni = h->nodes[j];
        if (!ni.live()) continue;
        const float *now = ni.feat.size() == K ? ni.feat.data() : zeros.data();
        if (j >= snap_n || memcmp(now, s->feat_snap.data() + (size_t)j * K, (size_t)K * 4) != 0) out.push_back(j);
    }
    return out;
}

// The affinity change set of DESIGN.md 3.15: a live node's cost does not depend on its weight, so REPLACE is every interned node not
// live now and CANDIDATES every changed node live now that was not live before; a live -> live weight change is a no-op.  The
// refeatured (and, for failure-domain lists, relabelled) live nodes are added as REPLACE | CANDIDATE by the caller.
ChangeSetHost build_affinity_change_set(const rio_placement *h, const uint32_t *idx, const uint32_t *prev_weight, size_t k) {
    ChangeSetHost cs(h);
    for (size_t i = 0; i < k; i++)
        if (h->nodes[idx[i]].live() && !prev_weight[i]) cs.mark(idx[i], kChgCandidate);
    return cs;
}

// the kernels a resident set of `kind` needs (the hash kinds' depend on the handle's solver)
void require_set_kernels(ListKind kind, uint32_t solver) {
    if (is_affinity(kind)) require_affinity_set_kernels(is_spread(kind));
    else if (is_spread(kind)) require_spread_set_kernels(solver);
    else require_ranked_set_kernels(solver);
}

// set_assign_ranked (3.11), set_assign_ranked_spread (3.13) and set_assign_ranked_affinity(_spread) (3.15): fresh lists of `kind`, the
// affinity kinds on the path affinity_path() gives now, column 0 into idx, the counters rebuilt from it, and what the lists were
// computed under recorded: the policy, for the affinity kinds the path, K and node features, for the spread kinds the labels
void set_assign_lists(rio_objset *s, ListKind kind, uint32_t ranks) {
    rio_placement *h = s->h;
    const bool affinity = is_affinity(kind);
    check_ranked_args(s->n, ranks);
    if (affinity) {
        REQUIRE(h->K > 0, "assign with object features needs node features");
        REQUIRE(s->K > 0 && s->K == h->K && s->feats.bytes >= s->n * (size_t)s->K * 4, "set features / node features missing or of different K");
    }
    require_set_kernels(kind, h->solver);
    ensure_tab(h);
    s->drop_lists();
    s->lists.ensure(std::max<uint64_t>(s->capacity, 1) * ranks * 4, h->stream);
    set_ensure_counters(s);
    const AffinityPath path = affinity_path(h);
    run_lists(h, kind, affinity ? s->feats.p : s->keys.p, s->n, ranks, s->lists.as<uint32_t>(), path);
    launch_ranked_primary(h->L(), s->lists.as<uint32_t>(), s->n, ranks, s->idx.as<uint32_t>());
    set_zero_counters(s);
    launch_histogram(h->L(), s->idx.as<uint32_t>(), s->n, s->counters.as<uint32_t>(), s->counters_n);
    s->assigned = true;
    s->ranks = ranks;
    s->rank_solver = h->solver;
    s->rank_bits = h->trie_bits;
    s->kind = kind;
    if (affinity) record_affinity(s, path);
    if (is_spread(kind)) snapshot_labels(s);
}

// set_rebalance_changes_ranked (DESIGN.md 3.11, 3.13, 3.15): one pass classifies every list (S1 to s->sel, S2 rows merged with the
// candidates in place), then the S1 rows are computed afresh and scattered back; hash lists under HRW2 re-walk every key instead.
// The relabels (spread kinds) and refeatures (affinity kinds) since the set's snapshots belong to the change set.
void rebalance_lists(rio_objset *s, const uint32_t *idx, const uint32_t *prev_weight, size_t k, uint64_t &moved, uint64_t &changed) {
    rio_placement *h = s->h;
    const ListKind kind = s->kind;
    const bool affinity = is_affinity(kind), spread = is_spread(kind);
    const uint32_t R = s->ranks;
    const std::vector<uint32_t> refeatured = affinity ? refeatured_live(s) : std::vector<uint32_t>{};
    const std::vector<uint32_t> relabelled = spread ? relabelled_live(s) : std::vector<uint32_t>{};
    if (k || !refeatured.empty() || !relabelled.empty()) {
        ensure_tab(h);
        if (kind == ListKind::kSpread) ensure_spread_tab(h);
        if (kind == ListKind::kAffinitySpread) ensure_aff_dom(h);
        set_ensure_counters(s);
        zero_scalar(h, S_MOVED);
        zero_scalar(h, S_CHANGED);
        uint32_t *lists = s->lists.as<uint32_t>(), *d_idx = s->idx.as<uint32_t>(), *counters = s->counters.as<uint32_t>(), *sel = s->sel.as<uint32_t>();
        const uint64_t *keys = s->keys.as<uint64_t>();
        const uint32_t n_total = h->tabs.tab.n_total;
        unsigned long long *d_nsel = h->d_scalars + S_NSEL, *d_moved = h->d_scalars + S_MOVED, *d_changed = h->d_scalars + S_CHANGED;
        if (!affinity && h->solver == RIO_SOLVER_HRW2) {   // one ranked re-walk of every key, only the changed rows written
            if (spread) {
                launch_reassign_trie_spread(h->L(), keys, s->n, h->tabs.trie, h->spread_tab, R, lists, d_idx, counters, n_total, d_moved, d_changed);
            } else {
                ensure_rank_tab(h);
                launch_reassign_trie_ranked(h->L(), keys, s->n, h->tabs.trie, h->rank_tab, R, lists, d_idx, counters, n_total, d_moved, d_changed);
            }
        } else {
            ChangeSetHost cs = affinity ? build_affinity_change_set(h, idx, prev_weight, k) : build_change_set(h, idx, prev_weight, k);
            add_relabels(cs, refeatured);
            add_relabels(cs, relabelled);
            const ChangeSetDev dcs = upload_change_set(h, cs);
            zero_scalar(h, S_NSEL);
            if (kind == ListKind::kHash)
                launch_rebalance_changes_ranked(h->L(), keys, lists, R, d_idx, s->n, h->tabs.tab, dcs, counters, sel, d_nsel, d_moved, d_changed);
            else if (kind == ListKind::kSpread)
                launch_rebalance_changes_spread(h->L(), keys, lists, R, d_idx, s->n, h->tabs.tab, dcs, h->spread_tab, counters, sel, d_nsel, d_moved, d_changed);
            else
                launch_rebalance_changes_affinity(h->L(), s->feats.as<float>(), s->aff_K, lists, R, d_idx, s->n, h->d_fnode.as<float>(), n_total, dcs,
                                                  spread ? h->aff_dom.as<uint32_t>() : nullptr, counters, sel, d_nsel, d_moved, d_changed);
            const uint64_t n_sel = read_scalar(h, S_NSEL);
            if (n_sel) {   // S1: the selected objects' lists computed afresh, scattered back
                // the hash kinds on the flat kernels (the solver is HRW here), the affinity kinds on the recorded path
                h->s_idx.ensure(n_sel * R * 4, h->stream);
                const void *in;
                if (affinity) {
                    h->s_feats.ensure(n_sel * s->aff_K * 4, h->stream);
                    launch_gather_rows(h->L(), s->feats.as<float>(), s->aff_K, sel, n_sel, h->s_feats.as<float>());
                    in = h->s_feats.p;
                } else {
                    h->s_keys2.ensure(n_sel * 8, h->stream);
                    launch_gather_keys(h->L(), keys, sel, n_sel, h->s_keys2.as<uint64_t>(), nullptr, nullptr);
                    in = h->s_keys2.p;
                }
                run_lists(h, kind, in, n_sel, R, h->s_idx.as<uint32_t>(), affinity_path(h, s->aff_tensor));
                launch_scatter_ranked(h->L(), h->s_idx.as<uint32_t>(), sel, n_sel, R, lists, d_idx, counters, n_total, d_moved, d_changed);
            }
        }
        moved = read_scalar(h, S_MOVED);
        changed = read_scalar(h, S_CHANGED);
    }
    if (affinity) snapshot_feats(s);
    if (spread) snapshot_labels(s);
}

}  // namespace

rio_status rio_cuda_set_assign_ranked(rio_objset *s, uint32_t ranks) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    return guarded(s->h, [&] { set_assign_lists(s, ListKind::kHash, ranks); });
}

rio_status rio_cuda_set_assign_ranked_spread(rio_objset *s, uint32_t ranks) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    return guarded(s->h, [&] { set_assign_lists(s, ListKind::kSpread, ranks); });
}

rio_status rio_cuda_set_assign_ranked_affinity(rio_objset *s, uint32_t ranks) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    return guarded(s->h, [&] { set_assign_lists(s, ListKind::kAffinity, ranks); });
}

rio_status rio_cuda_set_assign_ranked_affinity_spread(rio_objset *s, uint32_t ranks) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    return guarded(s->h, [&] { set_assign_lists(s, ListKind::kAffinitySpread, ranks); });
}

rio_status rio_cuda_set_read_ranked(rio_objset *s, uint64_t first, uint64_t n, uint32_t *out) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(s->ranks, "set holds no ranked lists");
        REQUIRE(out, "null buffer");
        REQUIRE(first <= s->n && n <= s->n - first, "range outside the set");
        if (n) CUDA_TRY(cudaMemcpyAsync(out, s->lists.as<uint32_t>() + first * s->ranks, n * s->ranks * 4, cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(cudaStreamSynchronize(h->stream));
    });
}

rio_status rio_cuda_set_rebalance_changes_ranked(rio_objset *s, const uint32_t *idx, const uint32_t *prev_weight, size_t k, uint64_t *out_moved,
                                                 uint64_t *out_changed) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        check_change_set(h, idx, prev_weight, k);
        require_set_kernels(s->kind, h->solver);   // the hash kind's when the set holds no lists
        REQUIRE(s->ranks, "set holds no ranked lists");
        if (is_affinity(s->kind))   // affinity lists (DESIGN.md 3.15): the solver and trie_bits play no part
            REQUIRE(h->K == s->aff_K, "the set's affinity lists were computed under another node feature K: assign the lists again");
        else
            REQUIRE(s->rank_solver == h->solver && s->rank_bits == h->trie_bits, "the set's ranked lists were computed under another solver or trie_bits");
        uint64_t moved = 0, changed = 0;
        rebalance_lists(s, idx, prev_weight, k, moved, changed);
        if (out_moved) *out_moved = moved;
        if (out_changed) *out_changed = changed;
    });
}

// ---- bounded-load affinity sets kept through change sets (DESIGN.md 3.17) ---------------------------------------------------------
rio_status rio_cuda_set_rebalance_changes_bounded_affinity(rio_objset *s, const uint32_t *idx, const uint32_t *prev_weight, size_t k, uint64_t n_total,
                                                          uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds, uint64_t *out_moved, uint32_t *out_passes) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(s->bounded_aff, "set holds no bounded affinity assignment (set_assign_bounded_affinity first)");
        REQUIRE(h->K == s->aff_K, "the set's bounded affinity assignment was computed under another node feature K: assign it again");
        REQUIRE(s->K > 0 && s->K == h->K && s->feats.bytes >= s->n * (size_t)s->K * 4, "set features / node features missing or of different K");
        check_change_set(h, idx, prev_weight, k);
        REQUIRE(cap_den > 0 && max_rounds > 0, "bad capacity factor / rounds");
        REQUIRE(!s->bs.active, "a bounded call is already in flight on this set (call _end first)");
        require_bounded_affinity_kernels();
        if (!launch_rebalance_changes_bounded_affinity || !launch_count_diff)
            throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no bounded affinity change-set kernels (k_set_bounded_affinity.cuh launchers are not linked)"};
        ensure_tab(h);
        set_ensure_counters(s);   // a join may have interned a node
        const uint64_t n = s->n;
        const uint32_t K = s->aff_K, n_total_nodes = h->tabs.tab.n_total;
        uint32_t *d_idx = s->idx.as<uint32_t>(), *counters = s->counters.as<uint32_t>(), *d_sel = s->sel.as<uint32_t>();
        const float *d_feats = s->feats.as<float>();
        // pass 0: the change set of 3.15 (refeatured live nodes as REPLACE | CANDIDATE), S2 in place, S1 re-placed over the live set
        ChangeSetHost cs = build_affinity_change_set(h, idx, prev_weight, k);
        add_relabels(cs, refeatured_live(s));
        const ChangeSetDev dcs = upload_change_set(h, cs);
        const AffinityPath path = affinity_path(h, s->aff_tensor);
        h->s_idx.ensure(std::max<uint64_t>(n, 1) * 4, h->stream);   // each object's node before the call
        uint32_t *d_prev = h->s_idx.as<uint32_t>();
        zero_scalar(h, S_NSEL);
        launch_rebalance_changes_bounded_affinity(h->L(), d_feats, K, d_idx, d_prev, n, h->d_fnode.as<float>(), n_total_nodes, dcs, counters, d_sel,
                                                  h->d_scalars + S_NSEL);
        const uint64_t n_sel = read_scalar(h, S_NSEL);
        affinity_replace(h, path, nullptr, d_feats, d_sel, n_sel, d_idx, counters);
        // the rounds of 3.16 from the counters pass 0 left, spilled objects re-placed on the same path
        if (!n_total) n_total = n * (uint64_t)h->world;
        bounded_begin(h, s->bs, s->keys.as<uint64_t>(), n, d_idx, counters, s->counters_n, n_total, cap_num, cap_den, max_rounds, true, true, nullptr);
        const uint32_t passes = bounded_end(h, s->bs, s->keys.as<uint64_t>(), n, d_idx, counters, d_sel, [&](const std::vector<uint8_t> &closed, uint64_t nsel) {
            affinity_replace(h, path, &closed, d_feats, d_sel, nsel, d_idx, counters);
        });
        zero_scalar(h, S_MOVED);
        launch_count_diff(h->L(), d_idx, d_prev, n, h->d_scalars + S_MOVED);
        const uint64_t moved = read_scalar(h, S_MOVED);
        snapshot_feats(s);
        if (out_moved) *out_moved = moved;
        if (out_passes) *out_passes = passes;
    });
}

// ---- weighted bounded sets kept within load capacity (DESIGN.md 3.21) -----------------------------------------------------------
namespace {

void require_weight_key_kernels() {
    if (!launch_weight_keys_build || !launch_weight_keys_apply)
        throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no weighted change-set kernels (k_set_weighted_changes.cuh launchers are not linked)"};
}

// The HRW2 change set of 3.21, by weight: REPLACE is every interned node not live now (ChangeSetHost) and every changed live node that
// lost weight; CANDIDATES every changed live node that joined (prev_weight 0) or gained weight.
ChangeSetHost build_walk_change_set(const rio_placement *h, const uint32_t *idx, const uint32_t *prev_weight, size_t k) {
    ChangeSetHost cs(h);
    for (size_t i = 0; i < k; i++) {
        const NodeInfo &ni = h->nodes[idx[i]];
        if (!ni.live()) continue;   // REPLACE already
        if (prev_weight[i] && ni.weight < prev_weight[i]) cs.mark(idx[i], kChgReplace);
        else if (!prev_weight[i] || ni.weight > prev_weight[i]) cs.mark(idx[i], kChgCandidate);
    }
    return cs;
}

// Pass 0 under the hash policy, on the set's idx (counters not kept: the caller rebuilds them).  Flat HRW: R1 / R2 of 3.10.  HRW2 with
// candidates: one walk of every key into s_idx2, merged by launch_merge_walk_changes; without: the S1 objects selected and walked.
void hash_changes_pass0(rio_objset *s, const uint32_t *idx, const uint32_t *prev_weight, size_t k) {
    rio_placement *h = s->h;
    const bool trie = h->solver == RIO_SOLVER_HRW2;
    const ChangeSetHost cs = trie ? build_walk_change_set(h, idx, prev_weight, k) : build_change_set(h, idx, prev_weight, k);
    const ChangeSetDev dcs = upload_change_set(h, cs);
    const uint64_t n = s->n;
    const uint64_t *keys = s->keys.as<uint64_t>();
    uint32_t *d_idx = s->idx.as<uint32_t>(), *d_sel = s->sel.as<uint32_t>();
    h->s_idx2.ensure(std::max<uint64_t>(n, 1) * 4, h->stream);   // the walk of every key, or the old node of each selected object
    if (trie && cs.n_cand) {
        run_assign(h, RIO_SOLVER_HRW2, h->tabs, keys, n, h->s_idx2.as<uint32_t>(), nullptr, nullptr, 0);
        launch_merge_walk_changes(h->L(), d_idx, h->s_idx2.as<uint32_t>(), n, dcs.flag, h->tabs.tab.n_total);
        return;
    }
    zero_scalar(h, S_NSEL);
    launch_rebalance_changes(h->L(), keys, d_idx, n, h->tabs.tab, dcs, nullptr, d_sel, h->s_idx2.as<uint32_t>(), h->d_scalars + S_NSEL, h->d_scalars + S_MOVED);
    const uint64_t n_sel = read_scalar(h, S_NSEL);
    if (n_sel) run_assign(h, h->solver, h->tabs, keys, n, d_idx, nullptr, d_sel, n_sel);
}

}  // namespace

rio_status rio_cuda_set_write_weights_by_key(rio_objset *s, const uint64_t *keys, const uint32_t *w, size_t m, uint64_t *out_written) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE((keys && w) || !m, "null keys or weights");
        REQUIRE(!s->bs.active, "a bounded call is in flight on this set (call _end first)");
        if (out_written) *out_written = 0;
        if (!m) return;
        require_weight_key_kernels();
        REQUIRE(m < 0xFFFFFFFFull, "too many keys (positions are u32)");
        cudaStream_t st = h->stream;
        // one allocation: the table's keys (1 << lg slots, at least 2m), their positions, then the position of a key equal to ~0
        uint32_t lg = 6;
        while ((1ull << lg) < 2 * (uint64_t)m) lg++;
        const size_t o_pos = (size_t)8 << lg, o_empty = o_pos + ((size_t)4 << lg);
        h->s_churn.ensure(o_empty + 16, st);
        unsigned char *base = h->s_churn.as<unsigned char>();
        CUDA_TRY(cudaMemsetAsync(base, 0xFF, o_pos, st));   // kEmptyKey
        CUDA_TRY(cudaMemsetAsync(base + o_pos, 0, o_empty + 16 - o_pos, st));
        h->s_keys.ensure(m * 8, st);
        h->s_weights.ensure(m * 4, st);
        CUDA_TRY(cudaMemcpyAsync(h->s_keys.p, keys, m * 8, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(h->s_weights.p, w, m * 4, cudaMemcpyHostToDevice, st));
        if (!s->has_weights) {   // first write: the column, every row 1, as set_write_weights allocates it
            s->weights.ensure(s->capacity * 4, st);
            launch_fill_u32(h->L(), s->weights.as<uint32_t>(), s->n, 1u);
            s->has_weights = true;
        }
        unsigned long long *table = reinterpret_cast<unsigned long long *>(base);
        uint32_t *pos = reinterpret_cast<uint32_t *>(base + o_pos), *empty_pos = reinterpret_cast<uint32_t *>(base + o_empty);
        launch_weight_keys_build(h->L(), h->s_keys.as<uint64_t>(), m, table, pos, lg, empty_pos);
        zero_scalar(h, S_MOVED);
        launch_weight_keys_apply(h->L(), s->keys.as<uint64_t>(), s->n, table, pos, lg, empty_pos, h->s_weights.as<uint32_t>(), s->weights.as<uint32_t>(),
                                 h->d_scalars + S_MOVED);
        const uint64_t written = read_scalar(h, S_MOVED);
        if (out_written) *out_written = written;
    });
}

rio_status rio_cuda_set_rebalance_changes_bounded_weighted(rio_objset *s, const uint32_t *idx, const uint32_t *prev_weight, size_t k, uint64_t load_total,
                                                          uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds, uint64_t *out_moved, uint32_t *out_passes) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        // argument errors, decided on each rank before any exchange
        REQUIRE(s->bounded_w, "set holds no weighted bounded assignment (set_assign_bounded_weighted first)");
        const bool affinity = s->plain_aff;
        if (affinity) {
            REQUIRE(h->K == s->aff_K, "the set's weighted bounded assignment was computed under another node feature K: assign it again");
            REQUIRE(s->K > 0 && s->K == h->K && s->feats.bytes >= s->n * (size_t)s->K * 4, "set features / node features missing or of different K");
        } else {
            REQUIRE(s->bw_solver == h->solver && s->bw_bits == h->trie_bits, "the set's weighted bounded assignment was computed under another solver or trie_bits");
        }
        check_change_set(h, idx, prev_weight, k);
        REQUIRE(cap_den > 0 && max_rounds > 0, "bad capacity factor / rounds");
        REQUIRE(!s->bs.active, "a bounded call is already in flight on this set (call _end first)");
        require_weighted_kernels();
        if (!launch_merge_walk_changes || !launch_rebalance_changes || !launch_count_diff || (affinity && !launch_rebalance_changes_bounded_affinity))
            throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no weighted change-set kernels (k_set_weighted_changes.cuh, k_changes.cuh or "
                                             "k_set_bounded_affinity.cuh launchers are not linked)"};
        if (affinity) require_bounded_affinity_kernels();
        // range errors, decided from the global weight sum, so that every rank refuses together
        const uint32_t *d_w = s->weights_or_null();
        const uint64_t L = weighted_load_total(global_weight_sum(h, local_weight_sum(h, d_w, s->n)), load_total);
        ensure_tab(h);
        set_ensure_counters(s);   // a join may have interned a node
        const uint64_t n = s->n;
        const uint32_t M = s->counters_n;
        s->loads.ensure((size_t)std::max(M, 1u) * 4, h->stream);
        uint32_t *d_idx = s->idx.as<uint32_t>(), *counters = s->counters.as<uint32_t>(), *d_sel = s->sel.as<uint32_t>();
        const float *d_feats = s->feats.as<float>();
        h->s_idx.ensure(std::max<uint64_t>(n, 1) * 4, h->stream);   // each object's node before the call
        uint32_t *d_prev = h->s_idx.as<uint32_t>();
        const AffinityPath path = affinity ? affinity_path(h, s->aff_tensor) : affinity_path(h);
        if (affinity) {   // pass 0 of 3.17: the change set of 3.15 with the refeatured live nodes, S2 in place, S1 over the live set
            ChangeSetHost cs = build_affinity_change_set(h, idx, prev_weight, k);
            add_relabels(cs, refeatured_live(s));
            const ChangeSetDev dcs = upload_change_set(h, cs);
            zero_scalar(h, S_NSEL);
            launch_rebalance_changes_bounded_affinity(h->L(), d_feats, s->aff_K, d_idx, d_prev, n, h->d_fnode.as<float>(), h->tabs.tab.n_total, dcs, counters,
                                                      d_sel, h->d_scalars + S_NSEL);
            affinity_replace(h, path, nullptr, d_feats, d_sel, read_scalar(h, S_NSEL), d_idx, counters);
        } else {
            CUDA_TRY(cudaMemcpyAsync(d_prev, d_idx, n * 4, cudaMemcpyDeviceToDevice, h->stream));
            if (k) hash_changes_pass0(s, idx, prev_weight, k);
        }
        const uint32_t passes = weighted_rounds(h, s->bs, s->keys.as<uint64_t>(), d_feats, d_w, n, d_idx, s->loads.as<uint32_t>(), M, d_sel, L, cap_num, cap_den,
                                                max_rounds, affinity, path);
        // the counters stay object counts, whatever the rounds balanced
        set_zero_counters(s);
        launch_histogram(h->L(), d_idx, n, counters, M);
        zero_scalar(h, S_MOVED);
        launch_count_diff(h->L(), d_idx, d_prev, n, h->d_scalars + S_MOVED);
        const uint64_t moved = read_scalar(h, S_MOVED);
        if (affinity) snapshot_feats(s);
        if (out_moved) *out_moved = moved;
        if (out_passes) *out_passes = passes;
    });
}

// ---- object churn in resident sets (DESIGN.md 3.18) ---------------------------------------------------------------------------
namespace {

void require_churn_kernels() {
    if (!launch_churn_build || !launch_churn_mark || !launch_churn_pairs || !launch_churn_move)
        throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no set churn kernels (k_set_churn.cuh launchers are not linked)"};
}

// b grows to hold `need` bytes with its first `keep` bytes kept (DevBuf::ensure keeps nothing); at most `limit` bytes unless need is more
void grow_keeping(rio_placement *h, DevBuf &b, size_t need, size_t keep, size_t limit) {
    if (need <= b.bytes) return;
    DevBuf nb;
    nb.ensure(std::max(need, std::min(limit, b.bytes + b.bytes / 2)), h->stream);
    if (keep) CUDA_TRY(cudaMemcpyAsync(nb.p, b.p, keep, cudaMemcpyDeviceToDevice, h->stream));
    b.release(h->stream);
    b = nb;
}

// The m new rows' idx (and list rows) as the set's current kind places a fresh object, computed on the staged keys / feature rows into
// the handle's scratch, never on the set's columns at row n: the HRW2 walk and the K = 16 kernels read their inputs in 16-byte pieces.
// Returns the m indices on the device; their counters are added.  Lists go straight to rows [n, n + m) of s->lists.
const uint32_t *place_new_rows(rio_objset *s, const uint64_t *d_keys, const float *d_feats, uint64_t m) {
    rio_placement *h = s->h;
    cudaStream_t st = h->stream;
    uint32_t *counters = s->counters.as<uint32_t>();
    h->s_idx.ensure(m * std::max(s->ranks, 1u) * 4, st);
    uint32_t *out = h->s_idx.as<uint32_t>();
    if (s->ranks) {   // the batch call of the list kind, over the current table; an affinity kind on its recorded path
        const ListKind kind = s->kind;
        const uint32_t R = s->ranks;
        run_lists(h, kind, is_affinity(kind) ? (const void *)d_feats : (const void *)d_keys, m, R, out, affinity_path(h, s->aff_tensor));
        CUDA_TRY(cudaMemcpyAsync(s->lists.as<uint32_t>() + s->n * R, out, m * R * 4, cudaMemcpyDeviceToDevice, st));
        h->s_sel.ensure(m * 4, st);
        launch_ranked_primary(h->L(), out, m, R, h->s_sel.as<uint32_t>());
        launch_histogram(h->L(), h->s_sel.as<uint32_t>(), m, counters, s->counters_n);
        return h->s_sel.as<uint32_t>();
    }
    if (s->bounded_aff) run_affinity(h, d_feats, m, out, nullptr, counters, affinity_path(h, s->aff_tensor));
    else if (s->plain_aff) run_affinity(h, d_feats, m, out, nullptr, counters, affinity_path(h, s->plain_tensor));
    else run_assign(h, h->solver, h->tabs, d_keys, m, out, counters, nullptr, 0);
    return out;
}

}  // namespace

rio_status rio_cuda_set_insert(rio_objset *s, const uint64_t *keys, const float *feats, uint64_t m, uint64_t *out_first) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(keys || !m, "null keys");
        if (out_first) *out_first = s->n;
        if (!m) return;
        REQUIRE(s->K ? feats != nullptr : feats == nullptr, s->K ? "the set has features: insert needs the new rows' features"
                                                                  : "the set has no features: insert takes none");
        REQUIRE(m <= s->capacity - s->n, "n + m exceeds the set's capacity");
        REQUIRE(!s->bs.active, "a bounded call is in flight on this set (call _end first)");
        require_churn_kernels();
        const bool lists = s->assigned && s->ranks;
        if (lists && is_affinity(s->kind))
            REQUIRE(h->K == s->aff_K, "the set's affinity lists were computed under another node feature K: assign the lists again");
        else if (lists)
            REQUIRE(s->rank_solver == h->solver && s->rank_bits == h->trie_bits, "the set's ranked lists were computed under another solver or trie_bits");
        else if (s->assigned && s->bounded_aff)
            REQUIRE(h->K == s->aff_K, "the set's bounded affinity assignment was computed under another node feature K: assign it again");
        else if (s->assigned && s->plain_aff)
            REQUIRE(h->K == s->K, "the set's affinity assignment was computed under another node feature K: assign it again");
        if (lists && !launch_ranked_primary)
            throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no ranked-set kernels (k_ranked_changes.cuh launchers are not linked)"};
        cudaStream_t st = h->stream;
        const uint64_t n = s->n;
        const size_t K = s->K;
        h->s_keys.ensure(m * 8, st);
        CUDA_TRY(cudaMemcpyAsync(h->s_keys.p, keys, m * 8, cudaMemcpyHostToDevice, st));
        if (K) {
            h->s_feats.ensure(m * K * 4, st);
            CUDA_TRY(cudaMemcpyAsync(h->s_feats.p, feats, m * K * 4, cudaMemcpyHostToDevice, st));
            grow_keeping(h, s->feats, (n + m) * K * 4, std::min(s->feats.bytes, n * K * 4), s->capacity * K * 4);
        }
        if (s->assigned) {
            ensure_tab(h);
            set_ensure_counters(s);
            const uint32_t *d_new = place_new_rows(s, h->s_keys.as<uint64_t>(), h->s_feats.as<float>(), m);
            CUDA_TRY(cudaMemcpyAsync(s->idx.as<uint32_t>() + n, d_new, m * 4, cudaMemcpyDeviceToDevice, st));
        } else {
            CUDA_TRY(cudaMemsetAsync(s->idx.as<uint32_t>() + n, 0xFF, m * 4, st));   // RIO_NONE
        }
        CUDA_TRY(cudaMemcpyAsync(s->keys.as<uint64_t>() + n, h->s_keys.p, m * 8, cudaMemcpyDeviceToDevice, st));
        if (K) CUDA_TRY(cudaMemcpyAsync(s->feats.as<float>() + n * K, h->s_feats.p, m * K * 4, cudaMemcpyDeviceToDevice, st));
        if (s->has_weights) launch_fill_u32(h->L(), s->weights.as<uint32_t>() + n, m, 1u);   // the caller writes the real weights at n
        CUDA_TRY(cudaStreamSynchronize(st));
        s->n = n + m;
    });
}

rio_status rio_cuda_set_erase(rio_objset *s, const uint64_t *keys, uint64_t m, uint64_t *out_erased) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(keys || !m, "null keys");
        if (out_erased) *out_erased = 0;
        if (!m) return;
        REQUIRE(!s->bs.active, "a bounded call is in flight on this set (call _end first)");
        require_churn_kernels();
        if (s->has_weights && !launch_churn_move_weights)   // the weight column must move with its rows: refuse rather than split them
            throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no weighted bounded kernels (k_bounded_weighted.cuh launchers are not linked): "
                                             "erase cannot move the set's weight column"};
        const uint64_t n = s->n;
        if (!n) return;
        cudaStream_t st = h->stream;
        if (s->assigned) set_ensure_counters(s);
        // one allocation: the hash set (1 << lg slots, at least 2m), its empty-key flag, then per block of kChurnRows rows the flagged
        // count, the hole offset and the mover offset, then a flag byte per row
        uint32_t lg = 6;
        while ((1ull << lg) < 2 * m) lg++;
        const uint64_t nb = (n + kChurnRows - 1) / kChurnRows;
        const size_t o_flag = (size_t)8 << lg, o_cnt = o_flag + 16, o_hoff = o_cnt + nb * 4, o_moff = o_hoff + nb * 4, o_row = o_moff + nb * 4,
                     total = o_row + n;
        h->s_churn.ensure(total, st);
        unsigned char *base = h->s_churn.as<unsigned char>();
        unsigned long long *table = reinterpret_cast<unsigned long long *>(base);
        uint32_t *has_empty = reinterpret_cast<uint32_t *>(base + o_flag), *cnt = reinterpret_cast<uint32_t *>(base + o_cnt);
        CUDA_TRY(cudaMemsetAsync(table, 0xFF, o_flag, st));   // kEmptyKey
        CUDA_TRY(cudaMemsetAsync(has_empty, 0, 4, st));
        h->s_keys.ensure(m * 8, st);
        CUDA_TRY(cudaMemcpyAsync(h->s_keys.p, keys, m * 8, cudaMemcpyHostToDevice, st));
        launch_churn_build(h->L(), h->s_keys.as<uint64_t>(), m, table, lg, has_empty);
        zero_scalar(h, S_MOVED);
        launch_churn_mark(h->L(), s->keys.as<uint64_t>(), s->idx.as<uint32_t>(), n, table, lg, has_empty, s->assigned ? s->counters.as<uint32_t>() : nullptr,
                          s->counters_n, base + o_row, cnt, h->d_scalars + S_MOVED);
        const uint64_t erased = read_scalar(h, S_MOVED);
        const uint64_t n_new = n - erased, max_pairs = std::min(erased, n_new);
        if (max_pairs) {
            h->s_idx.ensure(max_pairs * 4, st);
            h->s_idx2.ensure(max_pairs * 4, st);
            zero_scalar(h, S_NSEL);
            launch_churn_pairs(h->L(), base + o_row, n, n_new, cnt, reinterpret_cast<uint32_t *>(base + o_hoff), reinterpret_cast<uint32_t *>(base + o_moff),
                               h->s_idx.as<uint32_t>(), h->s_idx2.as<uint32_t>(), h->d_scalars + S_NSEL);
            const bool feats = s->K && s->feats.bytes >= n * (size_t)s->K * 4;   // feature rows that cover the set move with it
            launch_churn_move(h->L(), h->s_idx.as<uint32_t>(), h->s_idx2.as<uint32_t>(), max_pairs, h->d_scalars + S_NSEL, s->keys.as<uint64_t>(),
                              s->idx.as<uint32_t>(), s->ranks ? s->lists.as<uint32_t>() : nullptr, s->ranks, feats ? s->feats.as<float>() : nullptr, s->K);
            if (s->has_weights)
                launch_churn_move_weights(h->L(), h->s_idx.as<uint32_t>(), h->s_idx2.as<uint32_t>(), max_pairs, h->d_scalars + S_NSEL, s->weights.as<uint32_t>());
            CUDA_TRY(cudaStreamSynchronize(st));
        }
        s->n = n_new;
        if (out_erased) *out_erased = erased;
    });
}

rio_status rio_cuda_set_counters(rio_objset *s, uint32_t *out, uint32_t cap) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        set_ensure_counters(s);
        const uint32_t M = s->counters_n;
        REQUIRE(out && cap >= M, "counter buffer too small");
        if (!M) return;
        h->s_misc.ensure((size_t)M * 4, h->stream);
        exchange_counters(h, s->counters.as<uint32_t>(), h->s_misc.as<uint32_t>(), M);
        CUDA_TRY(cudaMemcpyAsync(out, h->s_misc.p, (size_t)M * 4, cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(cudaStreamSynchronize(h->stream));
    });
}

rio_status rio_cuda_set_read(rio_objset *s, uint64_t first, uint64_t n, uint64_t *out_keys, uint32_t *out_idx) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(first + n <= s->n, "range outside the set");
        if (out_keys && n) CUDA_TRY(cudaMemcpyAsync(out_keys, s->keys.as<uint64_t>() + first, n * 8, cudaMemcpyDeviceToHost, h->stream));
        if (out_idx && n) CUDA_TRY(cudaMemcpyAsync(out_idx, s->idx.as<uint32_t>() + first, n * 4, cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(cudaStreamSynchronize(h->stream));
    });
}

rio_status rio_cuda_set_size(rio_objset *s, uint64_t *out_n) {
    if (!s || !out_n) { g_last_error = "null argument"; return RIO_ERR_UNKNOWN; }
    *out_n = s->n;
    return RIO_OK;
}

rio_status rio_cuda_set_commit(rio_objset *s) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(s->assigned, "set has no assignment yet");
        dir_reserve(h, s->n);
        dir_upsert_dev(h, s->keys.as<uint64_t>(), s->idx.as<uint32_t>(), 0, s->n);
        reconcile_dir_keys(h);
        check_device_error(h);
    });
}

rio_status rio_cuda_set_commit_changes(rio_objset *s, uint32_t dry_run, uint64_t cap, uint64_t *out_rows, uint64_t *out_keys, uint32_t *out_from,
                                       uint32_t *out_to, uint64_t *out_n) {
    if (!s) { g_last_error = "null set"; return RIO_ERR_UNKNOWN; }
    rio_placement *h = s->h;
    return guarded(h, [&] {
        REQUIRE(s->assigned, "set has no assignment yet");
        REQUIRE(!s->bs.active, "a bounded call is in flight on this set (call _end first)");
        if (!launch_commit_diff || !launch_commit_list)
            throw RioError{RIO_ERR_UPSTREAM, "this build of the engine has no set commit kernels (k_set_commit.cuh launchers are not linked)"};
        const uint64_t n = s->n;
        const bool want = out_rows || out_keys || out_from || out_to;
        if (!n) { if (out_n) *out_n = 0; return; }
        cudaStream_t st = h->stream;
        // one allocation: per block of kCommitRows rows the selected count and its offset, then per row the directory's answer (written
        // for selected rows only) and a flag byte
        const uint64_t nb = (n + kCommitRows - 1) / kCommitRows;
        const size_t o_off = nb * 4, o_from = (o_off + nb * 4 + 15) & ~(size_t)15, o_flag = o_from + n * 4, total = o_flag + n;
        h->s_commit.ensure(total, st);
        unsigned char *base = h->s_commit.as<unsigned char>();
        uint32_t *cnt = reinterpret_cast<uint32_t *>(base), *off = reinterpret_cast<uint32_t *>(base + o_off), *from = reinterpret_cast<uint32_t *>(base + o_from);
        uint8_t *flag = base + o_flag;
        launch_commit_diff(h->L(), h->dir, s->keys.as<uint64_t>(), s->idx.as<uint32_t>(), n, flag, from, cnt, off, h->d_scalars + S_NSEL);
        const uint64_t m = read_scalar(h, S_NSEL);   // the call's one synchronisation before the write
        if (out_n) *out_n = m;
        REQUIRE(!want || m <= cap, "the manifest has more entries than cap (*out_n holds its size)");
        if (!m || (dry_run && !want)) return;
        // the manifest: rows (u64), keys (u64), from (u32), to (u32), m entries each
        h->s_manifest.ensure(m * 24, st);
        uint64_t *d_rows = h->s_manifest.as<uint64_t>(), *d_keys = d_rows + m;
        uint32_t *d_from = reinterpret_cast<uint32_t *>(d_keys + m), *d_to = d_from + m;
        launch_commit_list(h->L(), s->keys.as<uint64_t>(), s->idx.as<uint32_t>(), n, flag, from, cnt, off, d_rows, d_keys, d_from, d_to);
        if (!dry_run) {   // row order: among selected rows of one key the last wins, as in every upsert batch
            dir_reserve(h, m);
            dir_upsert_dev(h, d_keys, d_to, 0, m);
        }
        if (out_rows) CUDA_TRY(cudaMemcpyAsync(out_rows, d_rows, m * 8, cudaMemcpyDeviceToHost, st));
        if (out_keys) CUDA_TRY(cudaMemcpyAsync(out_keys, d_keys, m * 8, cudaMemcpyDeviceToHost, st));
        if (out_from) CUDA_TRY(cudaMemcpyAsync(out_from, d_from, m * 4, cudaMemcpyDeviceToHost, st));
        if (out_to) CUDA_TRY(cudaMemcpyAsync(out_to, d_to, m * 4, cudaMemcpyDeviceToHost, st));
        if (dry_run) {
            CUDA_TRY(cudaStreamSynchronize(st));
        } else {
            reconcile_dir_keys(h);
            check_device_error(h);
        }
    });
}

// ---- multi-GPU ---------------------------------------------------------------------------------------------------------
rio_status rio_cuda_comm_unique_id(uint8_t out_id[RIO_COMM_ID_BYTES]) {
    return guarded(nullptr, [&] {
        std::lock_guard<std::mutex> g(g_nccl_mu);
        if (!g_nccl.load()) throw RioError{RIO_ERR_UPSTREAM, "cannot load libnccl: " + g_nccl.load_error};
        NcclId id;
        NCCL_TRY(g_nccl.GetUniqueId(&id));
        memcpy(out_id, id.internal, RIO_COMM_ID_BYTES);
    });
}

rio_status rio_cuda_comm_init(rio_placement *h, int32_t rank, int32_t world, const uint8_t id[RIO_COMM_ID_BYTES]) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(world >= 1 && rank >= 0 && rank < world && id, "bad rank/world");
        {
            std::lock_guard<std::mutex> g(g_nccl_mu);
            if (!g_nccl.load()) throw RioError{RIO_ERR_UPSTREAM, "cannot load libnccl: " + g_nccl.load_error};
        }
        if (h->comm) { g_nccl.CommDestroy(h->comm); h->comm = nullptr; }
        NcclId nid;
        memcpy(nid.internal, id, RIO_COMM_ID_BYTES);
        NCCL_TRY(g_nccl.CommInitRank(&h->comm, world, nid, rank));
        h->rank = rank; h->world = world;
    });
}

/* Peer-memory exchange: export this rank's window, then attach every rank's handle (gathered by the host bootstrap). */
rio_status rio_cuda_comm_ipc_export(rio_placement *h, int32_t world, uint32_t max_nodes, uint8_t out_handle[RIO_IPC_HANDLE_BYTES]) {
    if (!h || !out_handle) { g_last_error = "null argument"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(world >= 1 && world <= 16 && max_nodes > 0, "bad world / max_nodes (at most 16 ranks)");
        static_assert(sizeof(cudaIpcMemHandle_t) <= RIO_IPC_HANDLE_BYTES, "IPC handle does not fit");
        if (h->xchg_mine) { CUDA_TRY(cudaStreamSynchronize(h->stream)); CUDA_TRY(cudaFree(h->xchg_mine)); h->xchg_mine = nullptr; h->xchg_ready = false; }
        const size_t words = (size_t)2 * world * max_nodes + world;
        CUDA_TRY(cudaMalloc(reinterpret_cast<void **>(&h->xchg_mine), words * 4));   // cudaMalloc (not the async pool): IPC needs a plain allocation
        CUDA_TRY(cudaMemset(h->xchg_mine, 0, words * 4));
        h->xchg_nodes = max_nodes;
        h->xchg_epoch = 0;
        cudaIpcMemHandle_t hd;
        CUDA_TRY(cudaIpcGetMemHandle(&hd, h->xchg_mine));
        memset(out_handle, 0, RIO_IPC_HANDLE_BYTES);
        memcpy(out_handle, &hd, sizeof hd);
    });
}

rio_status rio_cuda_comm_ipc_attach(rio_placement *h, int32_t rank, int32_t world, const uint8_t *handles) {
    if (!h || !handles) { g_last_error = "null argument"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(world >= 1 && world <= 16 && rank >= 0 && rank < world && h->xchg_mine, "export the window first / bad rank");
        for (int p = 0; p < world; p++) {
            if (p == rank) { h->xchg_peer[p] = h->xchg_mine; continue; }
            cudaIpcMemHandle_t hd;
            memcpy(&hd, handles + (size_t)p * RIO_IPC_HANDLE_BYTES, sizeof hd);
            void *ptr = nullptr;
            CUDA_TRY(cudaIpcOpenMemHandle(&ptr, hd, cudaIpcMemLazyEnablePeerAccess));
            h->xchg_peer[p] = reinterpret_cast<uint32_t *>(ptr);
        }
        h->rank = rank; h->world = world;
        h->xchg_ready = true;
    });
}

rio_status rio_cuda_comm_info(rio_placement *h, int32_t *rank, int32_t *world) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    if (rank) *rank = h->rank;
    if (world) *world = h->world;
    return RIO_OK;
}

rio_status rio_cuda_comm_sum_counters(rio_placement *h, uint32_t *inout, uint32_t M) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        if (!M) return;
        REQUIRE(inout, "null buffer");
        h->s_misc.ensure((size_t)M * 8, h->stream);
        uint32_t *d_in = h->s_misc.as<uint32_t>(), *d_out = d_in + M;
        CUDA_TRY(cudaMemcpyAsync(d_in, inout, (size_t)M * 4, cudaMemcpyHostToDevice, h->stream));
        exchange_counters(h, d_in, d_out, M);
        CUDA_TRY(cudaMemcpyAsync(inout, d_out, (size_t)M * 4, cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(cudaStreamSynchronize(h->stream));
    });
}

// ---- device memory / timing helpers --------------------------------------------------------------------------------
rio_status rio_cuda_dev_alloc(rio_placement *h, size_t bytes, void **out_dev) {
    if (!h || !out_dev) { g_last_error = "null argument"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { CUDA_TRY(cudaMalloc(out_dev, bytes ? bytes : 1)); });
}
rio_status rio_cuda_dev_free(rio_placement *h, void *dev) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { CUDA_TRY(cudaStreamSynchronize(h->stream)); if (dev) CUDA_TRY(cudaFree(dev)); });
}
rio_status rio_cuda_host_alloc(rio_placement *h, size_t bytes, void **out_pinned) {
    if (!h || !out_pinned) { g_last_error = "null argument"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { CUDA_TRY(cudaMallocHost(out_pinned, bytes ? bytes : 1)); });
}
rio_status rio_cuda_host_free(rio_placement *h, void *pinned) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { if (pinned) CUDA_TRY(cudaFreeHost(pinned)); });
}
rio_status rio_cuda_memcpy_h2d(rio_placement *h, void *dev, const void *host, size_t bytes) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { if (bytes) CUDA_TRY(cudaMemcpyAsync(dev, host, bytes, cudaMemcpyHostToDevice, h->stream)); });
}
rio_status rio_cuda_memcpy_d2h(rio_placement *h, void *host, const void *dev, size_t bytes) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { if (bytes) CUDA_TRY(cudaMemcpyAsync(host, dev, bytes, cudaMemcpyDeviceToHost, h->stream)); });
}
rio_status rio_cuda_flush_l2(rio_placement *h) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        const size_t words = (size_t)64 << 20;   // 256 MiB > 50 MB of L2
        h->s_flush.ensure(words * 4, h->stream);
        static uint32_t v = 0;
        launch_l2_flush(h->L(), h->s_flush.as<uint32_t>(), words, ++v);
    });
}
rio_status rio_cuda_bench_mix_rate(rio_placement *h, uint32_t iters, double *out_pairs_per_s) {
    if (!h || !out_pairs_per_s) { g_last_error = "null argument"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        h->s_misc.ensure(4096, h->stream);
        {   // opaque per-object constants for the probe
            std::vector<uint32_t> seed(1024);
            for (uint32_t i = 0; i < 1024; i++) seed[i] = (uint32_t)mix64(i + 1);
            CUDA_TRY(cudaMemcpyAsync(h->s_misc.p, seed.data(), 4096, cudaMemcpyHostToDevice, h->stream));
            CUDA_TRY(cudaStreamSynchronize(h->stream));
        }
        launch_mix_rate(h->L(), 16, h->s_misc.as<uint32_t>());   // warm-up
        CUDA_TRY(cudaEventRecord(h->events[RIO_MAX_EVENTS - 2], h->stream));
        const uint64_t pairs = launch_mix_rate(h->L(), iters ? iters : 1, h->s_misc.as<uint32_t>());
        CUDA_TRY(cudaEventRecord(h->events[RIO_MAX_EVENTS - 1], h->stream));
        CUDA_TRY(cudaEventSynchronize(h->events[RIO_MAX_EVENTS - 1]));
        float ms = 0;
        CUDA_TRY(cudaEventElapsedTime(&ms, h->events[RIO_MAX_EVENTS - 2], h->events[RIO_MAX_EVENTS - 1]));
        *out_pairs_per_s = (double)pairs / ((double)ms * 1e-3);
    });
}
/* development hook, deliberately not in include/rio_cuda.h: per-CTA cycle counters of the tensor-core affinity kernel */
rio_status rio_dev_umma_timing(rio_placement *h, unsigned long long *d_buf) {
    if (!h) return RIO_ERR_UNKNOWN;
    return guarded(h, [&] { CUDA_TRY(cudaStreamSynchronize(h->stream)); affinity_umma_set_timing_buffer(d_buf); });
}
rio_status rio_cuda_event_record(rio_placement *h, uint32_t slot) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] { REQUIRE(slot < RIO_MAX_EVENTS, "event slot out of range"); CUDA_TRY(cudaEventRecord(h->events[slot], h->stream)); });
}
rio_status rio_cuda_event_elapsed_ms(rio_placement *h, uint32_t a, uint32_t b, float *out_ms) {
    if (!h || !out_ms) { g_last_error = "null argument"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(a < RIO_MAX_EVENTS && b < RIO_MAX_EVENTS, "event slot out of range");
        CUDA_TRY(cudaEventSynchronize(h->events[b]));
        CUDA_TRY(cudaEventElapsedTime(out_ms, h->events[a], h->events[b]));
    });
}
rio_status rio_cuda_launch_count(rio_placement *h, uint64_t *out) {
    if (!h || !out) { g_last_error = "null argument"; return RIO_ERR_UNKNOWN; }
    std::lock_guard<std::mutex> g(h->mu);
    *out = h->launches;
    return RIO_OK;
}

// ---- string-level provider calls (what impl ObjectPlacement for GpuObjectPlacement forwards) ---------------------------------
rio_status rio_cuda_update_str(rio_placement *h, const char *type, size_t type_len, const char *id, size_t id_len, const char *address, size_t address_len) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(type && id, "null id");
        const uint64_t key = rio_cuda_object_key(type, type_len, id, id_len);
        uint32_t idx = kNone;
        if (address) idx = intern_node(h, std::string(address, address_len));     // any address may be recorded, live or not (local.rs:34-36)
        dir_reserve(h, 1);
        h->s_keys.ensure(8, h->stream);
        CUDA_TRY(cudaMemcpyAsync(h->s_keys.p, &key, 8, cudaMemcpyHostToDevice, h->stream));
        dir_upsert_dev(h, h->s_keys.as<uint64_t>(), nullptr, idx, 1);
        reconcile_dir_keys(h);
        check_device_error(h);
    });
}

rio_status rio_cuda_lookup_str(rio_placement *h, const char *type, size_t type_len, const char *id, size_t id_len, char *buf, size_t cap, size_t *out_len) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(type && id && out_len, "null argument");
        const uint64_t key = rio_cuda_object_key(type, type_len, id, id_len);
        h->s_keys.ensure(8, h->stream);
        h->s_idx.ensure(4, h->stream);
        CUDA_TRY(cudaMemcpyAsync(h->s_keys.p, &key, 8, cudaMemcpyHostToDevice, h->stream));
        launch_dir_lookup(h->L(), h->dir, h->s_keys.as<uint64_t>(), 1, h->s_idx.as<uint32_t>());
        uint32_t idx = kNone;
        CUDA_TRY(cudaMemcpyAsync(&idx, h->s_idx.p, 4, cudaMemcpyDeviceToHost, h->stream));
        CUDA_TRY(cudaStreamSynchronize(h->stream));
        if (idx == kNone || idx >= h->nodes.size()) { *out_len = (size_t)-1; return; }
        const std::string &a = h->nodes[idx].addr;
        *out_len = a.size();
        if (buf && cap) memcpy(buf, a.data(), std::min(cap, a.size()));
    });
}

rio_status rio_cuda_clean_server_str(rio_placement *h, const char *address, size_t address_len) {
    if (!h) { g_last_error = "null handle"; return RIO_ERR_UNKNOWN; }
    return guarded(h, [&] {
        REQUIRE(address, "null address");
        auto it = h->node_index.find(std::string(address, address_len));
        if (it == h->node_index.end()) return;   // never recorded: retain() would remove nothing (local.rs:56)
        zero_scalar(h, S_MOVED);
        launch_dir_clean_node(h->L(), h->dir, it->second, h->d_scalars + S_MOVED);
        CUDA_TRY(cudaStreamSynchronize(h->stream));
    });
}

rio_status rio_cuda_remove_str(rio_placement *h, const char *type, size_t type_len, const char *id, size_t id_len) {
    return rio_cuda_update_str(h, type, type_len, id, id_len, nullptr, 0);
}

}  // extern "C"

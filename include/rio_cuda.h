/*
 * rio_cuda.h -- C ABI of librio_cuda.so: the GPU-native (H100) object-placement engine that sits behind
 * rio-rs's `ObjectPlacement` trait.  This header is what a `rio-cuda-sys` FFI crate binds
 * (INTEGRATION.md shows the Rust declarations); there are no C++ or torch types in any signature.
 *
 * Reference interface replaced (all paths relative to /root/reference):
 *   trait ObjectPlacement { prepare, update, lookup, clean_server, remove }
 *                                              rio-rs/src/object_placement/mod.rs:38-56
 *   ObjectPlacementItem { object_id, server_address: Option<String> }
 *                                              rio-rs/src/object_placement/mod.rs:20-34
 *   ObjectId(String, String)                   rio-rs/src/service_object.rs:19-26
 *   ObjectPlacementError::{Upstream, Unknown}  rio-rs/src/errors.rs:136-142
 *   the per-request policy around it           rio-rs/src/service.rs:193-254 (get_or_create_placement)
 *   node identity "ip:port"                    rio-rs/src/cluster/storage/mod.rs:56-58 (Member::address)
 *
 * Conventions
 *   - Every function returns rio_status (0 = OK).  RIO_ERR_UPSTREAM maps to
 *     ObjectPlacementError::Upstream (CUDA / NCCL failure), RIO_ERR_UNKNOWN to
 *     ObjectPlacementError::Unknown (bad argument, internal error) -- errors.rs:136-142.
 *     rio_cuda_last_error() returns the message (thread-local, valid until the next call on the thread).
 *   - "lookup of a missing id is Ok(None), not an error" (tests/object_placement_backend.rs:14-15):
 *     a missing key yields status OK and the sentinel RIO_NONE.
 *   - An object is identified by a 64-bit key = rio_cuda_object_key(type, id), the hash of the exact
 *     byte string LocalObjectPlacement uses as its map key, format!("{}.{}", type, id) (local.rs:26-29).
 *     Two distinct ids collide with probability ~n^2/2^65 (2.7e-6 at 10 M objects); see DESIGN.md 4.2.
 *   - A node is identified by its address string; the engine interns it to a dense, stable u32 index
 *     (never reused for another address while the handle lives).  All batched calls speak indices.
 *   - All buffers are caller-owned; the library never keeps a caller pointer past the call.
 *     Functions with the `_dev` suffix take DEVICE pointers (allocated with rio_cuda_dev_alloc or by
 *     any CUDA allocator in the same process/device) and are asynchronous on the handle's stream:
 *     call rio_cuda_sync() before reading results on the host.  Everything else takes HOST pointers
 *     and returns with results in place.
 *   - Every function is thread-safe per handle (internal mutex; the work is serialised on one stream,
 *     which is what the outer `tokio::RwLock<P>.write()` does to `update` today, service.rs:246-248).
 *   - No C++ exception crosses this boundary.
 */
#ifndef RIO_CUDA_H
#define RIO_CUDA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RIO_ABI_VERSION 2

typedef int32_t rio_status;
#define RIO_OK            0
#define RIO_ERR_UPSTREAM (-1) /* -> ObjectPlacementError::Upstream(String), errors.rs:138 */
#define RIO_ERR_UNKNOWN  (-2) /* -> ObjectPlacementError::Unknown(String),  errors.rs:141 */

#define RIO_NONE 0xFFFFFFFFu  /* "no placement" / Option::None for a node index */

typedef struct rio_placement rio_placement; /* opaque engine handle == one provider instance (and its clones) */
typedef struct rio_objset rio_objset;       /* opaque resident object set (dense keys + assignment in HBM) */

typedef struct rio_config {
    uint32_t struct_size;        /* = sizeof(rio_config) */
    int32_t  device;             /* CUDA device ordinal; -1 = current device */
    uint64_t directory_capacity; /* initial directory slots (rounded up to a power of two); 0 = 1<<16 */
    uint32_t flags;              /* reserved, 0 */
    uint32_t reserved;
} rio_config;

/* ---- lifecycle: P::prepare() at server.rs:120-125 is rio_cuda_create + rio_cuda_set_nodes ------------- */
uint32_t    rio_cuda_abi_version(void);
rio_status  rio_cuda_create(const rio_config *cfg, rio_placement **out);
void        rio_cuda_destroy(rio_placement *h);                 /* when the last provider clone drops */
const char *rio_cuda_last_error(rio_placement *h);              /* h may be NULL (create failures) */
rio_status  rio_cuda_sync(rio_placement *h);                    /* wait for the handle's stream */
rio_status  rio_cuda_device_info(rio_placement *h, int32_t *device, int32_t *sm_count, uint64_t *hbm_bytes,
                                 char *name_buf, size_t name_cap);

/* ---- keys: ObjectId -> u64 (local.rs:26-29 key bytes) --------------------------------------------------- */
uint64_t    rio_cuda_object_key(const char *type, size_t type_len, const char *id, size_t id_len);
uint64_t    rio_cuda_node_seed(const char *address, size_t len);
/* Batched: ids packed back to back as the joined "{type}.{id}" byte strings; offsets has n+1 entries. */
rio_status  rio_cuda_hash_ids(rio_placement *h, const char *packed, const uint64_t *offsets, size_t n,
                              uint64_t *out_keys);

/* ---- node table: the live node set (MembershipStorage::active_members, storage/mod.rs:95-99) ----------- */
/* Replace the whole live set.  weights[j]==0 or weights==NULL(all 1).  feats: M x K row-major fp32 or NULL.
 * Nodes known to the engine but absent from addrs become inactive.  out_idx (may be NULL) receives the
 * interned index of each address. */
rio_status  rio_cuda_set_nodes(rio_placement *h, const char *const *addrs, const uint32_t *weights,
                               const float *feats, uint32_t M, uint32_t K, uint32_t *out_idx);
/* Add or re-weight one node (a join).  Returns its index. */
rio_status  rio_cuda_node_upsert(rio_placement *h, const char *address, uint32_t weight, const float *feat,
                                 uint32_t K, uint32_t *out_idx);
/* set_active / set_inactive (peer_to_peer.rs:170-191, storage/mod.rs:112-120) */
rio_status  rio_cuda_node_set_active(rio_placement *h, uint32_t idx, int32_t active);
rio_status  rio_cuda_node_index(rio_placement *h, const char *address, uint32_t *out_idx); /* RIO_NONE if unknown */
/* Intern an address without changing liveness (any address may be recorded by update, live or not: local.rs:34-36) */
rio_status  rio_cuda_node_intern(rio_placement *h, const char *address, uint32_t *out_idx);
rio_status  rio_cuda_node_address(rio_placement *h, uint32_t idx, char *buf, size_t cap, size_t *out_len);
rio_status  rio_cuda_node_count(rio_placement *h, uint32_t *out_total, uint32_t *out_live);
/* membership flag, weight and "address has no ip:port shape" (service.rs:213-222) of an interned node; any out may be NULL */
rio_status  rio_cuda_node_state(rio_placement *h, uint32_t idx, int32_t *active, uint32_t *weight, int32_t *malformed);
/* Failure-domain labels (DESIGN.md 3.12): node idx[i] gets label domain[i] (a rack or zone id from the deployment).  RIO_NONE, the
 * default of every interned node, means "a domain of its own".  Labels stay with the interned index across set_nodes, node_upsert and
 * node_set_active, count only while the node is live, and change no call other than rio_cuda_assign_ranked_spread_batch.
 * RIO_ERR_UNKNOWN for an index out of range, a duplicate index, or NULL arrays with k > 0; k == 0 does nothing. */
rio_status  rio_cuda_node_set_domains(rio_placement *h, const uint32_t *idx, const uint32_t *domain, size_t k);
rio_status  rio_cuda_node_domain(rio_placement *h, uint32_t idx, uint32_t *out_domain);

/* ---- solver policy of the handle (new; no reference counterpart) ----------------------------------------------------
 * RIO_SOLVER_HRW  = flat weighted rendezvous over all live nodes (DESIGN.md 3.4): M pair hashes per object, minimal movement
 *                   on a membership change.  The default.
 * RIO_SOLVER_HRW2 = hierarchical weighted rendezvous with fan-out 2 (DESIGN.md 3.8): the live nodes sit in a binary trie
 *                   over a hash of their address, every trie node is a 2-way weighted rendezvous between its subtrees decided
 *                   in closed form (one 31-bit hash of (object, level) against floor(2^31 W_left / (W_left + W_right))), so an
 *                   object costs trie_bits + O(1) contests instead of M pair hashes; P(node) = w/W as before, movement on a
 *                   membership change is about (1 + log2(M)/2) x minimal.  trie_bits in [1, 14]; 0 keeps the current depth
 *                   (default 12).
 * The policy applies to assign_batch(_dev), the resident-set calls and rebalance; place_batch carries its own policy. */
#define RIO_SOLVER_HRW  1u
#define RIO_SOLVER_HRW2 2u
rio_status  rio_cuda_set_solver(rio_placement *h, uint32_t solver, uint32_t trie_bits);
rio_status  rio_cuda_get_solver(rio_placement *h, uint32_t *solver, uint32_t *trie_bits);

/* ---- directory: batched LocalObjectPlacement (local.rs:22-68) ------------------------------------------- */
/* lookup (local.rs:42-49): out_idx[i] = node index or RIO_NONE */
rio_status  rio_cuda_lookup_batch(rio_placement *h, const uint64_t *keys, size_t n, uint32_t *out_idx);
/* update (local.rs:22-40): idx[i]==RIO_NONE is update(None) => the key is removed.  Duplicate keys in one
 * batch resolve as if applied in array order (the last one wins). */
rio_status  rio_cuda_upsert_batch(rio_placement *h, const uint64_t *keys, const uint32_t *idx, size_t n);
/* remove (local.rs:60-68) */
rio_status  rio_cuda_remove_batch(rio_placement *h, const uint64_t *keys, size_t n);
/* clean_server (local.rs:51-58): unassign every object recorded on node idx; out_removed may be NULL */
rio_status  rio_cuda_clean_node(rio_placement *h, uint32_t idx, uint64_t *out_removed);
rio_status  rio_cuda_directory_len(rio_placement *h, uint64_t *out_placed, uint64_t *out_slots);

/* ---- solver: the N_obj x M_node score grid + per-row argmin (new; no reference counterpart) ------------ */
/* Weighted rendezvous hash over the live nodes (DESIGN.md 3.4).  Pure function of (keys, live set):
 * does not touch the directory.  obj_feats != NULL (n x K fp32) selects the affinity cost instead
 * (cost = -dot, argmin; DESIGN.md 3.6) and requires node features of the same K. */
rio_status  rio_cuda_assign_batch(rio_placement *h, const uint64_t *keys, const float *obj_feats, size_t n,
                                  uint32_t *out_idx);
/* assign_batch followed by the bounded-load rounds of rio_cuda_set_assign_bounded (DESIGN.md 3.5) for host buffers: the
 * per-node histogram is fused into the score kernels of the chunk pipeline, the counter exchange + capacity check runs on
 * the device behind the last chunk.  n_total = global object count (0 = n * world).  Hash path; the affinity cost:
 * rio_cuda_assign_bounded_affinity_batch. */
rio_status  rio_cuda_assign_bounded_batch(rio_placement *h, const uint64_t *keys, size_t n, uint64_t n_total, uint32_t cap_num,
                                          uint32_t cap_den, uint32_t max_rounds, uint32_t *out_idx, uint32_t *out_passes);
/* rio_cuda_set_assign_bounded_affinity for host buffers: keys (n) feed the spill hash, obj_feats (n x K, K of set_nodes) the cost.
 * Returns exactly what the set call returns for the same keys and features.  Argument rules as for rio_cuda_assign_bounded_batch;
 * also RIO_ERR_UNKNOWN for NULL buffers or a handle without node features, RIO_ERR_UPSTREAM when the library was built without the
 * bounded affinity kernels. */
rio_status  rio_cuda_assign_bounded_affinity_batch(rio_placement *h, const uint64_t *keys, const float *obj_feats, size_t n,
                                                   uint64_t n_total, uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds,
                                                   uint32_t *out_idx, uint32_t *out_passes);
/* rio_cuda_set_assign_bounded_weighted for host buffers (DESIGN.md 3.19): keys (n) feed the hash policy and the spill hash;
 * obj_feats (n x K, K of set_nodes) selects the affinity cost, NULL the hash policy; weights (n) are the objects' loads, NULL = all 1.
 * Returns exactly what the set call returns for the same rows, with the same refusals (this rank's weight sum is that of `weights`);
 * also RIO_ERR_UNKNOWN for NULL keys or out_idx.  n == 0 returns at once and takes part in no exchange. */
rio_status  rio_cuda_assign_bounded_weighted_batch(rio_placement *h, const uint64_t *keys, const float *obj_feats, const uint32_t *weights,
                                                   size_t n, uint64_t load_total, uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds,
                                                   uint32_t *out_idx, uint32_t *out_passes);
/* Ranked placement (DESIGN.md 3.9): each object's first `ranks` distinct nodes under the handle's solver policy.  rank 1 is
 * exactly what assign_batch returns; rank r is the same policy's placement over the live set minus ranks 1..r-1 -- so rank 2 is
 * where a LEAVE of rank 1 sends the object (its failover target).  Pure function of (keys, live set); hash path only (the affinity cost: rio_cuda_assign_ranked_affinity_batch).
 * out_idx is n x ranks, row-major (object i's list at out_idx[i*ranks ..]); ranks beyond the live node count are RIO_NONE.
 * RIO_ERR_UNKNOWN for ranks outside [1, RIO_MAX_RANKS], NULL buffers, or n x ranks overflowing. */
#define RIO_MAX_RANKS 8u
rio_status  rio_cuda_assign_ranked_batch(rio_placement *h, const uint64_t *keys, size_t n, uint32_t ranks, uint32_t *out_idx);
/* Ranked placement across failure domains (DESIGN.md 3.12): rank 1 is exactly what assign_batch returns; rank r is the same policy's
 * placement over the live set minus every node whose domain is the domain of one of ranks 1..r-1.  The ranks lie in distinct
 * domains, rank 2 is where the object goes when rank 1's whole domain leaves, and the entries past the number of distinct live
 * domains are RIO_NONE.  With no labels set the result equals rio_cuda_assign_ranked_batch.  Output and argument errors as for
 * rio_cuda_assign_ranked_batch; RIO_ERR_UPSTREAM when the library was built without the spread kernels. */
rio_status  rio_cuda_assign_ranked_spread_batch(rio_placement *h, const uint64_t *keys, size_t n, uint32_t ranks, uint32_t *out_idx);
/* Ranked placement under the affinity cost (DESIGN.md 3.9): each object's `ranks` lowest-cost live nodes, cost = -dot(F_obj, F_node),
 * in increasing (cost, node index) order.  rank 1 is exactly what assign_batch with the same obj_feats returns; rank r is the
 * affinity placement over the live set minus ranks 1..r-1, so rank 2 is where a LEAVE of rank 1 sends the object.  obj_feats is
 * n x K (K of set_nodes), out_idx n x ranks row-major, RIO_NONE past the live node count.  RIO_ERR_UNKNOWN as for
 * rio_cuda_assign_ranked_batch, and when the handle has no node features. */
rio_status  rio_cuda_assign_ranked_affinity_batch(rio_placement *h, const float *obj_feats, size_t n, uint32_t ranks, uint32_t *out_idx);
/* Ranked placement under the affinity cost across failure domains (DESIGN.md 3.14): rank 1 is exactly what assign_batch with the
 * same obj_feats returns; rank r is the lowest (cost, node index) over the live set minus every node whose domain is the domain of
 * one of ranks 1..r-1.  The ranks lie in distinct domains, rank 2 is where the object goes when rank 1's whole domain leaves, and the
 * entries past the number of distinct live domains are RIO_NONE.  With no labels set the result is rio_cuda_assign_ranked_affinity_batch's.
 * Output and argument errors as for rio_cuda_assign_ranked_affinity_batch; RIO_ERR_UPSTREAM when the library was built without the
 * failure-domain affinity kernels. */
rio_status  rio_cuda_assign_ranked_affinity_spread_batch(rio_placement *h, const float *obj_feats, size_t n, uint32_t ranks, uint32_t *out_idx);
/* Service::get_or_create_placement for a batch (service.rs:193-254): existing & live => keep; recorded on an
 * inactive node => clean_server(that node) then re-place; none => place.  policy RIO_PLACE_SELF re-places on
 * self_idx (the reference's rule, service.rs:244-252); RIO_PLACE_HRW / RIO_PLACE_HRW2 re-place by the solver. */
#define RIO_PLACE_SELF 0u
#define RIO_PLACE_HRW  1u
#define RIO_PLACE_HRW2 2u   /* re-place by the hierarchical solver (RIO_SOLVER_HRW2 semantics, the handle's trie_bits) */
rio_status  rio_cuda_place_batch(rio_placement *h, const uint64_t *keys, size_t n, uint32_t policy,
                                 uint32_t self_idx, uint32_t *out_idx);
/* Service::check_address_mismatch for a batch (service.rs:261-298), the second half of the per-request policy: for the
 * address index the first half returned, RIO_ADDR_LOCAL = it is this server (Ok(())); RIO_ADDR_REDIRECT = the node is active
 * elsewhere (Err(Redirect(address))); RIO_ADDR_DEALLOCATE = the node is not active: clean_server(address) HAS BEEN APPLIED
 * to the directory (one table scan for all such nodes of the batch) and the caller answers DeallocateServiceObject;
 * RIO_ADDR_MALFORMED = the recorded address has no ':' (Err(Unknown("Malformed address: Missing PORT ..."))).  Like the
 * reference, only the first two ':'-separated pieces of the address are the (ip, port) asked of is_active.
 * out_cleaned (may be NULL) receives the number of directory entries the clean_server calls removed. */
#define RIO_ADDR_LOCAL      0u
#define RIO_ADDR_REDIRECT   1u
#define RIO_ADDR_DEALLOCATE 2u
#define RIO_ADDR_MALFORMED  3u
rio_status  rio_cuda_check_address_batch(rio_placement *h, const uint32_t *addr_idx, size_t n, uint32_t self_idx,
                                         uint8_t *out_verdict, uint64_t *out_cleaned);
/* Eager re-placement of the whole directory after a membership change (replaces the lazy per-object path
 * service.rs:224-238 / 286-297): RIO_EV_JOIN(idx) moves onto idx exactly the objects that now prefer it;
 * RIO_EV_LEAVE(idx) re-places exactly the objects recorded on idx.  Under RIO_SOLVER_HRW2 every placed key is walked
 * again and the ones whose node changed are rewritten (the state after the call is the fresh assignment over the
 * live set).  out_moved may be NULL.  A weight decrease under RIO_SOLVER_HRW is applied exactly only by
 * rio_cuda_rebalance_changes. */
#define RIO_EV_JOIN  1u
#define RIO_EV_LEAVE 2u
rio_status  rio_cuda_rebalance(rio_placement *h, uint32_t event, uint32_t idx, uint64_t *out_moved);
/* Eager re-placement of the whole directory after a SET of node changes (DESIGN.md 3.10), in one pass.  idx[0..k) are distinct
 * interned node indices; prev_weight[i] is node idx[i]'s weight before the change if it was live then (active, weight > 0),
 * else 0.  Apply the changes first (set_nodes / node_upsert / node_set_active); read the prior weights with
 * rio_cuda_node_state before.  With r = floor((2^32-1)/w) for a live node and 0 otherwise:
 *   REPLACE    = every interned node not live now, and every changed node live now whose r grew (it lost weight);
 *   CANDIDATES = every changed node live now that was not live before or whose r shrank (it joined or gained weight);
 *   a changed node whose r did not change is a no-op.
 * RIO_SOLVER_HRW: an entry (key, y) with y in REPLACE is re-placed over the current live set (it may stay on y); any other
 * placed entry goes to the best node of {y} u CANDIDATES under the order of 3.4.  If the directory was the flat assignment
 * over the previous live set, it is the fresh one over the current live set afterwards.  RIO_SOLVER_HRW2: any k > 0 walks
 * every placed key again once.  Entries become RIO_NONE when no node is live; k == 0 does nothing.  out_moved (may be NULL)
 * receives the number of entries whose node changed.  RIO_ERR_UNKNOWN: an index out of range, a duplicate index, NULL arrays
 * with k > 0; RIO_ERR_UPSTREAM under RIO_SOLVER_HRW when the library was built without the change-set kernels. */
rio_status  rio_cuda_rebalance_changes(rio_placement *h, const uint32_t *idx, const uint32_t *prev_weight, size_t k, uint64_t *out_moved);
/* Per-node object counts of the directory (out has node_count entries). */
rio_status  rio_cuda_load_counters(rio_placement *h, uint32_t *out, uint32_t cap);

/* ---- resident object sets: id-range shards kept in HBM (configs C4/C5) --------------------------------- */
rio_status  rio_cuda_set_create(rio_placement *h, uint64_t capacity, rio_objset **out);
void        rio_cuda_set_destroy(rio_objset *s);
rio_status  rio_cuda_set_load_keys(rio_objset *s, const uint64_t *keys, uint64_t n);      /* host -> HBM */
rio_status  rio_cuda_set_load_feats(rio_objset *s, const float *feats, uint32_t K);       /* n x K fp32 */
/* (Re)assign every object of the set over the live nodes; counters of the result are kept on device. */
rio_status  rio_cuda_set_assign(rio_objset *s, uint32_t use_affinity);
/* Bounded-load rounds (DESIGN.md 3.5): capacity = ceil(cap_num*N_total*w/(cap_den*W)), at most max_rounds
 * assignment passes, ONE counter exchange per pass (across ranks when a communicator is attached).
 * n_total = global object count (0 = this set's n * world).  out_passes may be NULL. */
rio_status  rio_cuda_set_assign_bounded(rio_objset *s, uint64_t n_total, uint32_t cap_num, uint32_t cap_den,
                                        uint32_t max_rounds, uint32_t *out_passes);
/* The same call in two halves.  _begin enqueues pass 0 -- under RIO_SOLVER_HRW2 ONE kernel: walk, histogram, counter exchange over
 * peer memory, capacity check -- and returns without waiting; _end waits for that check (two words in mapped pinned memory) and
 * runs the spill rounds it asks for.  Several sets of one handle may be between _begin and _end at the same time (a set takes
 * part in one bounded call at a time), which keeps the GPU's queue full across calls; with ranks > 1 every rank must issue its
 * _begin / _end calls in the same order.  rio_cuda_set_assign_bounded == _begin followed by _end. */
rio_status  rio_cuda_set_assign_bounded_begin(rio_objset *s, uint64_t n_total, uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds);
rio_status  rio_cuda_set_assign_bounded_end(rio_objset *s, uint32_t *out_passes);
/* Bounded-load rounds under the affinity cost (DESIGN.md 3.16): the capacities, counters, spill selection and closed set of
 * rio_cuda_set_assign_bounded, with pass 0 = rio_cuda_set_assign(s, 1) bit for bit, and a spilled object re-placed at its lowest
 * cost over the live nodes not closed, on the kernel path pass 0 took.  Node weights set the capacities; the costs ignore them.
 * Needs the set's keys (spill hash) and features (set_load_feats, K of the handle).  Drops ranked lists.  RIO_ERR_UNKNOWN for a
 * handle without node features, set features missing or of another K, or a bounded call in flight on the set (between _begin and
 * _end); RIO_ERR_UPSTREAM when the library was built without the bounded affinity kernels. */
rio_status  rio_cuda_set_assign_bounded_affinity(rio_objset *s, uint64_t n_total, uint32_t cap_num, uint32_t cap_den,
                                                 uint32_t max_rounds, uint32_t *out_passes);
/* Keeps a bounded-load affinity assignment within capacity through a change set (DESIGN.md 3.17), a change set as
 * rio_cuda_set_rebalance_changes takes (call AFTER the node table changed).  Pass 0: an object on a node that is not live, was
 * refeatured since the last call, or is past the table (or on none) is re-placed at its lowest cost over the live set on the path
 * the set recorded; any other object goes to the lowest-cost node of {its node} u {joined and refeatured live nodes}.  Then the
 * capacity rounds of rio_cuda_set_assign_bounded_affinity run from those counters, with capacities from n_total (0 = n * world),
 * cap_num / cap_den and the current live weights.  An object changes node only if pass 0 re-placed it, a candidate beat its node, or
 * it spilled from a node over capacity; the result is not a fresh bounded call.  out_moved (may be NULL) receives the objects whose
 * node differs from the one before the call, out_passes (may be NULL) 1 + the rounds run.  Needs the record a successful
 * rio_cuda_set_assign_bounded_affinity (or this call) leaves; every call that drops ranked lists, and set_load_feats, removes it.
 * RIO_ERR_UNKNOWN (nothing changed): no record, a handle K other than the recorded one, set features missing or of another K, the
 * argument errors of rio_cuda_set_rebalance_changes, cap_den == 0, max_rounds == 0, or a bounded call in flight on the set;
 * RIO_ERR_UPSTREAM when the library was built without the kernels of this call. */
rio_status  rio_cuda_set_rebalance_changes_bounded_affinity(rio_objset *s, const uint32_t *idx, const uint32_t *prev_weight, size_t k,
                                                            uint64_t n_total, uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds,
                                                            uint64_t *out_moved, uint32_t *out_passes);
/* Object churn in a resident set (DESIGN.md 3.18).  rio_cuda_set_insert appends m objects as rows [n, n+m) (*out_first = n, may
 * be NULL) and places them as the set's current kind places a fresh object: no node while the set is unassigned; the list the
 * batch call of the set's list kind returns, column 0 as idx, for a set holding ranked lists; the plain affinity argmin on the
 * recorded path for a bounded affinity record (a later rio_cuda_set_rebalance_changes_bounded_affinity with k = 0 brings the set
 * back within capacity); otherwise what rio_cuda_assign_batch returns for it (hash: the handle's current policy; affinity: the
 * recorded path).  feats (m x the set's K) is required exactly when the set has features.  The counters gain the new rows; no
 * existing row changes.  rio_cuda_set_erase removes every row whose key is one of keys[0..m) (duplicates allowed, absent keys
 * ignored; *out_erased, may be NULL, = rows removed): with n' the new size, the surviving rows at or above n' fill the removed rows
 * below n', both in increasing order, carrying key, idx, feature row and list row; nothing else moves.  The counters lose the
 * removed rows of an assigned set.  Lists, snapshots and records stay; the directory is not touched.  m == 0 does nothing.
 * RIO_ERR_UNKNOWN (nothing changed): keys NULL with m > 0, features missing or given to a set without them, n + m > capacity, a
 * bounded call in flight on the set, hash lists computed under another solver or trie_bits, or an affinity kind or record under
 * another K; RIO_ERR_UPSTREAM when the library was built without the churn kernels. */
rio_status  rio_cuda_set_insert(rio_objset *s, const uint64_t *keys, const float *feats, uint64_t m, uint64_t *out_first);
rio_status  rio_cuda_set_erase(rio_objset *s, const uint64_t *keys, uint64_t m, uint64_t *out_erased);
/* Weighted objects (DESIGN.md 3.19).  Every set has one uint32 weight per row, 1 unless written: rio_cuda_set_write_weights writes
 * rows [first, first+n) from w, rio_cuda_set_read_weights reads them into out (the range must lie inside [0, size)).  The column
 * (capacity x 4 bytes) is allocated by the first write; a set never written allocates nothing.  set_load_keys and set_synth_keys
 * reset every weight to 1, set_insert gives each new row weight 1 (write the real weights at *out_first), and set_erase moves each
 * row's weight with its key; no other call reads or changes them.
 * rio_cuda_set_assign_bounded_weighted is rio_cuda_set_assign_bounded (use_affinity = 0) or rio_cuda_set_assign_bounded_affinity
 * (use_affinity = 1) with node LOADS in place of object counts: a node's load is the global sum of the weights of its objects, its
 * capacity ceil(cap_num * L * w / (cap_den * W)) with L = load_total (0 = G, the weight sum of every rank's shard, reduced across ranks
 * by one exchange; an explicit load_total must be the same on every rank), and a round spills an object
 * of weight > 0 from a node over capacity iff its spill hash is below floor(2^32 (load - cap) / load).  Objects of weight 0 never
 * spill.  Pass 0 is rio_cuda_set_assign(s, use_affinity) bit for bit; a spilled object goes where pass 0's method places it over the
 * live nodes not closed.  With every weight 1 and load_total = n_total the result (idx, counters, passes) equals the count-based call
 * bit for bit.  Afterwards the counters are the object counts of the result (not loads), the set records a plain assignment (hash,
 * or affinity on the path taken) and holds no ranked lists or bounded affinity record.  Loads are u32: the global weight total
 * must stay below 2^32.  RIO_ERR_UNKNOWN (nothing changed): on each rank before any exchange (pass the same arguments on every rank),
 * cap_den == 0, max_rounds == 0, use_affinity > 1, a bounded call in flight on the set, the feature errors of
 * rio_cuda_set_assign_bounded_affinity (use_affinity = 1); on every rank together, after the reduction of G, G or load_total above
 * 2^32-1, or load_total != 0 below G.
 * rio_cuda_set_loads copies the global (all ranks, collective as rio_cuda_set_counters is) per-node weight sums of the current
 * assignment into out (cap >= node count), computed on demand; an unassigned set reports zeros; RIO_ERR_UNKNOWN, on every rank
 * together, for G above 2^32-1.  RIO_ERR_UPSTREAM for the weighted assign, rio_cuda_set_loads, and set_erase on a set with a weight
 * column, when the library was built without the weighted kernels. */
rio_status  rio_cuda_set_write_weights(rio_objset *s, uint64_t first, uint64_t n, const uint32_t *w);
rio_status  rio_cuda_set_read_weights(rio_objset *s, uint64_t first, uint64_t n, uint32_t *out);
rio_status  rio_cuda_set_assign_bounded_weighted(rio_objset *s, uint32_t use_affinity, uint64_t load_total, uint32_t cap_num,
                                                 uint32_t cap_den, uint32_t max_rounds, uint32_t *out_passes);
rio_status  rio_cuda_set_loads(rio_objset *s, uint32_t *out, uint32_t cap);
/* Weighted bounded sets kept within load capacity (DESIGN.md 3.21).
 * rio_cuda_set_write_weights_by_key gives every row whose key equals keys[j] the weight w[j] (a key listed several times: its last
 * occurrence; a key in several rows: every one of them; absent keys are ignored) and reports the rows written in *out_written
 * (nullable).  The first write allocates the column as rio_cuda_set_write_weights does, every other row 1.  m == 0 does nothing.
 * RIO_ERR_UNKNOWN (nothing changed): keys or w NULL with m > 0, a bounded call in flight on the set.
 * rio_cuda_set_rebalance_changes_bounded_weighted keeps a set that rio_cuda_set_assign_bounded_weighted (or this call) placed within
 * its load capacities after a change set (idx, prev_weight, k as in rio_cuda_rebalance_changes) and after weight or churn changes:
 * pass 0 is the change-set pass of the recorded kind (flat HRW: 3.10; HRW2: an object on a node that left or lost weight takes its
 * walk over the live set, any other object moves only to a node that joined or gained weight when its walk lands there; affinity:
 * the pass 0 of rio_cuda_set_rebalance_changes_bounded_affinity), then the weighted rounds of 3.19 from the loads it leaves, with
 * capacities from load_total as in rio_cuda_set_assign_bounded_weighted.  An object changes node only if pass 0 re-placed it or a
 * candidate took it, or it spilled from a node over its load capacity.  *out_moved = objects whose node changed, *out_passes = 1 +
 * the rounds run; the counters are object counts.  The record is kept by set_insert, set_erase, both weight writes and the commits,
 * and removed by every call that rewrites idx another way, by set_load_keys / set_synth_keys and, for affinity, set_load_feats.
 * RIO_ERR_UNKNOWN (nothing changed): on each rank before any exchange, no record, a solver or trie_bits (hash) or node feature K
 * (affinity) other than the recorded one, missing features, the change-set errors of rio_cuda_rebalance_changes, cap_den == 0,
 * max_rounds == 0, a bounded call in flight; on every rank together, G or load_total above 2^32-1, or load_total != 0 below G.
 * RIO_ERR_UPSTREAM for both calls when the library was built without their kernels. */
rio_status  rio_cuda_set_write_weights_by_key(rio_objset *s, const uint64_t *keys, const uint32_t *w, size_t m, uint64_t *out_written);
rio_status  rio_cuda_set_rebalance_changes_bounded_weighted(rio_objset *s, const uint32_t *idx, const uint32_t *prev_weight, size_t k,
                                                            uint64_t load_total, uint32_t cap_num, uint32_t cap_den, uint32_t max_rounds,
                                                            uint64_t *out_moved, uint32_t *out_passes);
/* Incremental rebalance of the set after the node table changed (call AFTER node_upsert / node_set_active). */
rio_status  rio_cuda_set_rebalance(rio_objset *s, uint32_t event, uint32_t idx, uint64_t *out_moved);
/* rio_cuda_rebalance_changes for the set, under the plain policy (capacity bounds of an earlier bounded call are not applied
 * again; sets assigned with affinity are not supported).  Objects with no node (RIO_NONE) are re-placed like REPLACE entries.
 * The counters stay exact.  Also RIO_ERR_UNKNOWN for a set with no assignment yet. */
rio_status  rio_cuda_set_rebalance_changes(rio_objset *s, const uint32_t *idx, const uint32_t *prev_weight, size_t k, uint64_t *out_moved);
/* Ranked resident sets (DESIGN.md 3.11).  rio_cuda_set_assign_ranked computes each key's first `ranks` nodes under the handle's
 * policy (as rio_cuda_assign_ranked_batch does), keeps them in the set (capacity x ranks x 4 bytes, grow-only, freed by
 * set_destroy), sets the set's assignment to column 0 and rebuilds the counters from it; the lists record the solver and trie_bits.
 * rio_cuda_set_read_ranked copies rows [first, first+n) row-major into out (n x ranks entries).
 * rio_cuda_set_rebalance_changes_ranked takes a change set as rio_cuda_set_rebalance_changes does and leaves every list equal to
 * the fresh ranked list over the current live set: under RIO_SOLVER_HRW a list with a member in REPLACE (or past the node table) is
 * recomputed, any other becomes the first `ranks` nodes of itself u CANDIDATES; under RIO_SOLVER_HRW2 any k > 0 walks every list
 * again.  Only changed rows are written; column 0 stays the set's assignment and the counters stay exact.  out_moved (may be NULL)
 * receives the number of objects whose rank 1 changed, out_changed (may be NULL) the number whose list changed at any rank.
 * RIO_ERR_UNKNOWN: ranks outside [1, RIO_MAX_RANKS], n x ranks overflowing, a read outside the set, NULL buffers, the argument
 * errors of rio_cuda_set_rebalance_changes, a set holding no lists, or a change set under another solver or trie_bits than the
 * lists were computed with (affinity lists ignore the solver: see rio_cuda_set_assign_ranked_affinity below).  RIO_ERR_UPSTREAM when the library was built without the ranked-set kernels.  Every call that rewrites
 * the set's assignment otherwise (set_load_keys, set_synth_keys, set_assign, set_assign_bounded(_begin), set_rebalance,
 * set_rebalance_changes) drops the lists. */
rio_status  rio_cuda_set_assign_ranked(rio_objset *s, uint32_t ranks);
rio_status  rio_cuda_set_read_ranked(rio_objset *s, uint64_t first, uint64_t n, uint32_t *out);
rio_status  rio_cuda_set_rebalance_changes_ranked(rio_objset *s, const uint32_t *idx, const uint32_t *prev_weight, size_t k, uint64_t *out_moved,
                                                  uint64_t *out_changed);
/* Failure-domain resident sets (DESIGN.md 3.13).  rio_cuda_set_assign_ranked_spread works as rio_cuda_set_assign_ranked, with each
 * key's failure-domain list (as rio_cuda_assign_ranked_spread_batch computes it) in place of its ranked list, and also records the
 * label of every interned node.  rio_cuda_set_read_ranked reads these lists unchanged.  On such a set
 * rio_cuda_set_rebalance_changes_ranked leaves every list equal to the fresh failure-domain list over the current live set and the
 * CURRENT labels: relabels made since the labels were recorded belong to the change set, so k = 0 with a relabel applies it, and
 * k = 0 without one does nothing.  A successful call records the labels again.  Errors as for the ranked sets; RIO_ERR_UPSTREAM
 * when the library was built without the spread-set kernels.  The calls that drop ranked lists drop these too, and
 * rio_cuda_set_assign_ranked makes the set a plain ranked set again (plain ranked sets ignore labels). */
rio_status  rio_cuda_set_assign_ranked_spread(rio_objset *s, uint32_t ranks);
/* Affinity resident sets (DESIGN.md 3.15).  rio_cuda_set_assign_ranked_affinity(_spread) works as rio_cuda_set_assign_ranked, with
 * each object's list from rio_cuda_assign_ranked_affinity_batch (or rio_cuda_assign_ranked_affinity_spread_batch) of the set's
 * features (rio_cuda_set_load_feats) in place of its ranked list, on the path that call takes now (column 0 is then bit for bit rio_cuda_set_assign(use_affinity = 1) on that path).  The
 * set records the kind of lists, the path (tensor cores or CUDA cores; RIO_AFFINITY_VARIANT is read here only), the handle's K, every
 * interned node's feature row and, for failure-domain lists, its label.  rio_cuda_set_read_ranked reads these lists unchanged.
 * On such a set rio_cuda_set_rebalance_changes_ranked ignores the solver and trie_bits and classifies by liveness (active, weight > 0):
 *   REPLACE    = every interned node not live now, every live node whose feature row differs from the recorded one (refeatured) and,
 *                for failure-domain lists, every relabelled live node;
 *   CANDIDATES = every changed node live now with prev_weight 0, and every refeatured or relabelled live node;
 *   a live -> live weight change is a no-op.
 * A list with a member in REPLACE, or with no member, is recomputed on the recorded path; any other becomes the first `ranks` of
 * itself u CANDIDATES in (fp32 cost, node index) order (for failure-domain lists the best `ranks` domain representatives).  k = 0
 * with a refeature or relabel applies it, k = 0 without one does nothing.  On the CUDA cores the lists then equal a fresh CUDA-core
 * call over the current live set, features and labels bit for bit.  On the tensor cores they agree with a fresh call but for near-ties
 * within the tolerance of 3.9, and column 0 of a row a candidate entered can differ from rio_cuda_set_assign(use_affinity = 1) at a
 * near-tie.  A tensor-core set recomputes on the CUDA cores while its padded live count exceeds the tensor path's limit.
 * RIO_ERR_UNKNOWN: ranks outside [1, RIO_MAX_RANKS], n x ranks overflowing, a handle without node features, set features missing or
 * of another K than the handle's, and on a change set the argument errors of rio_cuda_set_rebalance_changes or a handle K other than
 * the recorded one (a refused call leaves lists and records as they were).  RIO_ERR_UPSTREAM when the library was built without the
 * affinity-set kernels.  Every call that drops ranked lists drops these, and so does rio_cuda_set_load_feats;
 * rio_cuda_set_assign_ranked(_spread) makes the set a hash-policy set again. */
rio_status  rio_cuda_set_assign_ranked_affinity(rio_objset *s, uint32_t ranks);
rio_status  rio_cuda_set_assign_ranked_affinity_spread(rio_objset *s, uint32_t ranks);
/* Global (all ranks) per-node counters of the set's current assignment. */
rio_status  rio_cuda_set_counters(rio_objset *s, uint32_t *out, uint32_t cap);
rio_status  rio_cuda_set_read(rio_objset *s, uint64_t first, uint64_t n, uint64_t *out_keys, uint32_t *out_idx);
rio_status  rio_cuda_set_size(rio_objset *s, uint64_t *out_n);
/* Write the set's assignment through to the directory (update for every object). */
rio_status  rio_cuda_set_commit(rio_objset *s);
/* Delta commit (DESIGN.md 3.20): row i < n is selected iff idx[i] differs from what the directory answers for keys[i] at the start of
 * the call (RIO_NONE for an absent or removed key, the key normalised as the directory does).  The manifest is the selected rows in
 * increasing row order, entry j = {out_rows[j] = i, out_keys[j] = keys[i] as stored, out_from[j] = the directory's answer,
 * out_to[j] = idx[i]}; *out_n = its size.  Each out array may be NULL.  dry_run == 0 upserts the selected rows in row order
 * (to == RIO_NONE removes the key) and changes nothing else; dry_run == 1 leaves the directory as it was.  For distinct keys the
 * directory afterwards equals the one rio_cuda_set_commit leaves; with a key in several rows every row is compared with the directory
 * at the start and the last selected row wins.  Only idx is committed, and the set is not touched.  RIO_ERR_UNKNOWN (directory and
 * out arrays untouched): a null set, a set with no assignment, a bounded call in flight on the set, or *out_n > cap with any out
 * array non-NULL (*out_n is written then); RIO_ERR_UPSTREAM when the library was built without the set commit kernels. */
rio_status  rio_cuda_set_commit_changes(rio_objset *s, uint32_t dry_run, uint64_t cap, uint64_t *out_rows, uint64_t *out_keys, uint32_t *out_from,
                                        uint32_t *out_to, uint64_t *out_n);

/* ---- multi-GPU: one process per GPU; the only collective is the per-node load-counter all-gather -------- */
#define RIO_COMM_ID_BYTES 128
rio_status  rio_cuda_comm_unique_id(uint8_t out_id[RIO_COMM_ID_BYTES]);       /* rank 0; ship to the others */
rio_status  rio_cuda_comm_init(rio_placement *h, int32_t rank, int32_t world, const uint8_t id[RIO_COMM_ID_BYTES]);
/* Peer-memory variant of the exchange (preferred on one NVLink/NVSwitch box): every rank exports a small window, the host
 * gathers the world handles (any bootstrap) and attaches them; from then on the counter exchange is ONE kernel that stores
 * into the peers' windows over NVLink and spins on flags -- no NCCL launch on the critical path.  At most 16 ranks. */
#define RIO_IPC_HANDLE_BYTES 64
rio_status  rio_cuda_comm_ipc_export(rio_placement *h, int32_t world, uint32_t max_nodes, uint8_t out_handle[RIO_IPC_HANDLE_BYTES]);
rio_status  rio_cuda_comm_ipc_attach(rio_placement *h, int32_t rank, int32_t world, const uint8_t *handles /* world x RIO_IPC_HANDLE_BYTES */);
rio_status  rio_cuda_comm_info(rio_placement *h, int32_t *rank, int32_t *world);
/* all-gather + sum of an M-entry u32 counter vector (host in/out); exposed for tests and host-side logic */
rio_status  rio_cuda_comm_sum_counters(rio_placement *h, uint32_t *inout, uint32_t M);

/* ---- device-resident variants (inputs already in HBM; asynchronous on the handle's stream) -------------
 * Alignment: every d_ buffer must be naturally aligned for its element type -- 8 bytes for keys, 4 for node indices and
 * features.  Any other pointer is refused with RIO_ERR_UNKNOWN before anything is enqueued.  Any naturally aligned pointer is
 * accepted, such as a slice of a larger buffer.  Some kernels take wider loads: the HRW2 walk of assign_batch_dev reads keys 16
 * bytes and writes indices 8 bytes at a time, and every K == 16 affinity kernel reads feature rows 16 bytes at a time.  When such
 * a buffer does not start at that alignment, the call copies it on the stream into the handle's own buffer and runs from there;
 * the copy costs one extra pass over that buffer.  A buffer at 256 bytes, which is what rio_cuda_dev_alloc and cudaMalloc return,
 * is always used in place.  A call writes exactly n (or n x ranks) entries of d_out_idx and never writes its inputs. */
rio_status  rio_cuda_dev_alloc(rio_placement *h, size_t bytes, void **out_dev);
rio_status  rio_cuda_dev_free(rio_placement *h, void *dev);
rio_status  rio_cuda_host_alloc(rio_placement *h, size_t bytes, void **out_pinned);  /* pinned host memory */
rio_status  rio_cuda_host_free(rio_placement *h, void *pinned);
rio_status  rio_cuda_memcpy_h2d(rio_placement *h, void *dev, const void *host, size_t bytes);  /* async */
rio_status  rio_cuda_memcpy_d2h(rio_placement *h, void *host, const void *dev, size_t bytes);  /* async */
rio_status  rio_cuda_assign_batch_dev(rio_placement *h, const uint64_t *d_keys, const float *d_obj_feats,
                                      size_t n, uint32_t *d_out_idx);
rio_status  rio_cuda_assign_ranked_batch_dev(rio_placement *h, const uint64_t *d_keys, size_t n, uint32_t ranks, uint32_t *d_out_idx);
rio_status  rio_cuda_assign_ranked_spread_batch_dev(rio_placement *h, const uint64_t *d_keys, size_t n, uint32_t ranks, uint32_t *d_out_idx);
rio_status  rio_cuda_assign_ranked_affinity_batch_dev(rio_placement *h, const float *d_obj_feats, size_t n, uint32_t ranks, uint32_t *d_out_idx);
rio_status  rio_cuda_assign_ranked_affinity_spread_batch_dev(rio_placement *h, const float *d_obj_feats, size_t n, uint32_t ranks, uint32_t *d_out_idx);
rio_status  rio_cuda_lookup_batch_dev(rio_placement *h, const uint64_t *d_keys, size_t n, uint32_t *d_out_idx);
rio_status  rio_cuda_upsert_batch_dev(rio_placement *h, const uint64_t *d_keys, const uint32_t *d_idx, size_t n);
/* pre-size the directory for n more distinct keys (the _dev upsert cannot grow it mid-stream) */
rio_status  rio_cuda_directory_reserve(rio_placement *h, uint64_t n_more);

/* ---- string-level provider calls: exactly what `impl ObjectPlacement for GpuObjectPlacement` forwards ---- */
/* update(ObjectPlacementItem): address==NULL is server_address: None (mod.rs:46-49, local.rs:34-38) */
rio_status  rio_cuda_update_str(rio_placement *h, const char *type, size_t type_len, const char *id, size_t id_len,
                                const char *address, size_t address_len);
/* lookup(&ObjectId) -> Option<String>: *out_len = (size_t)-1 for None; the address is copied into buf */
rio_status  rio_cuda_lookup_str(rio_placement *h, const char *type, size_t type_len, const char *id, size_t id_len,
                                char *buf, size_t cap, size_t *out_len);
rio_status  rio_cuda_clean_server_str(rio_placement *h, const char *address, size_t address_len);
rio_status  rio_cuda_remove_str(rio_placement *h, const char *type, size_t type_len, const char *id, size_t id_len);

/* ---- micro-batching resolver: the per-request call site (service.rs:193-254), coalesced ------------------------- */
/* Service runs get_or_create_placement once per request on one task per connection (server.rs:303).  Concurrent
 * rio_cuda_resolver_resolve calls (any number of threads) are coalesced into one rio_cuda_place_batch as soon as
 * max_batch requests are pending or the oldest has waited max_wait_us; every caller gets its own answer back. */
typedef struct rio_resolver rio_resolver;
rio_status  rio_cuda_resolver_create(rio_placement *h, uint32_t policy, uint32_t self_idx, uint32_t max_batch,
                                     uint32_t max_wait_us, rio_resolver **out);
void        rio_cuda_resolver_destroy(rio_resolver *r);
rio_status  rio_cuda_resolver_resolve(rio_resolver *r, uint64_t key, uint32_t *out_idx);
rio_status  rio_cuda_resolver_resolve_str(rio_resolver *r, const char *type, size_t type_len, const char *id, size_t id_len,
                                          char *buf, size_t cap, size_t *out_len);
/* The trait's own per-id calls through the same queue (lookup / update / remove, mod.rs:46-55): concurrent callers share one
 * GPU round trip.  Inside one micro-batch the updates are applied first (in submission order), then the lookups, then the
 * resolves.  update with idx == RIO_NONE (or address == NULL) is update(None) = remove. */
rio_status  rio_cuda_resolver_lookup(rio_resolver *r, uint64_t key, uint32_t *out_idx);
rio_status  rio_cuda_resolver_update(rio_resolver *r, uint64_t key, uint32_t idx);
rio_status  rio_cuda_resolver_lookup_str(rio_resolver *r, const char *type, size_t type_len, const char *id, size_t id_len,
                                         char *buf, size_t cap, size_t *out_len);
rio_status  rio_cuda_resolver_update_str(rio_resolver *r, const char *type, size_t type_len, const char *id, size_t id_len,
                                         const char *address, size_t address_len);
rio_status  rio_cuda_resolver_stats(rio_resolver *r, uint64_t *calls, uint64_t *batches, uint64_t *largest_batch);
const char *rio_cuda_resolver_last_error(void);

/* ---- durable write-through into the reference's SQLite schema (SURVEY 8f row 3) -------------------------------------------
 * SqliteObjectPlacement (sqlite.rs:58-126) in front of which the GPU directory sits as the cache: the table
 * `object_placement(struct_name, object_id, server_address)` of migrations/0001-sqlite-init.sql:1-9 is the source of truth across
 * restarts, every call below executes the reference's own SQL text and the matching GPU mutation; lookups are answered by the
 * GPU directory.  libsqlite3.so.0 is dlopen'ed on first use.  Errors: RIO_ERR_UPSTREAM (SQLite / CUDA) like the reference's
 * From<sqlx::Error> (errors.rs:145-152); message in rio_cuda_durable_last_error() (thread-local). */
typedef struct rio_durable rio_durable;
rio_status  rio_cuda_durable_open(rio_placement *h, const char *path, rio_durable **out);      /* prepare(): migration in one transaction */
void        rio_cuda_durable_close(rio_durable *d);
rio_status  rio_cuda_durable_recover(rio_durable *d, uint64_t *out_rows);                      /* table -> GPU directory, in bulk */
rio_status  rio_cuda_durable_update(rio_durable *d, const char *type, size_t type_len, const char *id, size_t id_len,
                                    const char *address, size_t address_len);                  /* address NULL = update(None) = remove */
rio_status  rio_cuda_durable_lookup(rio_durable *d, const char *type, size_t type_len, const char *id, size_t id_len,
                                    char *buf, size_t cap, size_t *out_len);
rio_status  rio_cuda_durable_clean_server(rio_durable *d, const char *address, size_t address_len);
rio_status  rio_cuda_durable_remove(rio_durable *d, const char *type, size_t type_len, const char *id, size_t id_len);
/* n NUL-terminated (type, id, address-or-NULL) triples: ONE transaction on the table + one batched upsert on the GPU */
rio_status  rio_cuda_durable_update_batch(rio_durable *d, const char *const *types, const char *const *ids,
                                          const char *const *addresses, size_t n);
/* get_or_create_placement for n ids (service.rs:193-254) decided on the GPU, then written through in ONE transaction: rows of the
 * inactive servers the batch met are deleted (clean_server), changed placements upserted */
rio_status  rio_cuda_durable_place_batch(rio_durable *d, const char *const *types, const char *const *ids, size_t n,
                                         uint32_t policy, uint32_t self_idx, uint32_t *out_idx);
const char *rio_cuda_durable_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* RIO_CUDA_H */

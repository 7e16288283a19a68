//! Raw bindings for `include/rio_cuda.h` (ABI version 2).  One declaration per exported symbol.
#![allow(non_camel_case_types)]
use libc::{c_char, c_void, size_t};

pub type rio_status = i32;
pub const RIO_OK: rio_status = 0;
pub const RIO_ERR_UPSTREAM: rio_status = -1; // -> ObjectPlacementError::Upstream
pub const RIO_ERR_UNKNOWN: rio_status = -2; // -> ObjectPlacementError::Unknown
pub const RIO_NONE: u32 = 0xFFFF_FFFF;
pub const RIO_PLACE_SELF: u32 = 0;
pub const RIO_PLACE_HRW: u32 = 1;
pub const RIO_PLACE_HRW2: u32 = 2;
pub const RIO_SOLVER_HRW: u32 = 1;
pub const RIO_SOLVER_HRW2: u32 = 2;
pub const RIO_EV_JOIN: u32 = 1;
pub const RIO_EV_LEAVE: u32 = 2;
pub const RIO_COMM_ID_BYTES: usize = 128;
pub const RIO_MAX_RANKS: u32 = 8;

#[repr(C)]
pub struct rio_placement {
    _private: [u8; 0],
}
#[repr(C)]
pub struct rio_objset {
    _private: [u8; 0],
}
#[repr(C)]
pub struct rio_durable { _private: [u8; 0] }
#[repr(C)]
pub struct rio_resolver {
    _private: [u8; 0],
}
#[repr(C)]
#[derive(Clone, Copy, Default)]
pub struct rio_config {
    pub struct_size: u32,
    pub device: i32,
    pub directory_capacity: u64,
    pub flags: u32,
    pub reserved: u32,
}

extern "C" {
    pub fn rio_cuda_abi_version() -> u32;
    pub fn rio_cuda_create(cfg: *const rio_config, out: *mut *mut rio_placement) -> rio_status;
    pub fn rio_cuda_destroy(h: *mut rio_placement);
    pub fn rio_cuda_last_error(h: *mut rio_placement) -> *const c_char;
    pub fn rio_cuda_sync(h: *mut rio_placement) -> rio_status;
    pub fn rio_cuda_device_info(h: *mut rio_placement, device: *mut i32, sm_count: *mut i32, hbm_bytes: *mut u64, name_buf: *mut c_char, name_cap: size_t) -> rio_status;

    pub fn rio_cuda_object_key(ty: *const c_char, ty_len: size_t, id: *const c_char, id_len: size_t) -> u64;
    pub fn rio_cuda_node_seed(address: *const c_char, len: size_t) -> u64;
    pub fn rio_cuda_hash_ids(h: *mut rio_placement, packed: *const c_char, offsets: *const u64, n: size_t, out_keys: *mut u64) -> rio_status;

    pub fn rio_cuda_set_nodes(h: *mut rio_placement, addrs: *const *const c_char, weights: *const u32, feats: *const f32, m: u32, k: u32, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_node_upsert(h: *mut rio_placement, address: *const c_char, weight: u32, feat: *const f32, k: u32, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_node_set_active(h: *mut rio_placement, idx: u32, active: i32) -> rio_status;
    pub fn rio_cuda_node_index(h: *mut rio_placement, address: *const c_char, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_node_intern(h: *mut rio_placement, address: *const c_char, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_node_address(h: *mut rio_placement, idx: u32, buf: *mut c_char, cap: size_t, out_len: *mut size_t) -> rio_status;
    pub fn rio_cuda_node_count(h: *mut rio_placement, out_total: *mut u32, out_live: *mut u32) -> rio_status;
    pub fn rio_cuda_assign_bounded_batch(h: *mut rio_placement, keys: *const u64, n: usize, n_total: u64, cap_num: u32, cap_den: u32, max_rounds: u32, out_idx: *mut u32, out_passes: *mut u32) -> rio_status;
    pub fn rio_cuda_assign_bounded_affinity_batch(h: *mut rio_placement, keys: *const u64, obj_feats: *const f32, n: usize, n_total: u64, cap_num: u32, cap_den: u32, max_rounds: u32, out_idx: *mut u32, out_passes: *mut u32) -> rio_status;
    pub fn rio_cuda_assign_bounded_weighted_batch(h: *mut rio_placement, keys: *const u64, obj_feats: *const f32, weights: *const u32, n: usize, load_total: u64, cap_num: u32, cap_den: u32, max_rounds: u32, out_idx: *mut u32, out_passes: *mut u32) -> rio_status;
    pub fn rio_cuda_check_address_batch(h: *mut rio_placement, addr_idx: *const u32, n: usize, self_idx: u32, out_verdict: *mut u8, out_cleaned: *mut u64) -> rio_status;
    pub fn rio_cuda_node_state(h: *mut rio_placement, idx: u32, active: *mut i32, weight: *mut u32, malformed: *mut i32) -> rio_status;
    pub fn rio_cuda_node_set_domains(h: *mut rio_placement, idx: *const u32, domain: *const u32, k: size_t) -> rio_status;
    pub fn rio_cuda_node_domain(h: *mut rio_placement, idx: u32, out_domain: *mut u32) -> rio_status;
    pub fn rio_cuda_set_solver(h: *mut rio_placement, solver: u32, trie_bits: u32) -> rio_status;
    pub fn rio_cuda_get_solver(h: *mut rio_placement, solver: *mut u32, trie_bits: *mut u32) -> rio_status;

    pub fn rio_cuda_lookup_batch(h: *mut rio_placement, keys: *const u64, n: size_t, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_upsert_batch(h: *mut rio_placement, keys: *const u64, idx: *const u32, n: size_t) -> rio_status;
    pub fn rio_cuda_remove_batch(h: *mut rio_placement, keys: *const u64, n: size_t) -> rio_status;
    pub fn rio_cuda_clean_node(h: *mut rio_placement, idx: u32, out_removed: *mut u64) -> rio_status;
    pub fn rio_cuda_directory_len(h: *mut rio_placement, out_placed: *mut u64, out_slots: *mut u64) -> rio_status;
    pub fn rio_cuda_directory_reserve(h: *mut rio_placement, n_more: u64) -> rio_status;

    pub fn rio_cuda_assign_batch(h: *mut rio_placement, keys: *const u64, obj_feats: *const f32, n: size_t, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_assign_ranked_batch(h: *mut rio_placement, keys: *const u64, n: size_t, ranks: u32, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_assign_ranked_spread_batch(h: *mut rio_placement, keys: *const u64, n: size_t, ranks: u32, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_assign_ranked_affinity_batch(h: *mut rio_placement, obj_feats: *const f32, n: size_t, ranks: u32, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_assign_ranked_affinity_spread_batch(h: *mut rio_placement, obj_feats: *const f32, n: size_t, ranks: u32, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_place_batch(h: *mut rio_placement, keys: *const u64, n: size_t, policy: u32, self_idx: u32, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_rebalance(h: *mut rio_placement, event: u32, idx: u32, out_moved: *mut u64) -> rio_status;
    pub fn rio_cuda_rebalance_changes(h: *mut rio_placement, idx: *const u32, prev_weight: *const u32, k: size_t, out_moved: *mut u64) -> rio_status;
    pub fn rio_cuda_load_counters(h: *mut rio_placement, out: *mut u32, cap: u32) -> rio_status;

    pub fn rio_cuda_set_create(h: *mut rio_placement, capacity: u64, out: *mut *mut rio_objset) -> rio_status;
    pub fn rio_cuda_set_destroy(s: *mut rio_objset);
    pub fn rio_cuda_set_load_keys(s: *mut rio_objset, keys: *const u64, n: u64) -> rio_status;
    pub fn rio_cuda_set_load_feats(s: *mut rio_objset, feats: *const f32, k: u32) -> rio_status;
    pub fn rio_cuda_set_assign(s: *mut rio_objset, use_affinity: u32) -> rio_status;
    pub fn rio_cuda_set_assign_bounded(s: *mut rio_objset, n_total: u64, cap_num: u32, cap_den: u32, max_rounds: u32, out_passes: *mut u32) -> rio_status;
    pub fn rio_cuda_set_assign_bounded_begin(s: *mut rio_objset, n_total: u64, cap_num: u32, cap_den: u32, max_rounds: u32) -> rio_status;
    pub fn rio_cuda_set_assign_bounded_end(s: *mut rio_objset, out_passes: *mut u32) -> rio_status;
    pub fn rio_cuda_set_assign_bounded_affinity(s: *mut rio_objset, n_total: u64, cap_num: u32, cap_den: u32, max_rounds: u32, out_passes: *mut u32) -> rio_status;
    pub fn rio_cuda_set_rebalance_changes_bounded_affinity(s: *mut rio_objset, idx: *const u32, prev_weight: *const u32, k: size_t, n_total: u64, cap_num: u32, cap_den: u32, max_rounds: u32, out_moved: *mut u64, out_passes: *mut u32) -> rio_status;
    pub fn rio_cuda_set_insert(s: *mut rio_objset, keys: *const u64, feats: *const f32, m: u64, out_first: *mut u64) -> rio_status;
    pub fn rio_cuda_set_erase(s: *mut rio_objset, keys: *const u64, m: u64, out_erased: *mut u64) -> rio_status;
    pub fn rio_cuda_set_write_weights(s: *mut rio_objset, first: u64, n: u64, w: *const u32) -> rio_status;
    pub fn rio_cuda_set_read_weights(s: *mut rio_objset, first: u64, n: u64, out: *mut u32) -> rio_status;
    pub fn rio_cuda_set_assign_bounded_weighted(s: *mut rio_objset, use_affinity: u32, load_total: u64, cap_num: u32, cap_den: u32, max_rounds: u32, out_passes: *mut u32) -> rio_status;
    pub fn rio_cuda_set_loads(s: *mut rio_objset, out: *mut u32, cap: u32) -> rio_status;
    pub fn rio_cuda_set_write_weights_by_key(s: *mut rio_objset, keys: *const u64, w: *const u32, m: usize, out_written: *mut u64) -> rio_status;
    pub fn rio_cuda_set_rebalance_changes_bounded_weighted(s: *mut rio_objset, idx: *const u32, prev_weight: *const u32, k: usize, load_total: u64, cap_num: u32, cap_den: u32, max_rounds: u32, out_moved: *mut u64, out_passes: *mut u32) -> rio_status;
    pub fn rio_cuda_set_rebalance(s: *mut rio_objset, event: u32, idx: u32, out_moved: *mut u64) -> rio_status;
    pub fn rio_cuda_set_rebalance_changes(s: *mut rio_objset, idx: *const u32, prev_weight: *const u32, k: size_t, out_moved: *mut u64) -> rio_status;
    pub fn rio_cuda_set_assign_ranked(s: *mut rio_objset, ranks: u32) -> rio_status;
    pub fn rio_cuda_set_read_ranked(s: *mut rio_objset, first: u64, n: u64, out: *mut u32) -> rio_status;
    pub fn rio_cuda_set_rebalance_changes_ranked(s: *mut rio_objset, idx: *const u32, prev_weight: *const u32, k: size_t, out_moved: *mut u64,
                                                 out_changed: *mut u64) -> rio_status;
    pub fn rio_cuda_set_assign_ranked_spread(s: *mut rio_objset, ranks: u32) -> rio_status;
    pub fn rio_cuda_set_assign_ranked_affinity(s: *mut rio_objset, ranks: u32) -> rio_status;
    pub fn rio_cuda_set_assign_ranked_affinity_spread(s: *mut rio_objset, ranks: u32) -> rio_status;
    pub fn rio_cuda_set_counters(s: *mut rio_objset, out: *mut u32, cap: u32) -> rio_status;
    pub fn rio_cuda_set_read(s: *mut rio_objset, first: u64, n: u64, out_keys: *mut u64, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_set_size(s: *mut rio_objset, out_n: *mut u64) -> rio_status;
    pub fn rio_cuda_set_commit(s: *mut rio_objset) -> rio_status;
    pub fn rio_cuda_set_commit_changes(s: *mut rio_objset, dry_run: u32, cap: u64, out_rows: *mut u64, out_keys: *mut u64, out_from: *mut u32, out_to: *mut u32, out_n: *mut u64) -> rio_status;

    pub fn rio_cuda_comm_unique_id(out_id: *mut u8) -> rio_status;
    pub fn rio_cuda_comm_init(h: *mut rio_placement, rank: i32, world: i32, id: *const u8) -> rio_status;
    pub fn rio_cuda_comm_ipc_export(h: *mut rio_placement, world: i32, max_nodes: u32, out_handle: *mut u8) -> rio_status;
    pub fn rio_cuda_comm_ipc_attach(h: *mut rio_placement, rank: i32, world: i32, handles: *const u8) -> rio_status;
    pub fn rio_cuda_comm_info(h: *mut rio_placement, rank: *mut i32, world: *mut i32) -> rio_status;
    pub fn rio_cuda_comm_sum_counters(h: *mut rio_placement, inout: *mut u32, m: u32) -> rio_status;

    pub fn rio_cuda_dev_alloc(h: *mut rio_placement, bytes: size_t, out_dev: *mut *mut c_void) -> rio_status;
    pub fn rio_cuda_dev_free(h: *mut rio_placement, dev: *mut c_void) -> rio_status;
    pub fn rio_cuda_host_alloc(h: *mut rio_placement, bytes: size_t, out_pinned: *mut *mut c_void) -> rio_status;
    pub fn rio_cuda_host_free(h: *mut rio_placement, pinned: *mut c_void) -> rio_status;
    pub fn rio_cuda_memcpy_h2d(h: *mut rio_placement, dev: *mut c_void, host: *const c_void, bytes: size_t) -> rio_status;
    pub fn rio_cuda_memcpy_d2h(h: *mut rio_placement, host: *mut c_void, dev: *const c_void, bytes: size_t) -> rio_status;
    pub fn rio_cuda_assign_batch_dev(h: *mut rio_placement, d_keys: *const u64, d_obj_feats: *const f32, n: size_t, d_out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_assign_ranked_batch_dev(h: *mut rio_placement, d_keys: *const u64, n: size_t, ranks: u32, d_out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_assign_ranked_spread_batch_dev(h: *mut rio_placement, d_keys: *const u64, n: size_t, ranks: u32, d_out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_assign_ranked_affinity_batch_dev(h: *mut rio_placement, d_obj_feats: *const f32, n: size_t, ranks: u32, d_out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_assign_ranked_affinity_spread_batch_dev(h: *mut rio_placement, d_obj_feats: *const f32, n: size_t, ranks: u32, d_out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_lookup_batch_dev(h: *mut rio_placement, d_keys: *const u64, n: size_t, d_out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_upsert_batch_dev(h: *mut rio_placement, d_keys: *const u64, d_idx: *const u32, n: size_t) -> rio_status;

    pub fn rio_cuda_resolver_create(h: *mut rio_placement, policy: u32, self_idx: u32, max_batch: u32, max_wait_us: u32, out: *mut *mut rio_resolver) -> rio_status;
    pub fn rio_cuda_resolver_destroy(r: *mut rio_resolver);
    pub fn rio_cuda_resolver_resolve(r: *mut rio_resolver, key: u64, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_resolver_resolve_str(r: *mut rio_resolver, ty: *const c_char, ty_len: size_t, id: *const c_char, id_len: size_t, buf: *mut c_char, cap: size_t, out_len: *mut size_t) -> rio_status;
    pub fn rio_cuda_resolver_lookup(r: *mut rio_resolver, key: u64, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_resolver_update(r: *mut rio_resolver, key: u64, idx: u32) -> rio_status;
    pub fn rio_cuda_resolver_lookup_str(r: *mut rio_resolver, ty: *const c_char, ty_len: usize, id: *const c_char, id_len: usize, buf: *mut c_char, cap: usize, out_len: *mut usize) -> rio_status;
    pub fn rio_cuda_resolver_update_str(r: *mut rio_resolver, ty: *const c_char, ty_len: usize, id: *const c_char, id_len: usize, address: *const c_char, address_len: usize) -> rio_status;
    pub fn rio_cuda_resolver_stats(r: *mut rio_resolver, calls: *mut u64, batches: *mut u64, largest_batch: *mut u64) -> rio_status;
    pub fn rio_cuda_resolver_last_error() -> *const c_char;

    pub fn rio_cuda_durable_open(h: *mut rio_placement, path: *const c_char, out: *mut *mut rio_durable) -> rio_status;
    pub fn rio_cuda_durable_close(d: *mut rio_durable);
    pub fn rio_cuda_durable_recover(d: *mut rio_durable, out_rows: *mut u64) -> rio_status;
    pub fn rio_cuda_durable_update(d: *mut rio_durable, ty: *const c_char, ty_len: usize, id: *const c_char, id_len: usize, address: *const c_char, address_len: usize) -> rio_status;
    pub fn rio_cuda_durable_lookup(d: *mut rio_durable, ty: *const c_char, ty_len: usize, id: *const c_char, id_len: usize, buf: *mut c_char, cap: usize, out_len: *mut usize) -> rio_status;
    pub fn rio_cuda_durable_clean_server(d: *mut rio_durable, address: *const c_char, address_len: usize) -> rio_status;
    pub fn rio_cuda_durable_remove(d: *mut rio_durable, ty: *const c_char, ty_len: usize, id: *const c_char, id_len: usize) -> rio_status;
    pub fn rio_cuda_durable_update_batch(d: *mut rio_durable, types: *const *const c_char, ids: *const *const c_char, addresses: *const *const c_char, n: usize) -> rio_status;
    pub fn rio_cuda_durable_place_batch(d: *mut rio_durable, types: *const *const c_char, ids: *const *const c_char, n: usize, policy: u32, self_idx: u32, out_idx: *mut u32) -> rio_status;
    pub fn rio_cuda_durable_last_error() -> *const c_char;
    pub fn rio_cuda_update_str(h: *mut rio_placement, ty: *const c_char, ty_len: size_t, id: *const c_char, id_len: size_t, address: *const c_char, address_len: size_t) -> rio_status;
    pub fn rio_cuda_lookup_str(h: *mut rio_placement, ty: *const c_char, ty_len: size_t, id: *const c_char, id_len: size_t, buf: *mut c_char, cap: size_t, out_len: *mut size_t) -> rio_status;
    pub fn rio_cuda_clean_server_str(h: *mut rio_placement, address: *const c_char, address_len: size_t) -> rio_status;
    pub fn rio_cuda_remove_str(h: *mut rio_placement, ty: *const c_char, ty_len: size_t, id: *const c_char, id_len: size_t) -> rio_status;
}

"""ctypes binding of include/rio_cuda.h (the same declarations a rio-cuda-sys crate would carry)."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
NONE = 0xFFFFFFFF
RIO_OK, RIO_ERR_UPSTREAM, RIO_ERR_UNKNOWN = 0, -1, -2
PLACE_SELF, PLACE_HRW, PLACE_HRW2 = 0, 1, 2
SOLVER_HRW, SOLVER_HRW2 = 1, 2
EV_JOIN, EV_LEAVE = 1, 2
COMM_ID_BYTES = 128
MAX_RANKS = 8

_lib = None


def library_path():
    return os.path.join(HERE, "librio_cuda.so")


class RioConfig(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32),
        ("device", C.c_int32),
        ("directory_capacity", C.c_uint64),
        ("flags", C.c_uint32),
        ("reserved", C.c_uint32),
    ]


H = C.c_void_p
u8p, u32p, u64p, f32p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_float)
vp, sz = C.c_void_p, C.c_size_t

# name -> (restype, argtypes); must list EVERY function declared in include/rio_cuda.h (tests/test_abi.py checks)
SIGNATURES = {
    "rio_cuda_abi_version": (C.c_uint32, []),
    "rio_cuda_create": (C.c_int32, [C.POINTER(RioConfig), C.POINTER(H)]),
    "rio_cuda_destroy": (None, [H]),
    "rio_cuda_last_error": (C.c_char_p, [H]),
    "rio_cuda_sync": (C.c_int32, [H]),
    "rio_cuda_device_info": (C.c_int32, [H, C.POINTER(C.c_int32), C.POINTER(C.c_int32), u64p, C.c_char_p, sz]),
    "rio_cuda_object_key": (C.c_uint64, [C.c_char_p, sz, C.c_char_p, sz]),
    "rio_cuda_node_seed": (C.c_uint64, [C.c_char_p, sz]),
    "rio_cuda_hash_ids": (C.c_int32, [H, vp, vp, sz, vp]),
    "rio_cuda_set_nodes": (C.c_int32, [H, C.POINTER(C.c_char_p), vp, vp, C.c_uint32, C.c_uint32, vp]),
    "rio_cuda_node_upsert": (C.c_int32, [H, C.c_char_p, C.c_uint32, vp, C.c_uint32, u32p]),
    "rio_cuda_node_set_active": (C.c_int32, [H, C.c_uint32, C.c_int32]),
    "rio_cuda_node_index": (C.c_int32, [H, C.c_char_p, u32p]),
    "rio_cuda_node_intern": (C.c_int32, [H, C.c_char_p, u32p]),
    "rio_cuda_node_address": (C.c_int32, [H, C.c_uint32, C.c_char_p, sz, C.POINTER(sz)]),
    "rio_cuda_node_count": (C.c_int32, [H, u32p, u32p]),
    "rio_cuda_node_state": (C.c_int32, [H, C.c_uint32, C.POINTER(C.c_int32), u32p, C.POINTER(C.c_int32)]),
    "rio_cuda_node_set_domains": (C.c_int32, [H, vp, vp, sz]),
    "rio_cuda_node_domain": (C.c_int32, [H, C.c_uint32, u32p]),
    "rio_cuda_set_solver": (C.c_int32, [H, C.c_uint32, C.c_uint32]),
    "rio_cuda_get_solver": (C.c_int32, [H, u32p, u32p]),
    "rio_cuda_lookup_batch": (C.c_int32, [H, vp, sz, vp]),
    "rio_cuda_upsert_batch": (C.c_int32, [H, vp, vp, sz]),
    "rio_cuda_remove_batch": (C.c_int32, [H, vp, sz]),
    "rio_cuda_clean_node": (C.c_int32, [H, C.c_uint32, u64p]),
    "rio_cuda_directory_len": (C.c_int32, [H, u64p, u64p]),
    "rio_cuda_assign_batch": (C.c_int32, [H, vp, vp, sz, vp]),
    "rio_cuda_assign_bounded_batch": (C.c_int32, [H, vp, sz, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, vp, u32p]),
    "rio_cuda_assign_bounded_affinity_batch": (C.c_int32, [H, vp, vp, sz, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, vp, u32p]),
    "rio_cuda_assign_bounded_weighted_batch": (C.c_int32, [H, vp, vp, vp, sz, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, vp, u32p]),
    "rio_cuda_assign_ranked_batch": (C.c_int32, [H, vp, sz, C.c_uint32, vp]),
    "rio_cuda_assign_ranked_batch_dev": (C.c_int32, [H, vp, sz, C.c_uint32, vp]),
    "rio_cuda_assign_ranked_spread_batch": (C.c_int32, [H, vp, sz, C.c_uint32, vp]),
    "rio_cuda_assign_ranked_spread_batch_dev": (C.c_int32, [H, vp, sz, C.c_uint32, vp]),
    "rio_cuda_assign_ranked_affinity_batch": (C.c_int32, [H, vp, sz, C.c_uint32, vp]),
    "rio_cuda_assign_ranked_affinity_batch_dev": (C.c_int32, [H, vp, sz, C.c_uint32, vp]),
    "rio_cuda_assign_ranked_affinity_spread_batch": (C.c_int32, [H, vp, sz, C.c_uint32, vp]),
    "rio_cuda_assign_ranked_affinity_spread_batch_dev": (C.c_int32, [H, vp, sz, C.c_uint32, vp]),
    "rio_cuda_check_address_batch": (C.c_int32, [H, vp, sz, C.c_uint32, vp, u64p]),
    "rio_cuda_place_batch": (C.c_int32, [H, vp, sz, C.c_uint32, C.c_uint32, vp]),
    "rio_cuda_rebalance": (C.c_int32, [H, C.c_uint32, C.c_uint32, u64p]),
    "rio_cuda_rebalance_changes": (C.c_int32, [H, vp, vp, sz, u64p]),
    "rio_cuda_load_counters": (C.c_int32, [H, vp, C.c_uint32]),
    "rio_cuda_set_create": (C.c_int32, [H, C.c_uint64, C.POINTER(H)]),
    "rio_cuda_set_destroy": (None, [H]),
    "rio_cuda_set_load_keys": (C.c_int32, [H, vp, C.c_uint64]),
    "rio_cuda_set_load_feats": (C.c_int32, [H, vp, C.c_uint32]),
    "rio_cuda_set_assign": (C.c_int32, [H, C.c_uint32]),
    "rio_cuda_set_assign_bounded": (C.c_int32, [H, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, u32p]),
    "rio_cuda_set_assign_bounded_begin": (C.c_int32, [H, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32]),
    "rio_cuda_set_assign_bounded_end": (C.c_int32, [H, u32p]),
    "rio_cuda_set_assign_bounded_affinity": (C.c_int32, [H, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, u32p]),
    "rio_cuda_set_rebalance_changes_bounded_affinity": (C.c_int32, [H, vp, vp, sz, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, u64p, u32p]),
    "rio_cuda_set_insert": (C.c_int32, [H, vp, vp, C.c_uint64, u64p]),
    "rio_cuda_set_erase": (C.c_int32, [H, vp, C.c_uint64, u64p]),
    "rio_cuda_set_write_weights": (C.c_int32, [H, C.c_uint64, C.c_uint64, vp]),
    "rio_cuda_set_read_weights": (C.c_int32, [H, C.c_uint64, C.c_uint64, vp]),
    "rio_cuda_set_assign_bounded_weighted": (C.c_int32, [H, C.c_uint32, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, u32p]),
    "rio_cuda_set_loads": (C.c_int32, [H, vp, C.c_uint32]),
    "rio_cuda_set_write_weights_by_key": (C.c_int32, [H, vp, vp, sz, u64p]),
    "rio_cuda_set_rebalance_changes_bounded_weighted": (C.c_int32, [H, vp, vp, sz, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, u64p, u32p]),
    "rio_cuda_set_rebalance": (C.c_int32, [H, C.c_uint32, C.c_uint32, u64p]),
    "rio_cuda_set_rebalance_changes": (C.c_int32, [H, vp, vp, sz, u64p]),
    "rio_cuda_set_assign_ranked": (C.c_int32, [H, C.c_uint32]),
    "rio_cuda_set_read_ranked": (C.c_int32, [H, C.c_uint64, C.c_uint64, vp]),
    "rio_cuda_set_rebalance_changes_ranked": (C.c_int32, [H, vp, vp, sz, u64p, u64p]),
    "rio_cuda_set_assign_ranked_spread": (C.c_int32, [H, C.c_uint32]),
    "rio_cuda_set_assign_ranked_affinity": (C.c_int32, [H, C.c_uint32]),
    "rio_cuda_set_assign_ranked_affinity_spread": (C.c_int32, [H, C.c_uint32]),
    "rio_cuda_set_counters": (C.c_int32, [H, vp, C.c_uint32]),
    "rio_cuda_set_read": (C.c_int32, [H, C.c_uint64, C.c_uint64, vp, vp]),
    "rio_cuda_set_size": (C.c_int32, [H, u64p]),
    "rio_cuda_set_commit": (C.c_int32, [H]),
    "rio_cuda_set_commit_changes": (C.c_int32, [H, C.c_uint32, C.c_uint64, vp, vp, vp, vp, u64p]),
    "rio_cuda_comm_unique_id": (C.c_int32, [vp]),
    "rio_cuda_comm_init": (C.c_int32, [H, C.c_int32, C.c_int32, vp]),
    "rio_cuda_comm_ipc_export": (C.c_int32, [H, C.c_int32, C.c_uint32, vp]),
    "rio_cuda_comm_ipc_attach": (C.c_int32, [H, C.c_int32, C.c_int32, vp]),
    "rio_cuda_comm_info": (C.c_int32, [H, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "rio_cuda_comm_sum_counters": (C.c_int32, [H, vp, C.c_uint32]),
    "rio_cuda_dev_alloc": (C.c_int32, [H, sz, C.POINTER(vp)]),
    "rio_cuda_dev_free": (C.c_int32, [H, vp]),
    "rio_cuda_host_alloc": (C.c_int32, [H, sz, C.POINTER(vp)]),
    "rio_cuda_host_free": (C.c_int32, [H, vp]),
    "rio_cuda_memcpy_h2d": (C.c_int32, [H, vp, vp, sz]),
    "rio_cuda_memcpy_d2h": (C.c_int32, [H, vp, vp, sz]),
    "rio_cuda_assign_batch_dev": (C.c_int32, [H, vp, vp, sz, vp]),
    "rio_cuda_lookup_batch_dev": (C.c_int32, [H, vp, sz, vp]),
    "rio_cuda_upsert_batch_dev": (C.c_int32, [H, vp, vp, sz]),
    "rio_cuda_directory_reserve": (C.c_int32, [H, C.c_uint64]),
    "rio_cuda_resolver_create": (C.c_int32, [H, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.POINTER(H)]),
    "rio_cuda_resolver_destroy": (None, [H]),
    "rio_cuda_resolver_resolve": (C.c_int32, [H, C.c_uint64, u32p]),
    "rio_cuda_resolver_resolve_str": (C.c_int32, [H, C.c_char_p, sz, C.c_char_p, sz, C.c_char_p, sz, C.POINTER(sz)]),
    "rio_cuda_resolver_lookup": (C.c_int32, [H, C.c_uint64, u32p]),
    "rio_cuda_resolver_update": (C.c_int32, [H, C.c_uint64, C.c_uint32]),
    "rio_cuda_resolver_lookup_str": (C.c_int32, [H, C.c_char_p, sz, C.c_char_p, sz, C.c_char_p, sz, C.POINTER(sz)]),
    "rio_cuda_resolver_update_str": (C.c_int32, [H, C.c_char_p, sz, C.c_char_p, sz, C.c_char_p, sz]),
    "rio_cuda_resolver_stats": (C.c_int32, [H, u64p, u64p, u64p]),
    "rio_cuda_resolver_last_error": (C.c_char_p, []),
    "rio_cuda_durable_open": (C.c_int32, [H, C.c_char_p, C.POINTER(H)]),
    "rio_cuda_durable_close": (None, [H]),
    "rio_cuda_durable_recover": (C.c_int32, [H, u64p]),
    "rio_cuda_durable_update": (C.c_int32, [H, C.c_char_p, sz, C.c_char_p, sz, C.c_char_p, sz]),
    "rio_cuda_durable_lookup": (C.c_int32, [H, C.c_char_p, sz, C.c_char_p, sz, C.c_char_p, sz, C.POINTER(sz)]),
    "rio_cuda_durable_clean_server": (C.c_int32, [H, C.c_char_p, sz]),
    "rio_cuda_durable_remove": (C.c_int32, [H, C.c_char_p, sz, C.c_char_p, sz]),
    "rio_cuda_durable_update_batch": (C.c_int32, [H, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), sz]),
    "rio_cuda_durable_place_batch": (C.c_int32, [H, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), sz, C.c_uint32, C.c_uint32, vp]),
    "rio_cuda_durable_last_error": (C.c_char_p, []),
    "rio_cuda_update_str": (C.c_int32, [H, C.c_char_p, sz, C.c_char_p, sz, C.c_char_p, sz]),
    "rio_cuda_lookup_str": (C.c_int32, [H, C.c_char_p, sz, C.c_char_p, sz, C.c_char_p, sz, C.POINTER(sz)]),
    "rio_cuda_clean_server_str": (C.c_int32, [H, C.c_char_p, sz]),
    "rio_cuda_remove_str": (C.c_int32, [H, C.c_char_p, sz, C.c_char_p, sz]),
}

# include/rio_cuda_dev.h: measurement and test hooks, not part of the provider ABI
DEV_SIGNATURES = {
    "rio_cuda_set_synth_keys": (C.c_int32, [H, C.c_uint64, C.c_uint64, C.c_uint64]),
    "rio_cuda_flush_l2": (C.c_int32, [H]),
    "rio_cuda_event_record": (C.c_int32, [H, C.c_uint32]),
    "rio_cuda_event_elapsed_ms": (C.c_int32, [H, C.c_uint32, C.c_uint32, C.POINTER(C.c_float)]),
    "rio_cuda_bench_mix_rate": (C.c_int32, [H, C.c_uint32, C.POINTER(C.c_double)]),
    "rio_cuda_launch_count": (C.c_int32, [H, u64p]),
    "rio_dev_set_node_seed": (C.c_int32, [H, C.c_uint32, C.c_uint64]),
    "rio_dev_set_table_options": (C.c_int32, [H, C.c_uint32]),
    "rio_dev_umma_timing": (C.c_int32, [H, vp]),
}
ADDR_LOCAL, ADDR_REDIRECT, ADDR_DEALLOCATE, ADDR_MALFORMED = 0, 1, 2, 3
DEV_SPLIT_CLASSES = 1


def lib():
    """Load librio_cuda.so.  Fails loudly when the CUDA extension has not been built (no fallback)."""
    global _lib
    if _lib is None:
        path = library_path()
        if not os.path.exists(path):
            raise ImportError(
                "rio_rs_b200/librio_cuda.so is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a).  There is no CPU fallback."
            )
        L = C.CDLL(path)
        for name, (res, args) in list(SIGNATURES.items()) + list(DEV_SIGNATURES.items()):
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib

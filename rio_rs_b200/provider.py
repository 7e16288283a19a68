"""Host-side mirror of the reference's ObjectPlacement interface over the C ABI (include/rio_cuda.h).

Same names, argument meaning and error behaviour as the Rust trait so the parity tests read like the
reference's own tests (rio-rs/tests/object_placement_backend.rs):

    trait ObjectPlacement { prepare, update, lookup, clean_server, remove }   object_placement/mod.rs:38-56

plus the batched calls the north star adds (lookup_many / update_many / assign_batch / place_batch /
rebalance).  The Rust crate `gpu_object_placement` in INTEGRATION.md is this file in Rust.
"""
import ctypes as C

import numpy as np

from . import _native as N


class ObjectPlacementError(Exception):
    """errors.rs:136-142"""


class Upstream(ObjectPlacementError):
    """ObjectPlacementError::Upstream(String): the CUDA / NCCL layer failed."""


class Unknown(ObjectPlacementError):
    """ObjectPlacementError::Unknown(String)."""


class ObjectId(tuple):
    """ObjectId(pub String, pub String) -- (struct name, object id); service_object.rs:19-26"""

    def __new__(cls, struct_name, object_id):
        return super().__new__(cls, (str(struct_name), str(object_id)))

    @classmethod
    def new(cls, struct_name, object_id):
        return cls(struct_name, object_id)


class ObjectPlacementItem:
    """object_placement/mod.rs:20-34"""

    def __init__(self, object_id, server_address):
        self.object_id = object_id
        self.server_address = server_address

    @classmethod
    def new(cls, object_id, server_address):
        return cls(object_id, server_address)


def _check(L, h, st):
    if st == N.RIO_OK:
        return
    msg = L.rio_cuda_last_error(h)
    msg = msg.decode(errors="replace") if msg else ""
    raise (Upstream if st == N.RIO_ERR_UPSTREAM else Unknown)(msg)


def _read_str(call, first=256):
    """String results of the C ABI (`buf, cap, out_len`; out_len == (size_t)-1 is None): a per-call buffer (callers may be
    threads sharing one provider), read again into a larger one when the call reports more bytes than it was given room for."""
    cap = first
    while True:
        buf, n = C.create_string_buffer(cap), C.c_size_t(0)
        call(buf, cap, C.byref(n))
        if n.value == C.c_size_t(-1).value:
            return None
        if n.value <= cap:
            return buf.raw[: n.value].decode()
        cap = n.value


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _change_set(idx, prev_weight):
    idx = np.ascontiguousarray(idx, dtype=np.uint32)
    prev = np.ascontiguousarray(prev_weight, dtype=np.uint32)
    if idx.shape != prev.shape or idx.ndim != 1:
        raise Unknown("idx and prev_weight must be 1-D arrays of one length")
    return idx, prev


def object_key(type_, id_):
    t, i = type_.encode(), id_.encode()
    return N.lib().rio_cuda_object_key(t, len(t), i, len(i))


class _Engine:
    """Owns the rio_placement handle; shared by provider clones (Arc in the Rust crate)."""

    def __init__(self, device=-1, directory_capacity=0):
        self.L = N.lib()
        cfg = N.RioConfig(C.sizeof(N.RioConfig), device, directory_capacity, 0, 0)
        h = N.H()
        st = self.L.rio_cuda_create(C.byref(cfg), C.byref(h))
        if st != N.RIO_OK:
            msg = self.L.rio_cuda_last_error(None)
            raise (Upstream if st == N.RIO_ERR_UPSTREAM else Unknown)(msg.decode(errors="replace") if msg else "")
        self.h = h
        self._deps = 0             # live object sets / resolvers created on this handle
        self._finalized = False

    # Object sets and resolvers hold raw pointers into the engine, so the handle must outlive them whatever order the interpreter
    # finalizes things in: objects that die together in one garbage cycle (an exception traceback that captured a test's locals is
    # enough) get their __del__ called in ARBITRARY order.  The engine is therefore destroyed by whoever goes last.
    def _retain(self):
        self._deps += 1

    def _release(self):
        self._deps -= 1
        if self._deps == 0 and self._finalized:
            self._destroy()

    def _destroy(self):
        try:
            if getattr(self, "h", None):
                self.L.rio_cuda_destroy(self.h)
                self.h = None
        except Exception:
            pass

    def __del__(self):
        self._finalized = True
        if getattr(self, "_deps", 0) == 0:
            self._destroy()


class GpuObjectPlacement:
    """impl ObjectPlacement for GpuObjectPlacement (the drop-in provider) + batched extensions."""

    def __init__(self, device=-1, directory_capacity=0, _engine=None):
        self._e = _engine or _Engine(device, directory_capacity)
        self.L = self._e.L
        self.h = self._e.h
        self._buf = C.create_string_buffer(512)

    def clone(self):
        """#[derive(Clone)]: clones share state (local.rs:75-114)."""
        return GpuObjectPlacement(_engine=self._e)

    def _ck(self, st):
        _check(self.L, self.h, st)

    # ---- the trait -------------------------------------------------------------------------------------
    def prepare(self):  # mod.rs:41-43 (default Ok(()))
        return None

    def update(self, object_placement):  # mod.rs:46-49 / local.rs:22-40
        t, i = (s.encode() for s in object_placement.object_id)
        a = object_placement.server_address
        ab = None if a is None else a.encode()
        self._ck(self.L.rio_cuda_update_str(self.h, t, len(t), i, len(i), ab, 0 if ab is None else len(ab)))

    def lookup(self, object_id):  # mod.rs:51 / local.rs:42-49 -> Option<String>
        t, i = (s.encode() for s in object_id)
        return _read_str(lambda buf, cap, n: self._ck(self.L.rio_cuda_lookup_str(self.h, t, len(t), i, len(i), buf, cap, n)))

    def clean_server(self, address):  # mod.rs:53 / local.rs:51-58
        a = address.encode()
        self._ck(self.L.rio_cuda_clean_server_str(self.h, a, len(a)))

    def remove(self, object_id):  # mod.rs:55 / local.rs:60-68
        t, i = (s.encode() for s in object_id)
        self._ck(self.L.rio_cuda_remove_str(self.h, t, len(t), i, len(i)))

    # ---- node table (MembershipStorage view) ---------------------------------------------------------
    def set_nodes(self, addresses, weights=None, feats=None):
        M = len(addresses)
        arr = (C.c_char_p * max(M, 1))(*[a.encode() for a in addresses])
        w = None if weights is None else np.ascontiguousarray(weights, dtype=np.uint32)
        f = None if feats is None else np.ascontiguousarray(feats, dtype=np.float32)
        K = 0 if f is None else f.shape[1]
        out = np.empty(max(M, 1), dtype=np.uint32)
        self._ck(self.L.rio_cuda_set_nodes(self.h, arr, _ptr(w), _ptr(f), M, K, _ptr(out)))
        return out[:M]

    def node_upsert(self, address, weight=1, feat=None):
        f = None if feat is None else np.ascontiguousarray(feat, dtype=np.float32)
        idx = C.c_uint32(0)
        self._ck(self.L.rio_cuda_node_upsert(self.h, address.encode(), weight, _ptr(f), 0 if f is None else len(f), C.byref(idx)))
        return idx.value

    def node_set_active(self, idx, active):
        self._ck(self.L.rio_cuda_node_set_active(self.h, idx, int(active)))

    def node_index(self, address):
        idx = C.c_uint32(0)
        self._ck(self.L.rio_cuda_node_index(self.h, address.encode(), C.byref(idx)))
        return None if idx.value == N.NONE else idx.value

    def node_intern(self, address):
        idx = C.c_uint32(0)
        self._ck(self.L.rio_cuda_node_intern(self.h, address.encode(), C.byref(idx)))
        return idx.value

    def node_address(self, idx):
        return _read_str(lambda buf, cap, n: self._ck(self.L.rio_cuda_node_address(self.h, idx, buf, cap, n)))

    def node_count(self):
        a, b = C.c_uint32(0), C.c_uint32(0)
        self._ck(self.L.rio_cuda_node_count(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def node_state(self, idx):
        """(active, weight, malformed) of an interned node.  Read the weights of the nodes a change set is about before applying it:
        rebalance_changes takes them as prev_weight (0 for a node that was not live)."""
        a, w, m = C.c_int32(0), C.c_uint32(0), C.c_int32(0)
        self._ck(self.L.rio_cuda_node_state(self.h, idx, C.byref(a), C.byref(w), C.byref(m)))
        return bool(a.value), w.value, bool(m.value)

    # ---- batched directory ------------------------------------------------------------------------------
    def hash_ids(self, ids):
        """ids: iterable of (type, id) -> u64 keys, hashed on the GPU from the packed "{type}.{id}" bytes."""
        joined = [(t + "." + i).encode() for t, i in ids]
        offs = np.zeros(len(joined) + 1, dtype=np.uint64)
        if joined:
            offs[1:] = np.cumsum([len(b) for b in joined])
        packed = np.frombuffer(b"".join(joined) + b"\0" * 16, dtype=np.uint8)
        out = np.empty(len(joined), dtype=np.uint64)
        self._ck(self.L.rio_cuda_hash_ids(self.h, _ptr(packed), _ptr(offs), len(joined), _ptr(out)))
        return out

    def lookup_many(self, keys):
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        out = np.empty(len(keys), dtype=np.uint32)
        self._ck(self.L.rio_cuda_lookup_batch(self.h, _ptr(keys), len(keys), _ptr(out)))
        return out

    def update_many(self, keys, idx):
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        idx = np.ascontiguousarray(idx, dtype=np.uint32)
        assert len(keys) == len(idx)
        self._ck(self.L.rio_cuda_upsert_batch(self.h, _ptr(keys), _ptr(idx), len(keys)))

    def remove_many(self, keys):
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        self._ck(self.L.rio_cuda_remove_batch(self.h, _ptr(keys), len(keys)))

    def clean_node(self, idx):
        r = C.c_uint64(0)
        self._ck(self.L.rio_cuda_clean_node(self.h, idx, C.byref(r)))
        return r.value

    def directory_len(self):
        a, b = C.c_uint64(0), C.c_uint64(0)
        self._ck(self.L.rio_cuda_directory_len(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def load_counters(self):
        total, _ = self.node_count()
        out = np.zeros(max(total, 1), dtype=np.uint32)
        self._ck(self.L.rio_cuda_load_counters(self.h, _ptr(out), len(out)))
        return out[:total]

    # ---- solver ------------------------------------------------------------------------------------------
    def set_solver(self, solver="hrw", trie_bits=0):
        """'hrw' = flat weighted rendezvous (default); 'hrw2' = hierarchical, fan-out 2 (DESIGN.md 3.8)."""
        self._ck(self.L.rio_cuda_set_solver(self.h, N.SOLVER_HRW2 if solver == "hrw2" else N.SOLVER_HRW, trie_bits))

    def get_solver(self):
        a, b = C.c_uint32(0), C.c_uint32(0)
        self._ck(self.L.rio_cuda_get_solver(self.h, C.byref(a), C.byref(b)))
        return ("hrw2" if a.value == N.SOLVER_HRW2 else "hrw"), b.value

    def assign_batch(self, keys=None, obj_feats=None, out=None):
        if obj_feats is not None:
            obj_feats = np.ascontiguousarray(obj_feats, dtype=np.float32)
            n = obj_feats.shape[0]
        if keys is not None:
            keys = np.ascontiguousarray(keys, dtype=np.uint64)
            n = len(keys)
        if out is None:
            out = np.empty(n, dtype=np.uint32)
        self._ck(self.L.rio_cuda_assign_batch(self.h, _ptr(keys), _ptr(obj_feats), n, _ptr(out)))
        return out

    def assign_ranked(self, keys, ranks):
        """Each object's first `ranks` distinct nodes under the handle's policy (DESIGN.md 3.9) -> (n, ranks) uint32: column 0 is
        assign_batch, column 1 the failover target (where a LEAVE of column 0 sends the object); RIO_NONE past the live set."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        out = np.empty((len(keys), ranks), dtype=np.uint32)
        self._ck(self.L.rio_cuda_assign_ranked_batch(self.h, _ptr(keys), len(keys), ranks, _ptr(out)))
        return out

    def set_node_domains(self, idx, domain):
        """Failure-domain labels (DESIGN.md 3.12): node idx[i] gets label domain[i] (a rack or zone id); N.NONE = a domain of its own."""
        idx = np.ascontiguousarray(idx, dtype=np.uint32)
        dom = np.ascontiguousarray(domain, dtype=np.uint32)
        if idx.shape != dom.shape or idx.ndim != 1:
            raise Unknown("idx and domain must be 1-D arrays of one length")
        self._ck(self.L.rio_cuda_node_set_domains(self.h, _ptr(idx), _ptr(dom), len(idx)))

    def node_domain(self, idx):
        d = C.c_uint32(0)
        self._ck(self.L.rio_cuda_node_domain(self.h, idx, C.byref(d)))
        return d.value

    def assign_ranked_spread(self, keys, ranks):
        """Each object's first `ranks` nodes in distinct failure domains (DESIGN.md 3.12) -> (n, ranks) uint32: column 0 is
        assign_batch, column 1 where the object goes when column 0's whole domain leaves; RIO_NONE past the live domain count."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        out = np.empty((len(keys), ranks), dtype=np.uint32)
        self._ck(self.L.rio_cuda_assign_ranked_spread_batch(self.h, _ptr(keys), len(keys), ranks, _ptr(out)))
        return out

    def assign_ranked_affinity(self, obj_feats, ranks):
        """Each object's `ranks` lowest-cost live nodes under the affinity cost (DESIGN.md 3.9) -> (n, ranks) uint32: column 0 is
        assign_batch(obj_feats=...), column 1 where a LEAVE of column 0 sends the object; RIO_NONE past the live set."""
        obj_feats = np.ascontiguousarray(obj_feats, dtype=np.float32)
        n = obj_feats.shape[0]
        out = np.empty((n, ranks), dtype=np.uint32)
        self._ck(self.L.rio_cuda_assign_ranked_affinity_batch(self.h, _ptr(obj_feats), n, ranks, _ptr(out)))
        return out

    def assign_ranked_affinity_spread(self, obj_feats, ranks):
        """Each object's `ranks` lowest-cost live nodes in distinct failure domains under the affinity cost (DESIGN.md 3.14) ->
        (n, ranks) uint32: column 0 is assign_batch(obj_feats=...), column 1 where the object goes when column 0's whole domain
        leaves; RIO_NONE past the live domain count."""
        obj_feats = np.ascontiguousarray(obj_feats, dtype=np.float32)
        n = obj_feats.shape[0]
        out = np.empty((n, ranks), dtype=np.uint32)
        self._ck(self.L.rio_cuda_assign_ranked_affinity_spread_batch(self.h, _ptr(obj_feats), n, ranks, _ptr(out)))
        return out

    def assign_bounded_batch(self, keys, n_total=0, cap_num=5, cap_den=4, max_rounds=4, out=None):
        """assign_batch + bounded-load rounds for host buffers; returns (indices, passes)."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        if out is None:
            out = np.empty(len(keys), dtype=np.uint32)
        passes = C.c_uint32(0)
        self._ck(self.L.rio_cuda_assign_bounded_batch(self.h, _ptr(keys), len(keys), n_total, cap_num, cap_den, max_rounds, _ptr(out), C.byref(passes)))
        return out, passes.value

    def assign_bounded_affinity_batch(self, keys, obj_feats, n_total=0, cap_num=5, cap_den=4, max_rounds=4):
        """assign_batch(obj_feats) + bounded-load rounds (DESIGN.md 3.16) for host buffers: the keys feed the spill hash, the features
        the cost; returns (indices, passes), what ObjectSet.assign_bounded_affinity gives for the same keys and features."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        obj_feats = np.ascontiguousarray(obj_feats, dtype=np.float32)
        assert obj_feats.ndim == 2 and len(obj_feats) == len(keys)
        out = np.empty(len(keys), dtype=np.uint32)
        passes = C.c_uint32(0)
        self._ck(self.L.rio_cuda_assign_bounded_affinity_batch(self.h, _ptr(keys), _ptr(obj_feats), len(keys), n_total, cap_num, cap_den, max_rounds, _ptr(out),
                                                               C.byref(passes)))
        return out, passes.value

    def assign_bounded_weighted_batch(self, keys, weights=None, obj_feats=None, load_total=0, cap_num=5, cap_den=4, max_rounds=4):
        """Bounded-load rounds over object weights (DESIGN.md 3.19) for host buffers: weights (uint32 per key, None = all 1) are the
        loads the capacities bound; obj_feats selects the affinity cost, None the hash policy.  Returns (indices, passes), what
        ObjectSet.assign_bounded_weighted gives for the same rows."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        if weights is not None:
            weights = np.ascontiguousarray(weights, dtype=np.uint32)
            assert len(weights) == len(keys)
        if obj_feats is not None:
            obj_feats = np.ascontiguousarray(obj_feats, dtype=np.float32)
            assert obj_feats.ndim == 2 and len(obj_feats) == len(keys)
        out = np.empty(len(keys), dtype=np.uint32)
        passes = C.c_uint32(0)
        self._ck(self.L.rio_cuda_assign_bounded_weighted_batch(self.h, _ptr(keys), _ptr(obj_feats), _ptr(weights), len(keys), load_total, cap_num, cap_den,
                                                               max_rounds, _ptr(out), C.byref(passes)))
        return out, passes.value

    def place_batch(self, keys, policy="hrw", self_address=None):
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        out = np.empty(len(keys), dtype=np.uint32)
        pol = {"self": N.PLACE_SELF, "hrw": N.PLACE_HRW, "hrw2": N.PLACE_HRW2}[policy]
        self_idx = 0
        if pol == N.PLACE_SELF:
            self_idx = self.node_index(self_address)
            if self_idx is None:
                raise Unknown("self_address is not a known node")
        self._ck(self.L.rio_cuda_place_batch(self.h, _ptr(keys), len(keys), pol, self_idx, _ptr(out)))
        return out

    def check_address_batch(self, addr_idx, self_address):
        """Service::check_address_mismatch for a batch (service.rs:261-298) -> (verdicts u8[n] of N.ADDR_*, entries cleaned)."""
        addr_idx = np.ascontiguousarray(addr_idx, dtype=np.uint32)
        self_idx = self.node_index(self_address)
        if self_idx is None:
            raise Unknown("self_address is not a known node")
        out = np.empty(len(addr_idx), dtype=np.uint8)
        cleaned = C.c_uint64(0)
        self._ck(self.L.rio_cuda_check_address_batch(self.h, _ptr(addr_idx), len(addr_idx), self_idx, _ptr(out), C.byref(cleaned)))
        return out, cleaned.value

    def check_address_mismatch(self, self_address, server_address):
        """Per-request form with the reference's signature: -> N.ADDR_LOCAL (Ok) | ADDR_REDIRECT | ADDR_DEALLOCATE | ADDR_MALFORMED."""
        v, _ = self.check_address_batch([self.node_intern(server_address)], self_address)
        return int(v[0])

    # ---- test hooks (include/rio_cuda_dev.h) ------------------------------------------------------------------
    def dev_set_node_seed(self, idx, seed):
        self._ck(self.L.rio_dev_set_node_seed(self.h, idx, int(seed)))

    def dev_set_table_options(self, flags):
        self._ck(self.L.rio_dev_set_table_options(self.h, flags))

    def rebalance(self, event, idx):
        m = C.c_uint64(0)
        self._ck(self.L.rio_cuda_rebalance(self.h, N.EV_JOIN if event == "join" else N.EV_LEAVE, idx, C.byref(m)))
        return m.value

    def rebalance_changes(self, idx, prev_weight):
        """Eager re-placement of the directory after a set of node changes, in one pass (DESIGN.md 3.10): idx are distinct node
        indices, prev_weight[i] the weight of idx[i] before the change if it was live then, else 0.  Returns the number moved."""
        idx, prev = _change_set(idx, prev_weight)
        m = C.c_uint64(0)
        self._ck(self.L.rio_cuda_rebalance_changes(self.h, _ptr(idx), _ptr(prev), len(idx), C.byref(m)))
        return m.value

    # ---- misc --------------------------------------------------------------------------------------------
    def sync(self):
        self._ck(self.L.rio_cuda_sync(self.h))

    def device_info(self):
        d, s, m = C.c_int32(0), C.c_int32(0), C.c_uint64(0)
        self._ck(self.L.rio_cuda_device_info(self.h, C.byref(d), C.byref(s), C.byref(m), self._buf, 512))
        return {"device": d.value, "sm_count": s.value, "hbm_bytes": m.value, "name": self._buf.value.decode()}

    def launch_count(self):
        v = C.c_uint64(0)
        self._ck(self.L.rio_cuda_launch_count(self.h, C.byref(v)))
        return v.value

    def event_record(self, slot):
        self._ck(self.L.rio_cuda_event_record(self.h, slot))

    def event_elapsed_ms(self, a, b):
        ms = C.c_float(0)
        self._ck(self.L.rio_cuda_event_elapsed_ms(self.h, a, b, C.byref(ms)))
        return ms.value

    def bench_mix_rate(self, iters=2000):
        v = C.c_double(0)
        self._ck(self.L.rio_cuda_bench_mix_rate(self.h, iters, C.byref(v)))
        return v.value

    def flush_l2(self):
        self._ck(self.L.rio_cuda_flush_l2(self.h))

    def comm_init(self, rank, world, unique_id):
        buf = np.frombuffer(bytes(unique_id), dtype=np.uint8).copy()
        self._ck(self.L.rio_cuda_comm_init(self.h, rank, world, _ptr(buf)))

    def comm_ipc_export(self, world, max_nodes=8192):
        buf = np.zeros(64, dtype=np.uint8)
        self._ck(self.L.rio_cuda_comm_ipc_export(self.h, world, max_nodes, _ptr(buf)))
        return buf.tobytes()

    def comm_ipc_attach(self, rank, world, handles):
        buf = np.frombuffer(b"".join(handles), dtype=np.uint8).copy()
        self._ck(self.L.rio_cuda_comm_ipc_attach(self.h, rank, world, _ptr(buf)))

    def comm_sum_counters(self, counters):
        c = np.ascontiguousarray(counters, dtype=np.uint32).copy()
        self._ck(self.L.rio_cuda_comm_sum_counters(self.h, _ptr(c), len(c)))
        return c

    def new_set(self, capacity):
        return ObjectSet(self, capacity)


class Resolver:
    """Micro-batching front end for per-request resolves (Service::get_or_create_placement, service.rs:193-254)."""

    def __init__(self, provider, policy="hrw", self_address=None, max_batch=4096, max_wait_us=50):
        self.p = provider
        self.L = provider.L
        pol = {"self": N.PLACE_SELF, "hrw": N.PLACE_HRW, "hrw2": N.PLACE_HRW2}[policy]
        self_idx = 0
        if pol == N.PLACE_SELF:
            self_idx = provider.node_index(self_address)
            if self_idx is None:
                raise Unknown("self_address is not a known node")
        r = N.H()
        provider._ck(self.L.rio_cuda_resolver_create(provider.h, pol, self_idx, max_batch, max_wait_us, C.byref(r)))
        self.r = r
        self._e = provider._e
        self._e._retain()          # the worker thread calls into the engine until the resolver is destroyed: see _Engine._retain

    def close(self):
        if getattr(self, "r", None):
            self.L.rio_cuda_resolver_destroy(self.r)
            self.r = None
            self._e._release()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def resolve(self, key):
        out = C.c_uint32(0)
        st = self.L.rio_cuda_resolver_resolve(self.r, int(key), C.byref(out))
        if st != N.RIO_OK:
            msg = self.L.rio_cuda_resolver_last_error()
            raise (Upstream if st == N.RIO_ERR_UPSTREAM else Unknown)(msg.decode(errors="replace") if msg else "")
        return out.value

    def get_or_create_placement(self, handler_type, handler_id):
        """Same signature as the reference's per-request function (service.rs:193-197): -> address string."""
        t, i = handler_type.encode(), handler_id.encode()
        return _read_str(lambda buf, cap, n: self._rck(self.L.rio_cuda_resolver_resolve_str(self.r, t, len(t), i, len(i), buf, cap, n)))

    def _rck(self, st):
        if st != N.RIO_OK:
            msg = self.L.rio_cuda_resolver_last_error()
            raise (Upstream if st == N.RIO_ERR_UPSTREAM else Unknown)(msg.decode(errors="replace") if msg else "")

    # the trait's per-id calls, coalesced with every other caller's (mod.rs:46-55)
    def lookup(self, object_id):
        t, i = (s.encode() for s in object_id)
        return _read_str(lambda buf, cap, n: self._rck(self.L.rio_cuda_resolver_lookup_str(self.r, t, len(t), i, len(i), buf, cap, n)))

    def update(self, item):
        t, i = (s.encode() for s in item.object_id)
        a = None if item.server_address is None else item.server_address.encode()
        self._rck(self.L.rio_cuda_resolver_update_str(self.r, t, len(t), i, len(i), a, 0 if a is None else len(a)))

    def remove(self, object_id):
        t, i = (s.encode() for s in object_id)
        self._rck(self.L.rio_cuda_resolver_update_str(self.r, t, len(t), i, len(i), None, 0))

    def lookup_key(self, key):
        out = C.c_uint32(0)
        self._rck(self.L.rio_cuda_resolver_lookup(self.r, int(key), C.byref(out)))
        return out.value

    def stats(self):
        a, b, c = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        self.L.rio_cuda_resolver_stats(self.r, C.byref(a), C.byref(b), C.byref(c))
        return {"calls": a.value, "batches": b.value, "largest_batch": c.value}


def comm_unique_id():
    buf = np.zeros(N.COMM_ID_BYTES, dtype=np.uint8)
    L = N.lib()
    st = L.rio_cuda_comm_unique_id(_ptr(buf))
    _check(L, None, st)
    return buf.tobytes()


class ObjectSet:
    """A resident id-range shard: dense keys + assignment in HBM (configs C4/C5)."""

    def __init__(self, provider, capacity):
        self.p = provider
        self.L = provider.L
        s = N.H()
        provider._ck(self.L.rio_cuda_set_create(provider.h, capacity, C.byref(s)))
        self.s = s
        self._e = provider._e
        self._e._retain()          # the set points into the engine: see _Engine._retain

    def __del__(self):
        try:
            if getattr(self, "s", None):
                self.L.rio_cuda_set_destroy(self.s)
                self.s = None
                self._e._release()
        except Exception:
            pass

    def _ck(self, st):
        _check(self.L, self.p.h, st)

    def load_keys(self, keys):
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        self._ck(self.L.rio_cuda_set_load_keys(self.s, _ptr(keys), len(keys)))

    def synth_keys(self, first, n, seed):
        self._ck(self.L.rio_cuda_set_synth_keys(self.s, first, n, seed))

    def load_feats(self, feats):
        feats = np.ascontiguousarray(feats, dtype=np.float32)
        self._ck(self.L.rio_cuda_set_load_feats(self.s, _ptr(feats), feats.shape[1]))

    def assign(self, use_affinity=False):
        self._ck(self.L.rio_cuda_set_assign(self.s, int(use_affinity)))

    def assign_bounded(self, n_total=0, cap_num=5, cap_den=4, max_rounds=4):
        passes = C.c_uint32(0)
        self._ck(self.L.rio_cuda_set_assign_bounded(self.s, n_total, cap_num, cap_den, max_rounds, C.byref(passes)))
        return passes.value

    def assign_bounded_affinity(self, n_total=0, cap_num=5, cap_den=4, max_rounds=4):
        """Bounded-load rounds under the affinity cost of the set's features (load_feats; DESIGN.md 3.16); returns the passes run."""
        passes = C.c_uint32(0)
        self._ck(self.L.rio_cuda_set_assign_bounded_affinity(self.s, n_total, cap_num, cap_den, max_rounds, C.byref(passes)))
        return passes.value

    def rebalance_changes_bounded_affinity(self, idx, prev_weight, n_total=0, cap_num=5, cap_den=4, max_rounds=4):
        """Keeps the assignment of assign_bounded_affinity within capacity after a change set (DESIGN.md 3.17): one change-set pass,
        then the capacity rounds from the current assignment.  Returns (moved, passes): objects whose node changed, and 1 + the rounds
        run.  Calls that drop ranked lists, and load_feats, end the set's record; the call then refuses until the next
        assign_bounded_affinity."""
        idx, prev = _change_set(idx, prev_weight)
        m, passes = C.c_uint64(0), C.c_uint32(0)
        self._ck(self.L.rio_cuda_set_rebalance_changes_bounded_affinity(self.s, _ptr(idx), _ptr(prev), len(idx), n_total, cap_num, cap_den, max_rounds,
                                                                        C.byref(m), C.byref(passes)))
        return m.value, passes.value

    def insert(self, keys, feats=None):
        """Appends the objects as rows [n, n + len(keys)) and places them as the set's current kind places a fresh object (DESIGN.md
        3.18); feats (len(keys) x K) exactly when the set has features.  No existing row changes.  Returns the first new row."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        if feats is not None:
            feats = np.ascontiguousarray(feats, dtype=np.float32)
        first = C.c_uint64(0)
        self._ck(self.L.rio_cuda_set_insert(self.s, _ptr(keys), _ptr(feats), len(keys), C.byref(first)))
        return first.value

    def erase(self, keys):
        """Removes every row whose key is one of `keys` (DESIGN.md 3.18): the surviving rows past the new end fill the holes, in order;
        no remaining object changes node or list.  Returns the number of rows removed."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        erased = C.c_uint64(0)
        self._ck(self.L.rio_cuda_set_erase(self.s, _ptr(keys), len(keys), C.byref(erased)))
        return erased.value

    def write_weights(self, w, first=0):
        """Writes the weights of rows [first, first + len(w)) (DESIGN.md 3.19); every other row keeps its weight (1 unless written)."""
        w = np.ascontiguousarray(w, dtype=np.uint32)
        self._ck(self.L.rio_cuda_set_write_weights(self.s, first, len(w), _ptr(w)))

    def read_weights(self, first=0, n=None):
        """The weights of rows [first, first + n) -> uint32."""
        if n is None:
            n = self.size() - first
        out = np.empty(max(n, 0), dtype=np.uint32)
        self._ck(self.L.rio_cuda_set_read_weights(self.s, first, n, _ptr(out)))
        return out

    def write_weights_by_key(self, keys, w):
        """Writes weight w[j] into every row whose key is keys[j] (DESIGN.md 3.21): the last occurrence of a repeated key wins, absent
        keys are ignored.  Returns the rows written."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        w = np.ascontiguousarray(w, dtype=np.uint32)
        assert len(keys) == len(w)
        out = C.c_uint64(0)
        self._ck(self.L.rio_cuda_set_write_weights_by_key(self.s, _ptr(keys), _ptr(w), len(keys), C.byref(out)))
        return out.value

    def rebalance_changes_bounded_weighted(self, idx, prev_weight, load_total=0, cap_num=5, cap_den=4, max_rounds=4):
        """Keeps the assignment of assign_bounded_weighted within its load capacities after a change set, weight writes or churn
        (DESIGN.md 3.21): one change-set pass of the recorded kind, then the weighted capacity rounds from the current assignment.
        Returns (moved, passes): objects whose node changed, and 1 + the rounds run."""
        idx, prev = _change_set(idx, prev_weight)
        m, passes = C.c_uint64(0), C.c_uint32(0)
        self._ck(self.L.rio_cuda_set_rebalance_changes_bounded_weighted(self.s, _ptr(idx), _ptr(prev), len(idx), load_total, cap_num, cap_den, max_rounds,
                                                                        C.byref(m), C.byref(passes)))
        return m.value, passes.value

    def loads(self):
        """Global per-node sums of the object weights of the current assignment (collective across ranks, as counters())."""
        total, _ = self.p.node_count()
        out = np.zeros(max(total, 1), dtype=np.uint32)
        self._ck(self.L.rio_cuda_set_loads(self.s, _ptr(out), len(out)))
        return out[:total]

    def assign_bounded_weighted(self, use_affinity=False, load_total=0, cap_num=5, cap_den=4, max_rounds=4):
        """Bounded-load rounds over the set's object weights (DESIGN.md 3.19): the capacities bound each node's load, the sum of its
        objects' weights, under the hash policy or (use_affinity) the affinity cost of the set's features.  load_total 0 = the weight
        sum of every rank's shard (reduced across ranks); an explicit load_total must be the same on every rank.  The counters stay object counts; loads() gives the loads.  Returns the passes run."""
        passes = C.c_uint32(0)
        self._ck(self.L.rio_cuda_set_assign_bounded_weighted(self.s, int(use_affinity), load_total, cap_num, cap_den, max_rounds, C.byref(passes)))
        return passes.value

    def assign_bounded_begin(self, n_total=0, cap_num=5, cap_den=4, max_rounds=4):
        self._ck(self.L.rio_cuda_set_assign_bounded_begin(self.s, n_total, cap_num, cap_den, max_rounds))

    def assign_bounded_end(self):
        passes = C.c_uint32(0)
        self._ck(self.L.rio_cuda_set_assign_bounded_end(self.s, C.byref(passes)))
        return passes.value

    def rebalance(self, event, idx):
        m = C.c_uint64(0)
        self._ck(self.L.rio_cuda_set_rebalance(self.s, N.EV_JOIN if event == "join" else N.EV_LEAVE, idx, C.byref(m)))
        return m.value

    def rebalance_changes(self, idx, prev_weight):
        """GpuObjectPlacement.rebalance_changes for this set (plain policy); the counters stay exact."""
        idx, prev = _change_set(idx, prev_weight)
        m = C.c_uint64(0)
        self._ck(self.L.rio_cuda_set_rebalance_changes(self.s, _ptr(idx), _ptr(prev), len(idx), C.byref(m)))
        return m.value

    def assign_ranked(self, ranks):
        """Each key's first `ranks` nodes under the handle's policy, kept in the set (DESIGN.md 3.11): column 0 becomes the set's
        assignment (read, counters, commit), the other columns are its standbys.  Calls that assign the set otherwise drop the lists."""
        self._ck(self.L.rio_cuda_set_assign_ranked(self.s, ranks))
        self._ranks = int(ranks)

    def assign_ranked_spread(self, ranks):
        """Each key's first `ranks` nodes in distinct failure domains, kept in the set (DESIGN.md 3.13), with the labels they were
        computed under.  read_ranked reads them and rebalance_changes_ranked keeps them current, relabels since the last call included."""
        self._ck(self.L.rio_cuda_set_assign_ranked_spread(self.s, ranks))
        self._ranks = int(ranks)

    def assign_ranked_affinity(self, ranks):
        """Each object's `ranks` lowest-cost nodes under the affinity cost of the set's features (load_feats), kept in the set
        (DESIGN.md 3.15) with the path, K and node features they were computed under.  rebalance_changes_ranked keeps them current,
        node feature changes since the last call included; load_feats drops them."""
        self._ck(self.L.rio_cuda_set_assign_ranked_affinity(self.s, ranks))
        self._ranks = int(ranks)

    def assign_ranked_affinity_spread(self, ranks):
        """assign_ranked_affinity with each object's `ranks` lowest-cost nodes in distinct failure domains (DESIGN.md 3.15); the labels
        are recorded too, and relabels since the last call belong to the next change set."""
        self._ck(self.L.rio_cuda_set_assign_ranked_affinity_spread(self.s, ranks))
        self._ranks = int(ranks)

    def read_ranked(self, first=0, n=None):
        """Rows [first, first + n) of the ranked lists -> (n, ranks) uint32, RIO_NONE past the live set."""
        if n is None:
            n = self.size() - first
        out = np.empty((max(n, 0), getattr(self, "_ranks", 1)), dtype=np.uint32)
        self._ck(self.L.rio_cuda_set_read_ranked(self.s, first, n, _ptr(out)))
        return out

    def rebalance_changes_ranked(self, idx, prev_weight):
        """rebalance_changes for a set holding ranked lists: every list stays equal to the fresh one over the live set.  Returns
        (moved, changed): objects whose rank 1 changed, and objects whose list changed at any rank."""
        idx, prev = _change_set(idx, prev_weight)
        m, c = C.c_uint64(0), C.c_uint64(0)
        self._ck(self.L.rio_cuda_set_rebalance_changes_ranked(self.s, _ptr(idx), _ptr(prev), len(idx), C.byref(m), C.byref(c)))
        return m.value, c.value

    def counters(self):
        total, _ = self.p.node_count()
        out = np.zeros(max(total, 1), dtype=np.uint32)
        self._ck(self.L.rio_cuda_set_counters(self.s, _ptr(out), len(out)))
        return out[:total]

    def size(self):
        n = C.c_uint64(0)
        self._ck(self.L.rio_cuda_set_size(self.s, C.byref(n)))
        return n.value

    def read(self, first=0, n=None, want_keys=False):
        if n is None:
            n = self.size() - first
        idx = np.empty(n, dtype=np.uint32)
        keys = np.empty(n, dtype=np.uint64) if want_keys else None
        self._ck(self.L.rio_cuda_set_read(self.s, first, n, _ptr(keys), _ptr(idx)))
        return (keys, idx) if want_keys else idx

    def commit(self):
        self._ck(self.L.rio_cuda_set_commit(self.s))

    def commit_changes(self, dry_run=False, cap=None):
        """Writes into the directory only the rows whose node differs from what the directory answers for their key (DESIGN.md 3.20)
        and returns those moves as numpy arrays (rows, keys, from_, to), in row order; from_ is the directory's answer before the call
        (RIO_NONE: absent), to the set's node (RIO_NONE: the key is removed).  dry_run computes the same manifest and leaves the
        directory as it was.  cap=None asks for the count first, then calls again with buffers of that size."""
        n = C.c_uint64(0)
        if cap is None:
            self._ck(self.L.rio_cuda_set_commit_changes(self.s, 1, 0, None, None, None, None, C.byref(n)))
            cap = n.value
        rows, keys = np.empty(cap, np.uint64), np.empty(cap, np.uint64)
        from_, to = np.empty(cap, np.uint32), np.empty(cap, np.uint32)
        self._ck(self.L.rio_cuda_set_commit_changes(self.s, int(bool(dry_run)), cap, _ptr(rows), _ptr(keys), _ptr(from_), _ptr(to), C.byref(n)))
        m = n.value
        return rows[:m], keys[:m], from_[:m], to[:m]

//! `GpuObjectPlacement` — implements `rio_rs::object_placement::ObjectPlacement`
//! (rio-rs/src/object_placement/mod.rs:38-56) on top of librio_cuda, so `Server::builder()
//! .object_placement_provider(GpuObjectPlacement::new(..)?)` (rio-rs/src/server.rs:103-104) works unchanged.
//!
//! NOT COMPILED in the authoring image (no cargo/rustc); see rust/README.md.
use std::ffi::CStr;
use std::ptr;
use std::sync::Arc;

use async_trait::async_trait;
use rio_cuda_sys as sys;
use rio_rs::errors::ObjectPlacementError;
use rio_rs::object_placement::{ObjectPlacement, ObjectPlacementItem};
use rio_rs::ObjectId;

/// Owns the engine handle; dropped (rio_cuda_destroy) when the last provider clone goes away.
struct Engine(*mut sys::rio_placement);
// The C library is internally synchronised per handle (include/rio_cuda.h "Conventions").
unsafe impl Send for Engine {}
unsafe impl Sync for Engine {}
impl Drop for Engine {
    fn drop(&mut self) {
        unsafe { sys::rio_cuda_destroy(self.0) }
    }
}

/// Cheap to clone; clones share state like `LocalObjectPlacement` (local.rs:12-18, test local.rs:75-114).
#[derive(Clone)]
pub struct GpuObjectPlacement {
    engine: Arc<Engine>,
}

impl std::fmt::Debug for GpuObjectPlacement {
    fn fmt(&self, f: &mut std::fmt::Formatter<'_>) -> std::fmt::Result {
        f.debug_struct("GpuObjectPlacement").finish()
    }
}

fn check(h: *mut sys::rio_placement, st: sys::rio_status) -> Result<(), ObjectPlacementError> {
    if st == sys::RIO_OK {
        return Ok(());
    }
    let msg = unsafe {
        let p = sys::rio_cuda_last_error(h);
        if p.is_null() { String::new() } else { CStr::from_ptr(p).to_string_lossy().into_owned() }
    };
    Err(if st == sys::RIO_ERR_UPSTREAM { ObjectPlacementError::Upstream(msg) } else { ObjectPlacementError::Unknown(msg) })
}

/// What `place_batch` / the resolver do with an id that has no (live) placement: the reference's "the server that saw the
/// request claims it" (service.rs:244-252), or one of the two rendezvous solvers.
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum PlacePolicy {
    SelfNode(u32),
    Hrw,
    Hrw2,
}
impl PlacePolicy {
    fn raw(self) -> (u32, u32) {
        match self {
            PlacePolicy::SelfNode(i) => (sys::RIO_PLACE_SELF, i),
            PlacePolicy::Hrw => (sys::RIO_PLACE_HRW, 0),
            PlacePolicy::Hrw2 => (sys::RIO_PLACE_HRW2, 0),
        }
    }
}

/// Reads a string result of the C ABI (`buf, cap, out_len` convention; `out_len == usize::MAX` is `None`), growing the buffer
/// when the first call reports a longer string than it was given room for.
fn read_string(mut call: impl FnMut(*mut libc::c_char, libc::size_t, *mut libc::size_t) -> Result<(), ObjectPlacementError>) -> Result<Option<String>, ObjectPlacementError> {
    let mut buf = vec![0u8; 256];
    loop {
        let mut len: libc::size_t = 0;
        call(buf.as_mut_ptr() as *mut _, buf.len(), &mut len)?;
        if len == usize::MAX {
            return Ok(None);
        }
        if len <= buf.len() {
            buf.truncate(len);
            return Ok(Some(String::from_utf8_lossy(&buf).into_owned()));
        }
        buf = vec![0u8; len];
    }
}

impl GpuObjectPlacement {
    pub fn new(device: i32) -> Result<Self, ObjectPlacementError> {
        let cfg = sys::rio_config { struct_size: std::mem::size_of::<sys::rio_config>() as u32, device, ..Default::default() };
        let mut h = ptr::null_mut();
        check(ptr::null_mut(), unsafe { sys::rio_cuda_create(&cfg, &mut h) })?;
        Ok(Self { engine: Arc::new(Engine(h)) })
    }
    fn h(&self) -> *mut sys::rio_placement {
        self.engine.0
    }

    /// The live node set as seen by MembershipStorage::active_members (storage/mod.rs:95-99).
    pub fn set_nodes(&self, addresses: &[String], weights: Option<&[u32]>) -> Result<Vec<u32>, ObjectPlacementError> {
        let c: Vec<std::ffi::CString> = addresses.iter().map(|a| std::ffi::CString::new(a.as_str()).unwrap()).collect();
        let p: Vec<*const libc::c_char> = c.iter().map(|s| s.as_ptr()).collect();
        let mut out = vec![0u32; addresses.len()];
        check(self.h(), unsafe {
            sys::rio_cuda_set_nodes(self.h(), p.as_ptr(), weights.map_or(ptr::null(), |w| w.as_ptr()), ptr::null(), p.len() as u32, 0, out.as_mut_ptr())
        })?;
        Ok(out)
    }

    /// Batched resolve: Service::get_or_create_placement (service.rs:193-254) for many ids in one launch.
    /// `self_idx = Some(i)` is the reference's rule (claim for the serving node), `None` the flat rendezvous solver.
    pub fn place_batch(&self, keys: &[u64], self_idx: Option<u32>) -> Result<Vec<u32>, ObjectPlacementError> {
        self.place_batch_with(keys, self_idx.map_or(PlacePolicy::Hrw, PlacePolicy::SelfNode))
    }
    /// The same call with the rule for unplaced ids spelled out (`PlacePolicy::Hrw2` = the hierarchical solver, DESIGN.md 3.8).
    pub fn place_batch_with(&self, keys: &[u64], policy: PlacePolicy) -> Result<Vec<u32>, ObjectPlacementError> {
        let mut out = vec![sys::RIO_NONE; keys.len()];
        let (policy, me) = policy.raw();
        check(self.h(), unsafe { sys::rio_cuda_place_batch(self.h(), keys.as_ptr(), keys.len(), policy, me, out.as_mut_ptr()) })?;
        Ok(out)
    }
    /// Address of an interned node, whatever its length (two calls: the length, then the bytes).
    pub fn node_address(&self, idx: u32) -> Result<String, ObjectPlacementError> {
        let mut len: libc::size_t = 0;
        check(self.h(), unsafe { sys::rio_cuda_node_address(self.h(), idx, ptr::null_mut(), 0, &mut len) })?;
        let mut buf = vec![0u8; len];
        check(self.h(), unsafe { sys::rio_cuda_node_address(self.h(), idx, buf.as_mut_ptr() as *mut _, buf.len(), &mut len) })?;
        Ok(String::from_utf8_lossy(&buf).into_owned())
    }
    pub fn lookup_many(&self, keys: &[u64]) -> Result<Vec<u32>, ObjectPlacementError> {
        let mut out = vec![sys::RIO_NONE; keys.len()];
        check(self.h(), unsafe { sys::rio_cuda_lookup_batch(self.h(), keys.as_ptr(), keys.len(), out.as_mut_ptr()) })?;
        Ok(out)
    }
    pub fn update_many(&self, keys: &[u64], idx: &[u32]) -> Result<(), ObjectPlacementError> {
        assert_eq!(keys.len(), idx.len());
        check(self.h(), unsafe { sys::rio_cuda_upsert_batch(self.h(), keys.as_ptr(), idx.as_ptr(), keys.len()) })
    }
    pub fn assign_batch(&self, keys: &[u64]) -> Result<Vec<u32>, ObjectPlacementError> {
        let mut out = vec![sys::RIO_NONE; keys.len()];
        check(self.h(), unsafe { sys::rio_cuda_assign_batch(self.h(), keys.as_ptr(), ptr::null(), keys.len(), out.as_mut_ptr()) })?;
        Ok(out)
    }
    /// Each object's first `ranks` distinct nodes under the handle's policy (DESIGN.md 3.9), row-major: object i's list is
    /// `out[i * ranks..(i + 1) * ranks]`.  Rank 2 is the failover target: where a leave of rank 1 sends the object.
    pub fn assign_ranked(&self, keys: &[u64], ranks: u32) -> Result<Vec<u32>, ObjectPlacementError> {
        let len = keys.len().checked_mul(ranks as usize).ok_or_else(|| ObjectPlacementError::Unknown("n x ranks overflows".into()))?;
        let mut out = vec![sys::RIO_NONE; len];
        check(self.h(), unsafe { sys::rio_cuda_assign_ranked_batch(self.h(), keys.as_ptr(), keys.len(), ranks, out.as_mut_ptr()) })?;
        Ok(out)
    }
    /// Each object's first `ranks` nodes in distinct failure domains (DESIGN.md 3.12), row-major as for `assign_ranked`.  Rank 2
    /// is where the object goes when rank 1's whole domain leaves; entries past the number of live domains are `RIO_NONE`.
    pub fn assign_ranked_spread(&self, keys: &[u64], ranks: u32) -> Result<Vec<u32>, ObjectPlacementError> {
        let len = keys.len().checked_mul(ranks as usize).ok_or_else(|| ObjectPlacementError::Unknown("n x ranks overflows".into()))?;
        let mut out = vec![sys::RIO_NONE; len];
        check(self.h(), unsafe { sys::rio_cuda_assign_ranked_spread_batch(self.h(), keys.as_ptr(), keys.len(), ranks, out.as_mut_ptr()) })?;
        Ok(out)
    }
    /// Failure-domain labels (DESIGN.md 3.12): node `idx[i]` gets `domain[i]`, a rack or zone id; `RIO_NONE` is a domain of its own.
    pub fn set_node_domains(&self, idx: &[u32], domain: &[u32]) -> Result<(), ObjectPlacementError> {
        if idx.len() != domain.len() {
            return Err(ObjectPlacementError::Unknown("idx and domain differ in length".into()));
        }
        check(self.h(), unsafe { sys::rio_cuda_node_set_domains(self.h(), idx.as_ptr(), domain.as_ptr(), idx.len()) })
    }
    /// The failure-domain label of an interned node (`RIO_NONE` if none was set).
    pub fn node_domain(&self, idx: u32) -> Result<u32, ObjectPlacementError> {
        let mut d = sys::RIO_NONE;
        check(self.h(), unsafe { sys::rio_cuda_node_domain(self.h(), idx, &mut d) })?;
        Ok(d)
    }
    /// Each object's `ranks` lowest-cost live nodes under the affinity cost (DESIGN.md 3.9).  `obj_feats` is `n x K` row-major
    /// (K of set_nodes); the result is row-major as for `assign_ranked`, and rank 1 is `assign_batch` with the same features.
    pub fn assign_ranked_affinity(&self, obj_feats: &[f32], n: usize, ranks: u32) -> Result<Vec<u32>, ObjectPlacementError> {
        if n != 0 && obj_feats.len() % n != 0 {
            return Err(ObjectPlacementError::Unknown("obj_feats is not n x K".into()));
        }
        let len = n.checked_mul(ranks as usize).ok_or_else(|| ObjectPlacementError::Unknown("n x ranks overflows".into()))?;
        let mut out = vec![sys::RIO_NONE; len];
        check(self.h(), unsafe { sys::rio_cuda_assign_ranked_affinity_batch(self.h(), obj_feats.as_ptr(), n, ranks, out.as_mut_ptr()) })?;
        Ok(out)
    }
    /// Each object's `ranks` lowest-cost live nodes in distinct failure domains under the affinity cost (DESIGN.md 3.14).  Arguments
    /// and result as for `assign_ranked_affinity`; rank 2 is where the object goes when rank 1's whole domain leaves.
    pub fn assign_ranked_affinity_spread(&self, obj_feats: &[f32], n: usize, ranks: u32) -> Result<Vec<u32>, ObjectPlacementError> {
        if n != 0 && obj_feats.len() % n != 0 {
            return Err(ObjectPlacementError::Unknown("obj_feats is not n x K".into()));
        }
        let len = n.checked_mul(ranks as usize).ok_or_else(|| ObjectPlacementError::Unknown("n x ranks overflows".into()))?;
        let mut out = vec![sys::RIO_NONE; len];
        check(self.h(), unsafe { sys::rio_cuda_assign_ranked_affinity_spread_batch(self.h(), obj_feats.as_ptr(), n, ranks, out.as_mut_ptr()) })?;
        Ok(out)
    }
    /// Eager re-placement after a membership event (beside peer_to_peer.rs:170-191).
    pub fn rebalance(&self, join: bool, node_idx: u32) -> Result<u64, ObjectPlacementError> {
        let mut moved = 0u64;
        check(self.h(), unsafe { sys::rio_cuda_rebalance(self.h(), if join { sys::RIO_EV_JOIN } else { sys::RIO_EV_LEAVE }, node_idx, &mut moved) })?;
        Ok(moved)
    }
    /// Eager re-placement after a set of node changes, in one pass (DESIGN.md 3.10): each change is (node index, its weight before
    /// the change if it was live then, else 0), read with `rio_cuda_node_state` before the changes were applied.
    pub fn rebalance_changes(&self, changes: &[(u32 /*idx*/, u32 /*prev_weight*/)]) -> Result<u64, ObjectPlacementError> {
        let idx: Vec<u32> = changes.iter().map(|c| c.0).collect();
        let prev: Vec<u32> = changes.iter().map(|c| c.1).collect();
        let mut moved = 0u64;
        check(self.h(), unsafe { sys::rio_cuda_rebalance_changes(self.h(), idx.as_ptr(), prev.as_ptr(), idx.len(), &mut moved) })?;
        Ok(moved)
    }
    /// Solver policy of the handle: `hierarchical = false` is the flat weighted rendezvous (minimal movement, M pair hashes per
    /// object), `true` is HRW2 (DESIGN.md 3.8: ~log2 M contests per object, ~(1 + log2(M)/2)x the minimal movement).
    pub fn set_solver(&self, hierarchical: bool, trie_bits: u32) -> Result<(), ObjectPlacementError> {
        check(self.h(), unsafe { sys::rio_cuda_set_solver(self.h(), if hierarchical { sys::RIO_SOLVER_HRW2 } else { sys::RIO_SOLVER_HRW }, trie_bits) })
    }
    /// Service::check_address_mismatch (service.rs:261-298) for the owners a batched resolve returned: per entry
    /// 0 = Ok(()), 1 = Err(Redirect(address)), 2 = clean_server applied + Err(DeallocateServiceObject), 3 = Err(Unknown(malformed)).
    pub fn check_address_batch(&self, owner_idx: &[u32], self_idx: u32) -> Result<Vec<u8>, ObjectPlacementError> {
        let mut out = vec![0u8; owner_idx.len()];
        check(self.h(), unsafe { sys::rio_cuda_check_address_batch(self.h(), owner_idx.as_ptr(), owner_idx.len(), self_idx, out.as_mut_ptr(), ptr::null_mut()) })?;
        Ok(out)
    }
    /// assign_batch followed by the bounded-load rounds (capacity = cap_num/cap_den x fair share); returns (indices, passes).
    pub fn assign_bounded_batch(&self, keys: &[u64], cap_num: u32, cap_den: u32, max_rounds: u32) -> Result<(Vec<u32>, u32), ObjectPlacementError> {
        let mut out = vec![sys::RIO_NONE; keys.len()];
        let mut passes = 0u32;
        check(self.h(), unsafe { sys::rio_cuda_assign_bounded_batch(self.h(), keys.as_ptr(), keys.len(), 0, cap_num, cap_den, max_rounds, out.as_mut_ptr(), &mut passes) })?;
        Ok((out, passes))
    }
    pub fn object_key(id: &ObjectId) -> u64 {
        unsafe { sys::rio_cuda_object_key(id.0.as_ptr() as *const _, id.0.len(), id.1.as_ptr() as *const _, id.1.len()) }
    }
}

/// Micro-batching front end (rio_cuda_resolver_*): a blocking per-id call with the signature of
/// `Service::get_or_create_placement` (service.rs:193-197); concurrent callers are coalesced into one `place_batch`.
pub struct Resolver {
    raw: *mut sys::rio_resolver,
    _engine: Arc<Engine>, // keeps the engine alive for as long as the resolver exists
}
unsafe impl Send for Resolver {}
unsafe impl Sync for Resolver {}
impl Drop for Resolver {
    fn drop(&mut self) {
        unsafe { sys::rio_cuda_resolver_destroy(self.raw) }
    }
}
impl GpuObjectPlacement {
    /// `self_idx = Some(i)`: the reference's rule (claim for the serving node, service.rs:244-252); `None`: rendezvous solver.
    pub fn resolver(&self, self_idx: Option<u32>, max_batch: u32, max_wait_us: u32) -> Result<Resolver, ObjectPlacementError> {
        self.resolver_with(self_idx.map_or(PlacePolicy::Hrw, PlacePolicy::SelfNode), max_batch, max_wait_us)
    }
    pub fn resolver_with(&self, policy: PlacePolicy, max_batch: u32, max_wait_us: u32) -> Result<Resolver, ObjectPlacementError> {
        let (policy, me) = policy.raw();
        let mut raw = ptr::null_mut();
        check(self.h(), unsafe { sys::rio_cuda_resolver_create(self.h(), policy, me, max_batch, max_wait_us, &mut raw) })?;
        Ok(Resolver { raw, _engine: self.engine.clone() })
    }
}
impl Resolver {
    /// ObjectPlacement::lookup per id through the coalescing queue (mod.rs:51): node index or RIO_NONE.
    pub fn lookup_key(&self, key: u64) -> Result<u32, ObjectPlacementError> {
        let mut idx = sys::RIO_NONE;
        let st = unsafe { sys::rio_cuda_resolver_lookup(self.raw, key, &mut idx) };
        if st != sys::RIO_OK {
            let msg = unsafe { CStr::from_ptr(sys::rio_cuda_resolver_last_error()).to_string_lossy().into_owned() };
            return Err(if st == sys::RIO_ERR_UPSTREAM { ObjectPlacementError::Upstream(msg) } else { ObjectPlacementError::Unknown(msg) });
        }
        Ok(idx)
    }
    /// ObjectPlacement::update / remove per id through the coalescing queue (mod.rs:46-49, :55): `idx = RIO_NONE` removes.
    pub fn update_key(&self, key: u64, idx: u32) -> Result<(), ObjectPlacementError> {
        let st = unsafe { sys::rio_cuda_resolver_update(self.raw, key, idx) };
        if st != sys::RIO_OK {
            let msg = unsafe { CStr::from_ptr(sys::rio_cuda_resolver_last_error()).to_string_lossy().into_owned() };
            return Err(if st == sys::RIO_ERR_UPSTREAM { ObjectPlacementError::Upstream(msg) } else { ObjectPlacementError::Unknown(msg) });
        }
        Ok(())
    }
    /// Blocking; call it from `spawn_blocking` or a dedicated thread.
    pub fn get_or_create_placement(&self, handler_type: &str, handler_id: &str) -> Result<Option<String>, ObjectPlacementError> {
        // an address longer than the first buffer is read again from the directory (the placement exists by then)
        read_string(|buf, cap, len| {
            let st = unsafe {
                sys::rio_cuda_resolver_resolve_str(self.raw, handler_type.as_ptr() as *const _, handler_type.len(), handler_id.as_ptr() as *const _,
                                                   handler_id.len(), buf, cap, len)
            };
            if st != sys::RIO_OK {
                let msg = unsafe { CStr::from_ptr(sys::rio_cuda_resolver_last_error()).to_string_lossy().into_owned() };
                return Err(if st == sys::RIO_ERR_UPSTREAM { ObjectPlacementError::Upstream(msg) } else { ObjectPlacementError::Unknown(msg) });
            }
            Ok(())
        })
    }
}

/// FFI calls block for tens of microseconds: keep them off the async workers (SURVEY section 7 hard part 5).
async fn blocking<T: Send + 'static>(f: impl FnOnce() -> Result<T, ObjectPlacementError> + Send + 'static) -> Result<T, ObjectPlacementError> {
    tokio::task::spawn_blocking(f).await.map_err(|e| ObjectPlacementError::Unknown(e.to_string()))?
}

#[async_trait]
impl ObjectPlacement for GpuObjectPlacement {
    // prepare(): default Ok(()) (mod.rs:41-43); the engine was created in new().

    async fn update(&self, item: ObjectPlacementItem) -> Result<(), ObjectPlacementError> {
        let this = self.clone();
        blocking(move || {
            let (t, i) = (&item.object_id.0, &item.object_id.1);
            let (ap, al) = match &item.server_address { Some(a) => (a.as_ptr() as *const libc::c_char, a.len()), None => (ptr::null(), 0) };
            check(this.h(), unsafe { sys::rio_cuda_update_str(this.h(), t.as_ptr() as *const _, t.len(), i.as_ptr() as *const _, i.len(), ap, al) })
        })
        .await
    }

    async fn lookup(&self, object_id: &ObjectId) -> Result<Option<String>, ObjectPlacementError> {
        let this = self.clone();
        let (t, i) = (object_id.0.clone(), object_id.1.clone());
        blocking(move || {
            // a missing id is Ok(None), not an error (tests/object_placement_backend.rs:14-15)
            read_string(|buf, cap, len| {
                check(this.h(), unsafe { sys::rio_cuda_lookup_str(this.h(), t.as_ptr() as *const _, t.len(), i.as_ptr() as *const _, i.len(), buf, cap, len) })
            })
        })
        .await
    }

    async fn clean_server(&self, address: String) -> Result<(), ObjectPlacementError> {
        let this = self.clone();
        blocking(move || check(this.h(), unsafe { sys::rio_cuda_clean_server_str(this.h(), address.as_ptr() as *const _, address.len()) })).await
    }

    async fn remove(&self, object_id: &ObjectId) -> Result<(), ObjectPlacementError> {
        let this = self.clone();
        let (t, i) = (object_id.0.clone(), object_id.1.clone());
        blocking(move || check(this.h(), unsafe { sys::rio_cuda_remove_str(this.h(), t.as_ptr() as *const _, t.len(), i.as_ptr() as *const _, i.len()) })).await
    }
}

/// The durable flavour (SqliteObjectPlacement, rio-rs/src/object_placement/sqlite.rs:58-126): every mutation executes the
/// reference's own SQL against the reference's schema (migrations/0001-sqlite-init.sql:1-9) and the matching GPU mutation
/// (rio_cuda_durable_*, csrc/durable.cu); lookups are answered by the GPU directory; `recover()` rebuilds it after a restart.
struct DurableHandle {
    raw: *mut sys::rio_durable,
    _engine: Arc<Engine>, // the table handle must not outlive the engine it writes through to
}
unsafe impl Send for DurableHandle {}
unsafe impl Sync for DurableHandle {}
impl Drop for DurableHandle {
    fn drop(&mut self) {
        unsafe { sys::rio_cuda_durable_close(self.raw) }
    }
}

#[derive(Clone)]
pub struct DurableGpuObjectPlacement {
    gpu: GpuObjectPlacement,
    db: Arc<DurableHandle>,
}
impl std::fmt::Debug for DurableGpuObjectPlacement {
    fn fmt(&self, f: &mut std::fmt::Formatter<'_>) -> std::fmt::Result {
        f.debug_struct("DurableGpuObjectPlacement").finish()
    }
}

fn check_durable(st: sys::rio_status) -> Result<(), ObjectPlacementError> {
    if st == sys::RIO_OK {
        return Ok(());
    }
    // SQL failures surface as Upstream, like `From<sqlx::Error>` (errors.rs:145-152)
    let msg = unsafe { CStr::from_ptr(sys::rio_cuda_durable_last_error()).to_string_lossy().into_owned() };
    Err(if st == sys::RIO_ERR_UPSTREAM { ObjectPlacementError::Upstream(msg) } else { ObjectPlacementError::Unknown(msg) })
}

impl DurableGpuObjectPlacement {
    /// `path` as SqliteObjectPlacement takes it (a file, or ":memory:"); runs the migration like `prepare()` (sqlite.rs:58-66).
    pub fn open(gpu: GpuObjectPlacement, path: &str) -> Result<Self, ObjectPlacementError> {
        let c = std::ffi::CString::new(path).map_err(|e| ObjectPlacementError::Unknown(e.to_string()))?;
        let mut raw = ptr::null_mut();
        check_durable(unsafe { sys::rio_cuda_durable_open(gpu.h(), c.as_ptr(), &mut raw) })?;
        let db = Arc::new(DurableHandle { raw, _engine: gpu.engine.clone() });
        Ok(Self { gpu, db })
    }
    pub fn gpu(&self) -> &GpuObjectPlacement {
        &self.gpu
    }
    /// Bulk-load the table into the GPU directory (after a restart); returns the rows loaded.
    pub fn recover(&self) -> Result<u64, ObjectPlacementError> {
        let mut rows = 0u64;
        check_durable(unsafe { sys::rio_cuda_durable_recover(self.db.raw, &mut rows) })?;
        Ok(rows)
    }
    /// Service::get_or_create_placement for a batch of ids, written through in one transaction.
    pub fn place_batch(&self, ids: &[ObjectId], policy: PlacePolicy) -> Result<Vec<u32>, ObjectPlacementError> {
        let t: Vec<std::ffi::CString> = ids.iter().map(|o| std::ffi::CString::new(o.0.as_str()).unwrap()).collect();
        let i: Vec<std::ffi::CString> = ids.iter().map(|o| std::ffi::CString::new(o.1.as_str()).unwrap()).collect();
        let tp: Vec<*const libc::c_char> = t.iter().map(|s| s.as_ptr()).collect();
        let ip: Vec<*const libc::c_char> = i.iter().map(|s| s.as_ptr()).collect();
        let mut out = vec![sys::RIO_NONE; ids.len()];
        let (policy, me) = policy.raw();
        check_durable(unsafe { sys::rio_cuda_durable_place_batch(self.db.raw, tp.as_ptr(), ip.as_ptr(), ids.len(), policy, me, out.as_mut_ptr()) })?;
        Ok(out)
    }
}

#[async_trait]
impl ObjectPlacement for DurableGpuObjectPlacement {
    // prepare(): the migration ran in open() (sqlite.rs:58-66 does it here; running it twice is harmless: IF NOT EXISTS)

    async fn update(&self, item: ObjectPlacementItem) -> Result<(), ObjectPlacementError> {
        let this = self.clone();
        blocking(move || {
            let (t, i) = (&item.object_id.0, &item.object_id.1);
            let (ap, al) = match &item.server_address { Some(a) => (a.as_ptr() as *const libc::c_char, a.len()), None => (ptr::null(), 0) };
            check_durable(unsafe { sys::rio_cuda_durable_update(this.db.raw, t.as_ptr() as *const _, t.len(), i.as_ptr() as *const _, i.len(), ap, al) })
        })
        .await
    }

    async fn lookup(&self, object_id: &ObjectId) -> Result<Option<String>, ObjectPlacementError> {
        let this = self.clone();
        let (t, i) = (object_id.0.clone(), object_id.1.clone());
        blocking(move || {
            read_string(|buf, cap, len| {
                check_durable(unsafe { sys::rio_cuda_durable_lookup(this.db.raw, t.as_ptr() as *const _, t.len(), i.as_ptr() as *const _, i.len(), buf, cap, len) })
            })
        })
        .await
    }

    async fn clean_server(&self, address: String) -> Result<(), ObjectPlacementError> {
        let this = self.clone();
        blocking(move || check_durable(unsafe { sys::rio_cuda_durable_clean_server(this.db.raw, address.as_ptr() as *const _, address.len()) })).await
    }

    async fn remove(&self, object_id: &ObjectId) -> Result<(), ObjectPlacementError> {
        let this = self.clone();
        let (t, i) = (object_id.0.clone(), object_id.1.clone());
        blocking(move || check_durable(unsafe { sys::rio_cuda_durable_remove(this.db.raw, t.as_ptr() as *const _, t.len(), i.as_ptr() as *const _, i.len()) })).await
    }
}

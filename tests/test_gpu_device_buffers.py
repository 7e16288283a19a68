"""Every device-buffer entry point (rio_cuda_*_dev of include/rio_cuda.h) on the pointers a real caller hands it.

The caller owns the buffers of a _dev call: a slice of a tensor, an offset into a larger allocation.  The ABI asks for natural
alignment only, while some kernels load wider (csrc/buffer_align.cuh: the HRW2 walk's keys and indices, K = 16 feature rows); the engine
copies such a buffer into its own staging buffer when the caller's does not start at the wider alignment.  Every case here lays its
buffers out at chosen byte offsets inside one device arena, each with at least 256 guard bytes on both sides, fills the whole arena
with a canary pattern before the call, and checks that

  * the result equals the reference of the call (the oracle, tests/ranked_oracle.py, tests/spread_oracle.py, the exact fp32
    reference tests/affinity_c32_ref.py on the CUDA cores, the aligned call on the tensor cores), its host-buffer twin and the same
    call on 256-byte aligned views, bit for bit;
  * not one byte outside the output view changed: both guard zones and every input are as they were;
  * the call launched as many kernels as the aligned call (a staging copy is not a launch).

A pointer that is not naturally aligned is refused before anything is enqueued.  The last CPU test runs this module's GPU bodies
against the host-sim library, whose launcher doubles report an access the kernel could not make as a launch error."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import affinity_c32_ref as REF
import ranked_oracle as RO
import spread_oracle as SO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rio_rs_b200", "csrc")
NONE = 0xFFFFFFFF
OK, UNKNOWN = 0, -2
THREADS = os.cpu_count() or 8
GUARD = 256
CANARY = np.array([(i * 61 + 29) & 0xFF for i in range(256)], dtype=np.uint8)   # a permutation of 0..255: no 4-byte word of it is < 2^16 or NONE

# name: (source file under rio_rs_b200/csrc, the text that defines it, its value)
SIZES = {
    "trie_threads": ("k_trie.cu", "constexpr int kTrieThreads = 256;", 256),
    "trie_objs_per_thread": ("k_trie.cu", "constexpr int OPT = 4;\n#ifdef RIO_ASSIGN_TUNING", 4),
    "trie_smem_budget": ("k_trie.cu", "constexpr uint32_t kTrieSmemBudget = 200u * 1024u;", 200 * 1024),
    "umma_rows": ("k_affinity_umma.cu", "constexpr int kRows = 64;", 64),
}


def S(name):
    return SIZES[name][2]


TRIE_TILE = S("trie_threads") * S("trie_objs_per_thread")
LENGTHS = [1, 2, 3, TRIE_TILE - 1, TRIE_TILE, TRIE_TILE + 1, S("umma_rows") - 1, S("umma_rows"), S("umma_rows") + 1, 100_003]
KEY_OFFSETS = [0, 8, 16, 24, 248]
OUT_OFFSETS = [0, 4, 8, 12]
FEAT_OFFSETS = [0, 4, 8, 12, 64]
N = 5003   # a ragged count: four full HRW2 tiles and a tail, 78 full tensor-core row blocks and a tail


@pytest.fixture(scope="module")
def gp():
    from rio_rs_b200 import build

    build.build()
    import rio_rs_b200 as R

    return R


class variant:
    """RIO_AFFINITY_VARIANT for the calls inside the block: 'ffma' keeps every K = 16 call on the CUDA cores."""

    def __init__(self, v):
        self.v = v

    def __enter__(self):
        os.environ["RIO_AFFINITY_VARIANT"] = self.v

    def __exit__(self, *a):
        os.environ.pop("RIO_AFFINITY_VARIANT", None)


def host_sim(p):
    return p.device_info()["name"].startswith("host-sim")


# ---- the arena ---------------------------------------------------------------------------------------------------------------------
class Arena:
    """One rio_cuda_dev_alloc allocation with its base rounded up to 256 bytes.  Buffer b lives in its own 256-aligned region:
    GUARD bytes, offsets[b] bytes, the view, GUARD bytes."""

    def __init__(self, p, sizes, offsets):
        self.p, self.views, at = p, [], 0
        for nbytes, off in zip(sizes, offsets):
            self.views.append((at + GUARD + off, nbytes))
            at = (at + GUARD + off + nbytes + GUARD + 255) // 256 * 256
        self.total = at
        self.raw = C.c_void_p()
        p._ck(p.L.rio_cuda_dev_alloc(p.h, at + 256, C.byref(self.raw)))
        self.base = (self.raw.value + 255) // 256 * 256

    def ptr(self, b):
        return C.c_void_p(self.base + self.views[b][0])

    def write(self, img):
        self.p._ck(self.p.L.rio_cuda_memcpy_h2d(self.p.h, C.c_void_p(self.base), img.ctypes.data_as(C.c_void_p), self.total))

    def read(self):
        img = np.empty(self.total, dtype=np.uint8)
        self.p._ck(self.p.L.rio_cuda_memcpy_d2h(self.p.h, img.ctypes.data_as(C.c_void_p), C.c_void_p(self.base), self.total))
        self.p.sync()
        return img

    def free(self):
        self.p._ck(self.p.L.rio_cuda_dev_free(self.p.h, self.raw))


def run(p, call, ins, outs, refused=False):
    """ins: [(array, byte offset)], outs: [(dtype, shape, byte offset)].  Runs call(*input pointers, *output pointers) on views of
    one canary-filled arena and returns (status, outputs, kernels launched).  Asserts that nothing outside the output views changed,
    and for a refused call that nothing changed at all."""
    outs = [(np.dtype(dt), shape, off) for dt, shape, off in outs]
    sizes = [a.nbytes for a, _ in ins] + [dt.itemsize * int(np.prod(shape)) for dt, shape, _ in outs]
    ar = Arena(p, sizes, [off for _, off in ins] + [off for _, _, off in outs])
    try:
        img = np.resize(CANARY, ar.total)
        for b, (a, _) in enumerate(ins):
            v, nb = ar.views[b]
            img[v:v + nb] = np.ascontiguousarray(a).view(np.uint8).ravel()
        ar.write(img)
        l0 = p.launch_count()
        st = call(*[ar.ptr(b) for b in range(len(sizes))])
        launches = p.launch_count() - l0
        after = ar.read()
        keep = np.ones(ar.total, dtype=bool)
        got = []
        for b, (dt, shape, _) in enumerate(outs):
            v, nb = ar.views[len(ins) + b]
            got.append(after[v:v + nb].copy().view(dt).reshape(shape))
            keep[v:v + nb] = refused
        changed = np.flatnonzero((after != img) & keep)
        assert not len(changed), ("bytes outside the output views changed", changed[:8], ar.views)
        return st, got, launches
    finally:
        ar.free()


def offset_call(p, call, ins, out_shape, in_offs, out_off):
    """The call on views at in_offs / out_off and on 256-byte aligned views: both succeed with equal results and equal launch
    counts.  Returns the result."""
    st0, (want,), l0 = run(p, call, [(a, 0) for a in ins], [(np.uint32, out_shape, 0)])
    st, (got,), l1 = run(p, call, list(zip(ins, in_offs)), [(np.uint32, out_shape, out_off)])
    assert st0 == OK and st == OK, (st0, st, p.L.rio_cuda_last_error(p.h))
    assert (got == want).all(), "the offset views give another result than the aligned ones"
    assert l1 == l0, (l1, l0)
    return got


# ---- the calls -------------------------------------------------------------------------------------------------------------------
def assign_keys(p, n):
    return lambda k, o: p.L.rio_cuda_assign_batch_dev(p.h, k, None, n, o)


def assign_feats(p, n):
    return lambda f, o: p.L.rio_cuda_assign_batch_dev(p.h, None, f, n, o)


def ranked_call(p, kind, n, R):
    fn = {"ranked": p.L.rio_cuda_assign_ranked_batch_dev, "spread": p.L.rio_cuda_assign_ranked_spread_batch_dev,
          "ranked_affinity": p.L.rio_cuda_assign_ranked_affinity_batch_dev,
          "spread_affinity": p.L.rio_cuda_assign_ranked_affinity_spread_batch_dev}[kind]
    return lambda x, o: fn(p.h, x, n, R, o)


# ---- handles and references ------------------------------------------------------------------------------------------------------
HASH_CASES = {   # name: (policy, HRW2 trie bits, RIO_ASSIGN_VARIANT, nodes)
    "hrw_v1": ("hrw", 0, "1", 50),
    "hrw_v2": ("hrw", 0, "2", 50),
    "hrw2_12": ("hrw2", 12, None, 300),
    "hrw2_5": ("hrw2", 5, None, 300),
    "hrw2_global_table": ("hrw2", 12, None, 10_000),   # a blob past the shared-memory budget: the walk reads it from global memory
}


class assign_variant:
    def __init__(self, v):
        self.v = v

    def __enter__(self):
        if self.v:
            os.environ["RIO_ASSIGN_VARIANT"] = self.v

    def __exit__(self, *a):
        os.environ.pop("RIO_ASSIGN_VARIANT", None)


_REF = {}


def hash_handle(gp, oracle, case):
    policy, bits, _, M = HASH_CASES[case]
    p = gp.GpuObjectPlacement()
    p.set_solver(policy, bits)
    addrs, seeds, w = oracle.synth_nodes(M)
    p.set_nodes(addrs, w)
    return p, seeds, w


def hash_reference(oracle, case, keys, seeds, w):
    policy, bits, _, _ = HASH_CASES[case]
    key = (case, len(keys), int(keys[0]))
    if key not in _REF:
        _REF[key] = oracle.assign_hrw2(keys, seeds, w, bits=bits, threads=THREADS) if policy == "hrw2" else \
            oracle.assign_hrw(keys, seeds, w, threads=THREADS)
    return _REF[key]


def feats(n, M, K, seed=0):
    return (np.random.default_rng(100 + seed).uniform(-1, 1, (n, K)).astype(np.float32),
            np.random.default_rng(200 + seed).uniform(-1, 1, (M, K)).astype(np.float32))


def feat_handle(gp, oracle, fn, live=None, dom=None):
    p = gp.GpuObjectPlacement()
    addrs, _, _ = oracle.synth_nodes(len(fn))
    p.set_nodes(addrs, None, fn)
    if live is not None:
        for j in np.flatnonzero(~live):
            p.node_set_active(int(j), False)
    if dom is not None:
        p.set_node_domains(np.arange(len(fn), dtype=np.uint32), dom)
    return p


def group_minimum_check(got1, fo, fn, live):
    """Rank 1 of the tensor-core path is the exact (c32, j) minimum of the live nodes of its own group of 8 live positions."""
    c = REF.c32(fo, fn)
    lidx = np.flatnonzero(live)
    pos = np.full(len(fn), -1, np.int64)
    pos[lidx] = np.arange(len(lidx))
    head = got1.astype(np.int64)
    assert live[head].all()
    gpos = (pos[head] // 8)[:, None] * 8 + np.arange(8)[None, :]
    ok = gpos < len(lidx)
    gj = lidx[np.minimum(gpos, len(lidx) - 1)]
    gc = np.where(ok, c[np.arange(len(head))[:, None], gj], np.inf)
    want = gj[np.arange(len(head)), np.argmin(gc, axis=1)]
    bad = np.flatnonzero(want != head)
    assert not len(bad), ("rank 1 is not its group's c32 minimum", bad[:4])


def check_affinity(p, var, got, fo, fn, live, R=1, dom=None, aligned=None):
    """CUDA cores: the c32 lists bit for bit.  Tensor cores: the aligned call's result (offset_call checked it), rank 1 its group's
    c32 minimum."""
    if var == "ffma" or host_sim(p) or fo.shape[1] != 16:
        want = REF.ranked(fo, fn, live, R) if dom is None else REF.spread(fo, fn, live, dom, R)
        assert (got.reshape(len(fo), R) == want).all()
    else:
        group_minimum_check(got.reshape(len(fo), R)[:, 0], fo, fn, live)


# ---- assign_batch_dev with keys ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("out_off", OUT_OFFSETS)
@pytest.mark.parametrize("key_off", KEY_OFFSETS)
@pytest.mark.parametrize("case", list(HASH_CASES))
def test_assign_keys_at_offsets(gp, oracle, case, key_off, out_off):
    p, seeds, w = hash_handle(gp, oracle, case)
    keys = oracle.synth_keys(N, 3)
    with assign_variant(HASH_CASES[case][2]):
        twin = p.assign_batch(keys)
        got = offset_call(p, assign_keys(p, N), [keys], (N,), [key_off], out_off)
    assert (got == hash_reference(oracle, case, keys, seeds, w)).all()
    assert (got == twin).all()


def test_the_global_table_case_is_past_the_staging_budget(oracle):
    from test_gpu_boundaries import blob_bytes

    _, bits, _, M = HASH_CASES["hrw2_global_table"]
    _, seeds, w = oracle.synth_nodes(M)
    assert blob_bytes(seeds, w, bits) > S("trie_smem_budget")
    _, bits, _, M = HASH_CASES["hrw2_12"]
    _, seeds, w = oracle.synth_nodes(M)
    assert blob_bytes(seeds, w, bits) + 1024 < S("trie_smem_budget")


@pytest.mark.gpu
@pytest.mark.parametrize("n", LENGTHS)
@pytest.mark.parametrize("case", ["hrw_v2", "hrw2_12", "hrw2_5"])
def test_assign_keys_at_every_length(gp, oracle, case, n):
    """Keys 8 bytes past 16 and indices 4 bytes past 8: staged under HRW2, in place under the flat policy."""
    p, seeds, w = hash_handle(gp, oracle, case)
    keys = oracle.synth_keys(n, 5)
    with assign_variant(HASH_CASES[case][2]):
        twin = p.assign_batch(keys)
        got = offset_call(p, assign_keys(p, n), [keys], (n,), [8], 4)
    assert (got == hash_reference(oracle, case, keys, seeds, w)).all()
    assert (got == twin).all()


# ---- assign_batch_dev with features ----------------------------------------------------------------------------------------------
FEAT_CASES = [("ffma", 16), ("ffma", 8), ("ffma", 5), ("umma", 16)]


@pytest.mark.gpu
@pytest.mark.parametrize("out_off", OUT_OFFSETS)
@pytest.mark.parametrize("feat_off", FEAT_OFFSETS)
@pytest.mark.parametrize("var,K", FEAT_CASES)
def test_assign_feats_at_offsets(gp, oracle, var, K, feat_off, out_off):
    fo, fn = feats(N, 100, K)
    live = np.ones(len(fn), bool)
    p = feat_handle(gp, oracle, fn)
    with variant(var):
        twin = p.assign_batch(obj_feats=fo)
        got = offset_call(p, assign_feats(p, N), [fo], (N,), [feat_off], out_off)
    assert (got == twin).all()
    check_affinity(p, var, got, fo, fn, live)


@pytest.mark.gpu
@pytest.mark.parametrize("n", LENGTHS)
@pytest.mark.parametrize("var", ["ffma", "umma"])
def test_assign_feats_at_every_length(gp, oracle, var, n):
    """K = 16 rows 4 bytes past 16: staged on both paths."""
    fo, fn = feats(n, 100, 16, seed=1)
    live = np.ones(len(fn), bool)
    p = feat_handle(gp, oracle, fn)
    with variant(var):
        twin = p.assign_batch(obj_feats=fo)
        got = offset_call(p, assign_feats(p, n), [fo], (n,), [4], 4)
    assert (got == twin).all()
    check_affinity(p, var, got, fo, fn, live)


@pytest.mark.gpu
@pytest.mark.parametrize("var,K", FEAT_CASES)
def test_no_live_node_fills_every_entry_with_none(gp, oracle, var, K):
    n = 3001
    fo, fn = feats(n, 40, K, seed=2)
    p = feat_handle(gp, oracle, fn, live=np.zeros(len(fn), bool))
    with variant(var):
        got = offset_call(p, assign_feats(p, n), [fo], (n,), [4], 4)
        lists = offset_call(p, ranked_call(p, "ranked_affinity", n, 3), [fo], (n, 3), [4], 4)
        spread = offset_call(p, ranked_call(p, "spread_affinity", n, 3), [fo], (n, 3), [4], 4)
    assert (got == NONE).all() and (lists == NONE).all() and (spread == NONE).all()


# ---- ranked calls ----------------------------------------------------------------------------------------------------------------
def domains(M):
    """Racks of 3 nodes, every seventh node a domain of its own."""
    d = (np.arange(M) // 3).astype(np.uint32)
    d[::7] = NONE
    return d


@pytest.mark.gpu
@pytest.mark.parametrize("key_off,out_off", [(0, 0), (8, 4), (248, 12)])
@pytest.mark.parametrize("R", [1, 3, 8])
@pytest.mark.parametrize("kind", ["ranked", "spread"])
@pytest.mark.parametrize("policy", ["hrw", "hrw2"])
def test_ranked_hash_lists_at_offsets(gp, oracle, policy, kind, R, key_off, out_off):
    M, n = 60, 4099
    p = gp.GpuObjectPlacement()
    p.set_solver(policy, 0)
    addrs, seeds, w = oracle.synth_nodes(M)
    w = w.copy()
    w[5] = 0   # one node not live
    p.set_nodes(addrs, w)
    dom = domains(M)
    keys = oracle.synth_keys(n, 9)
    if kind == "spread":
        p.set_node_domains(np.arange(M, dtype=np.uint32), dom)
        twin = p.assign_ranked_spread(keys, R)
        want = SO.assign_spread(policy, keys, seeds, w, dom, R, threads=THREADS)
    else:
        twin = p.assign_ranked(keys, R)
        want = RO.assign_ranked(policy, keys, seeds, w, R, threads=THREADS)
    got = offset_call(p, ranked_call(p, kind, n, R), [keys], (n, R), [key_off], out_off)
    assert (got == want).all()
    assert (got == twin).all()


@pytest.mark.gpu
@pytest.mark.parametrize("feat_off,out_off", [(0, 0), (4, 4), (64, 12), (12, 8)])
@pytest.mark.parametrize("R", [1, 3, 8])
@pytest.mark.parametrize("kind", ["ranked_affinity", "spread_affinity"])
@pytest.mark.parametrize("var", ["ffma", "umma"])
def test_ranked_affinity_lists_at_offsets(gp, oracle, var, kind, R, feat_off, out_off):
    M, n = 90, S("umma_rows") * 40 + 3
    fo, fn = feats(n, M, 16, seed=3)
    live = np.ones(M, bool)
    live[[4, 50]] = False
    dom = domains(M) if kind == "spread_affinity" else None
    p = feat_handle(gp, oracle, fn, live=live, dom=dom)
    with variant(var):
        twin = p.assign_ranked_affinity(fo, R) if dom is None else p.assign_ranked_affinity_spread(fo, R)
        got = offset_call(p, ranked_call(p, kind, n, R), [fo], (n, R), [feat_off], out_off)
    assert (got == twin).all()
    check_affinity(p, var, got, fo, fn, live, R, dom)


# ---- directory ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("key_off,idx_off", [(0, 0), (8, 4), (24, 12), (248, 8)])
def test_directory_upsert_and_lookup_at_offsets(gp, oracle, key_off, idx_off):
    """Two upsert batches (the second overwrites half of the first and repeats keys inside itself: the last one wins), then a lookup
    of placed and unknown keys, against oracle.DirectoryModel fed the same updates and a twin handle fed them through host buffers."""
    M = 20
    addrs, _, w = oracle.synth_nodes(M)
    p, twin = gp.GpuObjectPlacement(), gp.GpuObjectPlacement()
    for q in (p, twin):
        q.set_nodes(addrs, w)
    model = oracle.DirectoryModel()
    rng = np.random.default_rng(7)
    k1 = oracle.synth_keys(3001, 21)
    k2 = np.concatenate([k1[::2], oracle.synth_keys(1000, 22)])
    k2 = np.concatenate([k2, k2[:300]])
    p._ck(p.L.rio_cuda_directory_reserve(p.h, len(k1) + len(k2)))
    for keys in (k1, k2):
        idx = rng.integers(0, M, len(keys)).astype(np.uint32)
        st, _, _ = run(p, lambda k, i: p.L.rio_cuda_upsert_batch_dev(p.h, k, i, len(keys)), [(keys, key_off), (idx, idx_off)], [])
        assert st == OK
        twin.update_many(keys, idx)
        for k, i in zip(keys, idx):
            model.update("t", str(int(k)), addrs[int(i)])
    probe = np.concatenate([k1, k2[-500:], oracle.synth_keys(700, 23)])
    by_addr = {a: j for j, a in enumerate(addrs)}
    want = np.array([by_addr.get(model.lookup("t", str(int(k))), NONE) for k in probe], dtype=np.uint32)
    got = offset_call(p, lambda k, o: p.L.rio_cuda_lookup_batch_dev(p.h, k, len(probe), o), [probe], (len(probe),), [key_off], idx_off)
    assert (got == want).all()
    assert (got == twin.lookup_many(probe)).all()
    assert (want == NONE).sum() == 700
    assert p.directory_len()[0] == len(model)


# ---- refusals ----------------------------------------------------------------------------------------------------------------------
def refusal_cases():
    cases = []
    for case in ("hrw", "hrw2"):
        cases += [("assign_keys", case, "keys", 4), ("assign_keys", case, "out", 2),
                  ("ranked", case, "keys", 4), ("ranked", case, "out", 2), ("spread", case, "keys", 4), ("spread", case, "out", 2)]
    for var in ("ffma", "umma"):
        for kind in ("assign_feats", "ranked_affinity", "spread_affinity"):
            cases += [(kind, var, "feats", 2), (kind, var, "out", 2)]
    cases += [("lookup", "hrw", "keys", 4), ("lookup", "hrw", "out", 2), ("upsert", "hrw", "keys", 4), ("upsert", "hrw", "idx", 2)]
    return cases


@pytest.mark.gpu
@pytest.mark.parametrize("call,mode,buf,off", refusal_cases())
def test_a_pointer_off_its_natural_alignment_is_refused(gp, oracle, call, mode, buf, off):
    """RIO_ERR_UNKNOWN, nothing launched, output and guards untouched (run() checks every byte), and the next aligned call on the
    handle is right."""
    n, M, R = 2051, 40, 3
    addrs, seeds, w = oracle.synth_nodes(M)
    keys = oracle.synth_keys(n, 31)
    fo, fn = feats(n, M, 16, seed=4)
    p = gp.GpuObjectPlacement()
    if call in ("assign_feats", "ranked_affinity", "spread_affinity"):
        p.set_nodes(addrs, w, fn)
        x, ctx = fo, variant(mode)
    else:
        p.set_solver(mode, 0)
        p.set_nodes(addrs, w)
        x, ctx = keys, assign_variant(None)
    if call == "spread" or call == "spread_affinity":
        p.set_node_domains(np.arange(M, dtype=np.uint32), domains(M))
    p._ck(p.L.rio_cuda_directory_reserve(p.h, n))
    idx = (np.arange(n) % M).astype(np.uint32)
    if call == "upsert":
        fn_call = lambda k, i: p.L.rio_cuda_upsert_batch_dev(p.h, k, i, n)
        st, _, launches = run(p, fn_call, [(keys, off if buf == "keys" else 0), (idx, off if buf == "idx" else 0)], [], refused=True)
        assert st == UNKNOWN and launches == 0 and p.directory_len()[0] == 0
        st, _, _ = run(p, fn_call, [(keys, 8), (idx, 4)], [])
        assert st == OK and (p.lookup_many(keys) == idx).all()
        return
    shape = (n, R) if call in ("ranked", "spread", "ranked_affinity", "spread_affinity") else (n,)
    fn_call = {"assign_keys": lambda: assign_keys(p, n), "assign_feats": lambda: assign_feats(p, n),
               "lookup": lambda: (lambda k, o: p.L.rio_cuda_lookup_batch_dev(p.h, k, n, o))}.get(call, lambda: ranked_call(p, call, n, R))()
    with ctx:
        st, _, launches = run(p, fn_call, [(x, 0 if buf == "out" else off)], [(np.uint32, shape, off if buf == "out" else 0)], refused=True)
        assert st == UNKNOWN and launches == 0
        assert "aligned" in p.L.rio_cuda_last_error(p.h).decode()
        st, (got,), _ = run(p, fn_call, [(x, 0)], [(np.uint32, shape, 0)])
        assert st == OK
        twin = {"assign_keys": lambda: p.assign_batch(keys), "assign_feats": lambda: p.assign_batch(obj_feats=fo),
                "ranked": lambda: p.assign_ranked(keys, R), "spread": lambda: p.assign_ranked_spread(keys, R),
                "ranked_affinity": lambda: p.assign_ranked_affinity(fo, R), "spread_affinity": lambda: p.assign_ranked_affinity_spread(fo, R),
                "lookup": lambda: np.full(n, NONE, np.uint32)}[call]()
    assert (got == twin).all()
    if call == "assign_keys":
        want = oracle.assign_hrw2(keys, seeds, w, threads=THREADS) if mode == "hrw2" else oracle.assign_hrw(keys, seeds, w, threads=THREADS)
        assert (got == want).all()


# ---- stream order ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("what", ["hrw2", "ffma", "umma"])
def test_two_staged_calls_in_a_row_without_a_host_sync(gp, oracle, what):
    """Two calls that both stage, the second larger (its staging buffers grow), write adjacent views of one output buffer; the host
    waits only once, after both.  Both halves must be right: the second call's staging must not overtake the first one's copy back."""
    n1, n2 = 5000, 70_002   # even counts: both output views sit 4 bytes past 8, both key views 8 past 16, both feature views 4 past 16
    n = n1 + n2
    if what == "hrw2":
        p, seeds, w = hash_handle(gp, oracle, "hrw2_12")
        x = oracle.synth_keys(n, 41)
        want = hash_reference(oracle, "hrw2_12", x, seeds, w)
        stride, ctx = 8, assign_variant(None)
        go = lambda xp, op, m: p.L.rio_cuda_assign_batch_dev(p.h, xp, None, m, op)
        in_off = 8
    else:
        x, fn = feats(n, 100, 16, seed=5)
        p = feat_handle(gp, oracle, fn)
        stride, ctx = 64, variant(what)
        go = lambda xp, op, m: p.L.rio_cuda_assign_batch_dev(p.h, None, xp, m, op)
        in_off = 4
    with ctx:
        if what != "hrw2":
            want = p.assign_batch(obj_feats=x)

        def both(xp, op):
            st1 = go(xp, op, n1)
            st2 = go(C.c_void_p(xp.value + n1 * stride), C.c_void_p(op.value + n1 * 4), n2)
            return st1 or st2

        st, (got,), _ = run(p, both, [(x, in_off)], [(np.uint32, (n,), 4)])
    assert st == OK
    assert (got[:n1] == want[:n1]).all() and (got[n1:] == want[n1:]).all()
    if what != "hrw2":
        check_affinity(p, what, got, x, fn, np.ones(len(fn), bool))


# ---- CPU -------------------------------------------------------------------------------------------------------------------------
def test_sizes_are_where_the_sources_define_them():
    for name, (f, text, _) in SIZES.items():
        assert text in open(os.path.join(CSRC, f)).read(), "%s: %r is no longer in %s" % (name, text, f)


def test_the_alignment_rules_are_declared_once():
    """buffer_align.cuh declares the wider alignments; the engine's _dev calls and the host-sim doubles read them from there."""
    decl = open(os.path.join(CSRC, "buffer_align.cuh")).read()
    for name in ("kAlignTrieKeys", "kAlignTrieOut", "affinity_feats_align"):
        assert re.search(r"\b%s\b" % name, decl), name
    engine = open(os.path.join(CSRC, "engine.cu")).read()
    sim = os.path.join(ROOT, "tests", "cpp", "hostsim")
    for name in ("kAlignTrieKeys", "kAlignTrieOut", "affinity_feats_align"):
        assert name in engine and name in open(os.path.join(sim, "launchers.cpp")).read(), name
    for f in ("affinity_ranked_launchers.cpp", "affinity_spread_launchers.cpp"):
        assert "affinity_feats_align" in open(os.path.join(sim, f)).read(), f


HOSTSIM_DOUBLES = ["ranked_launchers.cpp", "spread_launchers.cpp", "affinity_ranked_launchers.cpp", "affinity_spread_launchers.cpp"]


def test_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + the ranked, spread and
    affinity list doubles).  There allocations are 256-byte aligned, as on the device, and a double whose kernel would fault on a
    buffer reports a misaligned-address launch error; the tensor-core path is never selected."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, "librio_cuda_hostsim_device_buffers.so")
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + [os.path.join(HS.SIM, f) for f in HOSTSIM_DOUBLES] + ["-o", so, "-ldl", "-lpthread"])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=3000, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 300 and "failed" not in r.stdout, tail

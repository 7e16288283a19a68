"""The size thresholds the launchers branch on, tested on both sides.

Every launcher picks a kernel variant, a shared-memory layout or a counter path from a size: the number of live or interned nodes, the
bytes of a table, the number of objects in a host buffer.  The shapes of the other test modules sit well inside one side of those
thresholds; this module puts a case on each side of every one of them, against the oracles the other modules use (hash paths bit for
bit, the affinity path under the fp64 oracle of tests/affinity_ranked_oracle.py).  It also runs the ranked kernels at extreme weights:
more weight classes than the default node set has, weights of 1 and 2^32 - 1, and HRW2 subtree weights whose contests need all
128 bits of the exact compare.

THRESHOLDS holds the constants these cases are built around, each with the source line that defines it.  A CPU test checks that
those lines are still there, so moving a threshold breaks this module instead of leaving its boundary cases on one side.  The last
CPU test runs this module's GPU bodies, unchanged, against the engine's host logic compiled with g++ (the host-sim library of
tests/test_engine_host_sim.py plus both ranked launcher restatements); there the tensor-core path is never selected."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import affinity_ranked_oracle as AO
import ranked_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rio_rs_b200", "csrc")
NONE = 0xFFFFFFFF
THREADS = os.cpu_count() or 8

# name: (source file under rio_rs_b200/csrc, the text that defines it, its value)
THRESHOLDS = {
    "flat_chunk_nodes": ("k_assign.cu", "tab.n_live < 8192 ? tab.n_live : 8192", 8192),
    "flat_hist_bins": ("k_assign.cu", "(d_counters && tab.n_total <= 8192) ? tab.n_total : 0", 8192),
    "v2_max_live": ("k_assign.cu", "constexpr uint32_t kV2MaxLive = 0xFFFF;", 0xFFFF),
    "affinity_chunk_nodes": ("k_assign.cu", "n_total < 2048 ? n_total : 2048", 2048),
    "check_nodes_per_thread_trip": ("bounded_tail.cuh", "for (uint32_t j0 = threadIdx.x; j0 < M; j0 += 4 * blockDim.x)", 4),
    "check_threads_flat": ("k_directory.cu", "k_exchange_check<<<1, 256, 0, L.stream>>>", 256),
    "check_threads_hrw2": ("k_trie.cu", "constexpr int kTrieThreads = 256;", 256),
    "trie_hist_bins": ("k_trie.cu", "(want_hist && n_total <= 8192) ? n_total : 0", 8192),
    "trie_smem_budget": ("k_trie.cu", "constexpr uint32_t kTrieSmemBudget = 200u * 1024u;", 200 * 1024),
    "umma_small_pad": ("engine.cu", "nl <= 64 ? 64 : (nl + 255) / 256 * 256", 64),
    "umma_pad_step": ("engine.cu", "nl <= 64 ? 64 : (nl + 255) / 256 * 256", 256),
    "umma_max_nodes": ("k_affinity_umma.cu", "uint32_t affinity_umma_max_nodes() { return ((227u * 1024u) / 96u) / 256u * 256u; }",
                       ((227 * 1024) // 96) // 256 * 256),
    "umma_rows": ("k_affinity_umma.cu", "constexpr int kRows = 64;", 64),
    "resolve_hist_bins": ("k_affinity_umma.cu", "(d_counters && n_total <= 8192) ? n_total : 0", 8192),
    "feature_pipeline_chunk": ("engine.cu", "const size_t chunk = feats ? (size_t)(1u << 20)", 1 << 20),
    "ranked_flat_smem": ("k_ranked.cu", "if (smem <= 96u * 1024u) {", 96 * 1024),
    "rank_smem_budget": ("k_ranked.cu", "constexpr uint32_t kRankSmemBudget = 200u * 1024u;", 200 * 1024),
    "ranked_trie_staged": ("k_ranked.cu", "const size_t smem = (size_t)t.blob_bytes + rk.bytes;\n    if (smem <= kRankSmemBudget) {", 200 * 1024),
}


def T(name):
    return THRESHOLDS[name][2]


CHECK_TRIP = T("check_nodes_per_thread_trip") * T("check_threads_flat")   # nodes one trip of the capacity check covers
RANKED_FLAT_MAX_LIVE = T("ranked_flat_smem") // 16                      # 16-byte node records


@pytest.fixture(scope="module")
def gp():
    from rio_rs_b200 import build

    build.build()
    import rio_rs_b200 as R

    return R


def provider(gp, policy="hrw", bits=0):
    p = gp.GpuObjectPlacement()
    p.set_solver(policy, bits)
    return p


class variant:
    """RIO_AFFINITY_VARIANT for the calls inside the block: 'ffma' keeps every K = 16 call on the CUDA cores."""

    def __init__(self, v):
        self.v = v

    def __enter__(self):
        os.environ["RIO_AFFINITY_VARIANT"] = self.v

    def __exit__(self, *a):
        os.environ.pop("RIO_AFFINITY_VARIANT", None)


def feats(n, M, K=16):
    return (np.random.default_rng(11).uniform(-1, 1, (n, K)).astype(np.float32),
            np.random.default_rng(13).uniform(-1, 1, (M, K)).astype(np.float32))


def tensor_cores(p, var, K, n_live):
    step = T("umma_pad_step")
    padded = T("umma_small_pad") if n_live <= T("umma_small_pad") else (n_live + step - 1) // step * step
    # the host-sim build of the engine (tests/test_engine_host_sim.py) restates no tensor-core kernel
    return var == "umma" and K == 16 and 0 < padded <= T("umma_max_nodes") and not p.device_info()["name"].startswith("host-sim")


def plain(oracle, policy, keys, seeds, w):
    """The single assignment under the policy (HRW2 at the default 12 bits)."""
    if policy == "hrw2":
        return oracle.assign_hrw2(keys, seeds, w, threads=THREADS)
    return oracle.assign_hrw(keys, seeds, w, threads=THREADS)


def capacities(n, w, num, den):
    """Per-node capacity of a bounded call (DESIGN.md 3.5): ceil(num * n * w / (den * sum w)), 0 for weight 0."""
    total = int(np.asarray(w, dtype=np.uint64).sum())
    return np.array([min((num * n * int(x) + den * total - 1) // (den * total), NONE) if x else 0 for x in w], dtype=np.uint64)


# ---- HRW2 table bytes (DESIGN.md 4.1 / 3.9) -------------------------------------------------------------------------------------
SALT_POS = 0x8CB92BA72F3D8DD7   # kSaltPos of spec.cuh: a node's position in the trie


def mix64(x):
    x = np.asarray(x, dtype=np.uint64).copy()
    with np.errstate(over="ignore"):
        x ^= x >> np.uint64(30)
        x *= np.uint64(0xBF58476D1CE4E5B9)
        x ^= x >> np.uint64(27)
        x *= np.uint64(0x94D049BB133111EB)
        x ^= x >> np.uint64(31)
    return x


def blob_bytes(seeds, w, bits):
    """Bytes of the HRW2 blob: 8 * 2^bits of thresholds and leaf words padded to 16, then one 32-byte chain record per live member
    beyond the first of its bucket; at least 16."""
    live = np.asarray(w) > 0
    bucket = mix64(np.asarray(seeds, dtype=np.uint64)[live] ^ np.uint64(SALT_POS)) >> np.uint64(64 - bits) if bits else np.zeros(int(live.sum()))
    chains = int(live.sum()) - len(np.unique(bucket))
    return max(16, (8 * (1 << bits) + 15) // 16 * 16 + 32 * chains)


def rank_side_bytes(n_total, bits):
    """Bytes of the side table of the ranked HRW2 walk: the u64 subtree-weight heap, then one {bucket, weight} pair per interned node
    padded to 16 bytes."""
    return 16 * (1 << bits) + (8 * n_total + 15) // 16 * 16


def staged_ranked_trie_bytes(seeds, w, bits):
    return blob_bytes(seeds, w, bits) + rank_side_bytes(len(seeds), bits)


def largest_staged_ranked_trie(oracle, bits, hi):
    """The largest M whose ranked HRW2 table (blob + side table of synth_nodes(M)) is still staged in shared memory.  Growing the node
    set never shrinks the table, so the smallest unstaged one is M + 1."""
    _, seeds, w = oracle.synth_nodes(hi)
    lo, up = 1, hi   # staged(lo), not staged(up)
    assert staged_ranked_trie_bytes(seeds[:lo], w[:lo], bits) <= T("rank_smem_budget") < staged_ranked_trie_bytes(seeds, w, bits)
    while up - lo > 1:
        mid = (lo + up) // 2
        if staged_ranked_trie_bytes(seeds[:mid], w[:mid], bits) <= T("rank_smem_budget"):
            lo = mid
        else:
            up = mid
    return lo


# ---- load counters on every counter path ----------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("policy", ["hrw", "hrw2"])
@pytest.mark.parametrize("M", [T("flat_hist_bins"), T("flat_hist_bins") + 1])
def test_load_counters_on_both_sides_of_the_shared_memory_histogram(gp, oracle, policy, M):
    """Up to 8192 interned nodes the assignment kernels count in a shared-memory histogram, beyond that with global atomics.  Under
    the flat policy 8192 live nodes are also the largest table of one shared-memory chunk: the largest dynamic shared memory of
    k_assign_hrw_v2 (8192 records + 8192 bins)."""
    assert T("flat_hist_bins") == T("trie_hist_bins") == T("flat_chunk_nodes")
    p = provider(gp, policy)
    addrs, seeds, w = oracle.synth_nodes(M)
    p.set_nodes(addrs, w)
    keys = oracle.synth_keys(20_011, 3)
    s = p.new_set(len(keys))
    s.load_keys(keys)
    s.assign()
    want = plain(oracle, policy, keys, seeds, w)
    assert (s.read() == want).all()
    assert (s.counters() == oracle.counts(want, M)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("var", ["umma", "ffma"])
def test_affinity_load_counters_with_more_nodes_interned_than_the_histogram_holds(gp, oracle, var):
    """9000 interned nodes, 2248 of them live (every fourth has weight > 0, two of those are inactive): the tensor path's padded live
    set is its largest, 2304, and its resolve pass counts with global atomics; the CUDA-core kernel walks five node chunks."""
    M, n = 9000, 20_000
    fo, fn = feats(n, M)
    addrs, _, _ = oracle.synth_nodes(M)
    w = np.where(np.arange(M) % 4 == 0, 1, 0).astype(np.uint32)
    p = gp.GpuObjectPlacement()
    p.set_nodes(addrs, w, fn)
    live = w > 0
    for j in (8, 8196):
        p.node_set_active(j, False)
        live[j] = False
    n_live = int(live.sum())
    assert n_live == 2248 and M > T("resolve_hist_bins")
    s = p.new_set(n)
    s.load_keys(np.arange(n, dtype=np.uint64))
    s.load_feats(fo)
    with variant(var):
        one = p.assign_batch(obj_feats=fo)   # the table upload happens here, not in the counted call
        l0 = p.launch_count()
        s.assign(True)
        launches = p.launch_count() - l0
    assert launches == (2 if tensor_cores(p, var, 16, n_live) else 1), launches
    got = s.read()
    assert (got == one).all()
    AO.check(got[:, None], fo, fn, live)
    cnt = s.counters()
    assert (cnt == oracle.counts(got, M)).all()
    assert cnt[T("resolve_hist_bins"):].sum() > 0   # nodes past the histogram's reach were counted


# ---- bounded rounds beyond one trip of the capacity check -----------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("policy", ["hrw", "hrw2"])
@pytest.mark.parametrize("M", [CHECK_TRIP + 1, 4 * CHECK_TRIP + 4, 9000])
def test_bounded_rounds_past_one_trip_of_the_capacity_check(gp, oracle, policy, M):
    """The capacity check is one 256-thread block that covers 1024 nodes per trip: M = 1025 adds a second trip for one node, 4100 a
    fifth, 9000 also takes its counters from global atomics.  Passes, indices and counters equal the oracle's; some node past the
    first trip is over capacity after pass 0, so the later trips decide spills."""
    assert CHECK_TRIP == 1024 and T("check_threads_hrw2") == T("check_threads_flat")
    p = provider(gp, policy)
    addrs, seeds, w = oracle.synth_nodes(M)
    p.set_nodes(addrs, w)
    n = 40_000
    keys = oracle.synth_keys(n, 17)   # a key stream that puts node 1024 of the 1025-node set over capacity under both policies
    s = p.new_set(n)
    s.load_keys(keys)
    first = oracle.counts(plain(oracle, policy, keys, seeds, w), M).astype(np.uint64)
    bounded = oracle.assign_bounded_hrw2 if policy == "hrw2" else oracle.assign_bounded
    over_past_first_trip, spilled = False, False
    for cap in [(5, 4), (101, 100)]:
        passes = s.assign_bounded(0, cap[0], cap[1], 4)
        widx, wcnt, wpass = bounded(keys, seeds, w, cap[0], cap[1], 4, threads=THREADS)
        assert passes == wpass, cap
        assert (s.read() == widx).all(), cap
        assert (s.counters() == wcnt).all(), cap
        over_past_first_trip |= bool((first[CHECK_TRIP:] > capacities(n, w, *cap)[CHECK_TRIP:]).any())
        spilled |= wpass > 1
    assert spilled and over_past_first_trip


# ---- host buffers over more than one pipeline chunk -------------------------------------------------------------------------------
_PIPE = {}


@pytest.mark.gpu
@pytest.mark.parametrize("var", ["umma", "ffma"])
def test_feature_placement_over_several_pipeline_chunks(gp, oracle, var):
    """assign_batch(obj_feats) streams host buffers in chunks of 2^20 objects: 2^21 + 17 objects are two full chunks and a ragged
    one."""
    M, n = 100, 2 * T("feature_pipeline_chunk") + 17
    if "fo" not in _PIPE:
        fo, fn = feats(n, M)
        _PIPE.update(fo=fo, fn=fn, want=AO.ranked(fo, fn, np.ones(M, bool), 2))
    fo, fn = _PIPE["fo"], _PIPE["fn"]
    p = gp.GpuObjectPlacement()
    addrs, _, _ = oracle.synth_nodes(M)
    p.set_nodes(addrs, None, fn)
    with variant(var):
        got = p.assign_batch(obj_feats=fo)
    AO.check(got[:, None], fo, fn, np.ones(M, bool), _PIPE["want"])


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, T("umma_rows") - 1, T("umma_rows"), T("umma_rows") + 1])
def test_tensor_path_at_row_block_edges(gp, oracle, n):
    """The tensor-core kernels take objects in row blocks of 64: one object, a block short by one, one full block, one past it."""
    M = 300
    fo, fn = feats(n, M)
    p = gp.GpuObjectPlacement()
    addrs, _, _ = oracle.synth_nodes(M)
    p.set_nodes(addrs, None, fn)
    with variant("umma"):
        one = p.assign_batch(obj_feats=fo)
        l0 = p.launch_count()
        got = p.assign_ranked_affinity(fo, 3)
        launches = p.launch_count() - l0
    assert launches == (2 if tensor_cores(p, "umma", 16, M) else 1), launches
    assert got.shape == (n, 3) and (got[:, 0] == one).all()
    AO.check(one[:, None], fo, fn, np.ones(M, bool))
    AO.check(got, fo, fn, np.ones(M, bool))


# ---- ranked tables at their shared-memory limits -----------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("M", [RANKED_FLAT_MAX_LIVE, RANKED_FLAT_MAX_LIVE + 1])
def test_ranked_flat_table_at_the_shared_memory_limit(gp, oracle, M):
    """The flat ranked kernel stages the table in shared memory up to 96 KB of 16-byte records: 6144 live nodes, then reads it from
    global memory."""
    assert RANKED_FLAT_MAX_LIVE == 6144
    p = provider(gp, "hrw")
    addrs, seeds, w = oracle.synth_nodes(M)
    p.set_nodes(addrs, w)
    keys = oracle.synth_keys(10_007, 4)
    got = p.assign_ranked(keys, 3)
    assert (got[:, 0] == p.assign_batch(keys)).all()
    assert (got == RO.assign_ranked("hrw", keys, seeds, w, 3, threads=THREADS)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("past", [0, 1])
def test_ranked_trie_at_the_shared_memory_limit(gp, oracle, past):
    """The ranked HRW2 walk stages blob + side table in shared memory while they fit in 200 KB: the largest node set at the default
    12 bits whose table does (past = 0) and the smallest that does not (past = 1)."""
    bits = 12
    M = largest_staged_ranked_trie(oracle, bits, 6000) + past
    addrs, seeds, w = oracle.synth_nodes(M)
    assert (staged_ranked_trie_bytes(seeds, w, bits) > T("rank_smem_budget")) == bool(past)
    p = provider(gp, "hrw2", bits)
    p.set_nodes(addrs, w)
    keys = oracle.synth_keys(20_011, 5)
    got = p.assign_ranked(keys, 3)
    assert (got[:, 0] == p.assign_batch(keys)).all()
    assert (got == RO.assign_ranked("hrw2", keys, seeds, w, 3, bits=bits, threads=THREADS)).all()


# ---- ranked lists at extreme weights --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("ranks", [2, 8])
def test_ranked_flat_lists_with_hundreds_of_weight_classes(gp, oracle, ranks):
    """~300 distinct weights from [1, 2^31), one node of weight 2^32 - 1 and one of weight 1: every weight class merges its best R
    into the list, with the largest and the smallest inverse weight among them."""
    M = 302
    addrs, seeds, _ = oracle.synth_nodes(M)
    w = np.random.default_rng(4).integers(1, 2**31, M).astype(np.uint32)
    w[7], w[8] = 0xFFFFFFFF, 1
    assert len(np.unique(w)) > 290
    p = provider(gp, "hrw")
    p.set_nodes(addrs, w)
    keys = oracle.synth_keys(30_011, 6)
    got = p.assign_ranked(keys, ranks)
    assert (got[:, 0] == p.assign_batch(keys)).all()
    assert (got == RO.assign_ranked("hrw", keys, seeds, w, ranks, threads=THREADS)).all()
    assert (got[:, 0] == 7).sum() > (got[:, 0] == 6).sum()   # the heaviest class really competes


@pytest.mark.gpu
@pytest.mark.parametrize("ranks", [2, 8])
@pytest.mark.parametrize("bits,M", [(12, 5000), (4, 300), (1, 300)])
def test_ranked_trie_lists_near_the_largest_weight(gp, oracle, bits, M, ranks):
    """Weights within 16 of 2^32 - 1 and every 23rd node of weight 1: the subtree sums exceed 2^33, so at the root the product
    (v + 1)(wl' + wr') of the exact contest exceeds 2^64 and its high word decides; at 4 and 1 bits long chains hold several
    excluded nodes and weight-1 members side by side."""
    addrs, seeds, _ = oracle.synth_nodes(M)
    w = (0xFFFFFFFF - np.random.default_rng(5).integers(0, 17, M)).astype(np.uint32)
    w[::23] = 1
    assert int(w.astype(np.uint64).sum()) >= 2**33
    p = provider(gp, "hrw2", bits)
    p.set_nodes(addrs, w)
    keys = oracle.synth_keys(20_011 if M > 1000 else 30_011, 7)
    got = p.assign_ranked(keys, ranks)
    assert (got[:, 0] == p.assign_batch(keys)).all()
    assert (got == RO.assign_ranked("hrw2", keys, seeds, w, ranks, bits=bits, threads=THREADS)).all()
    bucket = mix64(seeds ^ np.uint64(SALT_POS)) >> np.uint64(64 - bits)
    assert np.isin(bucket[w == 1], bucket[w > 1]).any()   # weight-1 members in the chains of heavy ones


@pytest.mark.gpu
@pytest.mark.parametrize("var", ["umma", "ffma"])
@pytest.mark.parametrize("ranks", [5, 6, 7])
def test_ranked_affinity_lists_shorter_than_the_kept_groups(gp, oracle, ranks, var):
    """R = 5, 6 and 7 keep 8 groups per object on the tensor path and emit fewer ranks than they keep."""
    M, n = 1024, 20_000
    fo, fn = feats(n, M)
    p = gp.GpuObjectPlacement()
    addrs, _, _ = oracle.synth_nodes(M)
    p.set_nodes(addrs, None, fn)
    with variant(var):
        got = p.assign_ranked_affinity(fo, ranks)
        one = p.assign_batch(obj_feats=fo)
    assert got.shape == (n, ranks)
    assert (got[:, 0] == one).all()
    AO.check(got, fo, fn, np.ones(M, bool))


# ---- CPU ---------------------------------------------------------------------------------------------------------------------------
def test_thresholds_are_where_the_sources_define_them():
    for name, (f, text, _) in THRESHOLDS.items():
        src = open(os.path.join(CSRC, f)).read()
        assert text in src, "%s: %r is no longer in %s" % (name, text, f)
    assert T("umma_max_nodes") == 2304 and T("rank_smem_budget") == T("ranked_trie_staged")


BLOB_SIZE_PROGRAM = r"""
#include <cstdio>
#include "trie_table.hpp"
int main() {
    unsigned bits, m;
    std::vector<rio::TrieMember> mem;
    if (std::scanf("%u %u", &bits, &m) != 2) return 1;
    for (unsigned j = 0; j < m; j++) {
        unsigned long long seed; unsigned w;
        if (std::scanf("%llu %u", &seed, &w) != 2) return 1;
        mem.push_back(rio::TrieMember{seed, j, w});
    }
    std::printf("%u\n", rio::build_trie_blob(mem, bits).blob_bytes);
    return 0;
}
"""


def test_trie_blob_bytes_formula_matches_the_builder(tmp_path, oracle):
    """blob_bytes() above, which places the HRW2 boundary cases, against the blob csrc/trie_table.hpp builds."""
    import shutil

    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else shutil.which("g++")
    if not gxx:
        pytest.skip("no host C++ compiler")
    src, exe = tmp_path / "blob_size.cpp", str(tmp_path / "blob_size")
    src.write_text(BLOB_SIZE_PROGRAM)
    subprocess.check_call([gxx, "-std=c++17", "-O1", "-I" + CSRC, str(src), "-o", exe])
    _, seeds, w = oracle.synth_nodes(5000)
    w = w.copy()
    w[::7] = 0   # not live: no record, no bucket
    for bits in (0, 1, 4, 12, 14):
        for M in (0, 1, 2, 300, 4950, 5000):
            stdin = "%d %d\n" % (bits, M) + "".join("%d %d\n" % (int(seeds[j]), int(w[j])) for j in range(M))
            r = subprocess.run([exe], input=stdin, capture_output=True, text=True, timeout=60)
            assert r.returncode == 0, r.stderr
            assert int(r.stdout) == blob_bytes(seeds[:M], w[:M], bits), (bits, M)


def test_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + both ranked launcher
    restatements)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, "librio_cuda_hostsim_boundaries.so")
    doubles = [os.path.join(HS.SIM, f) for f in ("ranked_launchers.cpp", "affinity_ranked_launchers.cpp")]
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + doubles + ["-o", so, "-ldl", "-lpthread"])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 35 and "failed" not in r.stdout, tail

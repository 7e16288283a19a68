"""Failure-domain ranked placement (DESIGN.md 3.12): each object's first R nodes in R distinct domains under the handle's policy,
through the C ABI, compared list for list with the CPU oracle (tests/spread_oracle.c: one masked single assignment per rank with every
node of the earlier ranks' domains removed, the definition itself) under both policies.  Rank 1 is assign_batch bit for bit, the
entries are live and lie in distinct domains, NONE pads the lists past the live domain count, no labels give assign_ranked_batch, and
rank 2 is where the object goes when rank 1's whole domain leaves.

The CPU tests at the end run this module's GPU bodies, unchanged, against the engine's host logic compiled with g++ (the host-sim
library of tests/test_engine_host_sim.py) with plain restatements of the spread launchers, and check that a build without them
refuses the spread call while the ranked call keeps working."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import spread_oracle as SO

NONE = 0xFFFFFFFF
POLICIES = ["hrw", "hrw2"]
THREADS = os.cpu_count() or 8
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rio_rs_b200", "csrc")
HOSTSIM = bool(os.environ.get("RIO_HOSTSIM_LIBRARY"))

# the staging thresholds of k_spread.cu's launchers: (the text that defines it, its value); a CPU test checks the text is there
FLAT_STAGED = ("const size_t smem = (size_t)tab.n_live * 16 + ((size_t)tab.n_live * 4 + 15) / 16 * 16;\n    if (smem <= 96u * 1024u) {", 96 * 1024)
TRIE_STAGED = ("const size_t smem = (size_t)t.blob_bytes + sp.o_ndom;\n    if (smem <= kSpreadSmemBudget) {", 200 * 1024)
SPREAD_BUDGET = ("constexpr uint32_t kSpreadSmemBudget = 200u * 1024u;", 200 * 1024)


@pytest.fixture(scope="module")
def gp():
    from rio_rs_b200 import build

    build.build()
    import rio_rs_b200 as R

    return R


def provider(gp, policy, bits=0):
    p = gp.GpuObjectPlacement()
    p.set_solver(policy, bits)
    return p


def spread_oracle(policy, keys, seeds, w, dom, ranks, bits=12):
    return SO.assign_spread(policy, keys, seeds, w, dom, ranks, bits=bits or 12, threads=THREADS)


def domain_key(dom):
    """One value per node that is equal exactly for nodes of one domain (an unlabelled node is a domain of its own)."""
    dom = np.asarray(dom, dtype=np.uint64)
    return np.where(dom == NONE, np.uint64(1 << 32) + np.arange(len(dom), dtype=np.uint64), dom)


def check_shape(lists, w, dom):
    """Entries are live and lie in distinct domains; NONE exactly past the number of distinct live domains."""
    live = np.asarray(w) > 0
    n_dom = len(np.unique(domain_key(dom)[live]))
    R = lists.shape[1]
    assert (lists[:, min(R, n_dom):] == NONE).all()
    head = lists[:, : min(R, n_dom)]
    assert (head != NONE).all() and live[head].all()
    key = domain_key(dom)[head]
    for a in range(head.shape[1]):
        for b in range(a + 1, head.shape[1]):
            assert (key[:, a] != key[:, b]).all(), (a, b)


def layout(name, M, w, rng):
    """Labels per node (NONE = unlabelled) for the label layouts of the parity test; may set weights to 0 (not live)."""
    j = np.arange(M, dtype=np.uint32)
    if name == "racks32":
        return j // 32
    if name == "one":
        return np.full(M, 77, dtype=np.uint32)
    if name == "three":
        return (j * 7) % 3
    if name == "skewed":   # one domain holds half the weight, the rest spread over a few domains of random sizes
        dom = rng.integers(1, max(2, M // 8), size=M).astype(np.uint32)
        order = rng.permutation(M)
        half = np.cumsum(np.asarray(w, dtype=np.uint64)[order]) <= int(np.asarray(w, dtype=np.uint64).sum()) // 2
        dom[order[half]] = 0
        dom[order[: max(1, M // 50)][~half[: max(1, M // 50)]]] = NONE
        return dom
    if name == "dead":     # racks of 8 holding inactive and weight-0 nodes, one rack with no live node at all
        w[::5] = 0
        w[(j % 8) == 3] = 0
        if M >= 24:
            w[8:16] = 0
        return j // 8
    raise AssertionError(name)


def labelled_cluster(gp, oracle, policy, M, bits, name, weight_seed=7):
    p = provider(gp, policy, bits)
    addrs, seeds, w0 = oracle.synth_nodes(M, weight_seed=weight_seed)
    w = w0.copy()
    dom = layout(name, M, w, np.random.default_rng(M * 31 + len(name)))
    p.set_nodes(addrs, w)
    if M > 10:   # a weight-0 node and an inactive node are not live
        w[5] = 0
        p.node_upsert(addrs[5], 0)
        p.node_set_active(7, False)
        w[7] = 0
    if name == "dead":   # every other weight-0 node gets its weight back but leaves: both kinds of dead node sit in the racks
        for j in np.flatnonzero(w == 0)[::2]:
            p.node_upsert(addrs[j], int(w0[j]))
            p.node_set_active(int(j), False)
    p.set_node_domains(np.arange(M, dtype=np.uint32), dom)
    return p, addrs, seeds, w, dom


SHAPES = [(1, 1000, 12), (3, 2001, 12), (64, 4000, 1), (200, 4000, 5), (1024, 4000, 12), (500, 3000, 14), (5000, 3000, 12)]


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("M,n,bits", SHAPES)
@pytest.mark.parametrize("name", ["racks32", "skewed", "one", "three", "dead"])
def test_lists_equal_the_oracle(gp, oracle, policy, M, n, bits, name):
    """The shapes of test_gpu_ranked.py::test_rank_one_is_assign_batch (bits 1 and 5 put many nodes, and so several domains, in one
    bucket: the chain-skip path) under every label layout, at R = 1, 2, 3 and 8."""
    p, addrs, seeds, w, dom = labelled_cluster(gp, oracle, policy, M, bits, name)
    keys = oracle.synth_keys(n, 1 + (M % 3))
    want = spread_oracle(policy, keys, seeds, w, dom, 8, bits)
    first = p.assign_batch(keys)
    for R in (1, 2, 3, 8):
        got = p.assign_ranked_spread(keys, R)
        assert got.shape == (n, R) and got.dtype == np.uint32
        assert (got[:, 0] == first).all(), R
        assert (got == want[:, :R]).all(), (R, int((got != want[:, :R]).any(axis=1).sum()))
        check_shape(got, w, dom)
    if name == "one":
        assert (want[:, 1:] == NONE).all()
    if name == "three" and M >= 3:
        assert (want[:, 3:] == NONE).all() and (want[:, :3] != NONE).all()


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_no_labels_is_assign_ranked(gp, oracle, policy):
    """No labels, and every node labelled with a domain of its own: the spread lists equal the ranked lists bit for bit at every R."""
    M, n = 300, 20_000
    p = provider(gp, policy)
    addrs, seeds, w = oracle.synth_nodes(M)
    p.set_nodes(addrs, w)
    keys = oracle.synth_keys(n, 9)
    for labels in (None, np.arange(1000, 1000 + M, dtype=np.uint32)):
        if labels is not None:
            p.set_node_domains(np.arange(M, dtype=np.uint32), labels)
        for R in range(1, 9):
            assert (p.assign_ranked_spread(keys, R) == p.assign_ranked(keys, R)).all(), (labels is None, R)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_rank_two_is_where_a_domain_failure_sends_the_object(gp, oracle, policy):
    """A rack of 32 leaves.  For every object whose rank 1 was in it: assign_batch over the rest is its rank 2, the spread list over
    the rest is its old ranks 2..R, and rebalance_changes of the whole rack leaving moves a directory committed from rank 1 there."""
    M, n, R = 1024, 50_000, 4
    p = provider(gp, policy)
    addrs, seeds, w = oracle.synth_nodes(M)
    p.set_nodes(addrs, w)
    dom = (np.arange(M) // 32).astype(np.uint32)
    p.set_node_domains(np.arange(M, dtype=np.uint32), dom)
    keys = oracle.synth_keys(n, 5)
    lists = p.assign_ranked_spread(keys, R)
    assert (lists == spread_oracle(policy, keys, seeds, w, dom, R)).all()
    p.update_many(keys, lists[:, 0])
    for d in (5, 17):
        rack = np.flatnonzero(dom == d).astype(np.uint32)
        hit = np.isin(lists[:, 0], rack)
        assert hit.sum() > 0
        prev = np.array([p.node_state(int(j))[1] if p.node_state(int(j))[0] else 0 for j in rack], dtype=np.uint32)
        for j in rack:
            p.node_set_active(int(j), False)
        w[rack] = 0
        assert (p.assign_batch(keys)[hit] == lists[hit, 1]).all(), d
        after = p.assign_ranked_spread(keys, R)
        assert (after[hit, : R - 1] == lists[hit, 1:]).all(), d
        assert (after == spread_oracle(policy, keys, seeds, w, dom, R)).all(), d
        p.rebalance_changes(rack, prev)
        now = p.lookup_many(keys)
        assert (now[hit] == lists[hit, 1]).all(), d
        assert (now == after[:, 0]).all(), d
        lists = after


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_relabelling(gp, oracle, policy):
    """Labels set before the nodes join, changed between calls (the side table is rebuilt lazily), kept across set_nodes, node_upsert
    and node_set_active, absent on a node interned later, and cleared back to RIO_NONE."""
    M, n, R = 256, 20_000, 4
    p = provider(gp, policy)
    addrs, seeds, w = oracle.synth_nodes(M + 1)
    for a in addrs[:M]:
        p.node_intern(a)
    dom = (np.arange(M) // 16).astype(np.uint32)
    p.set_node_domains(np.arange(M, dtype=np.uint32), dom)           # before any node is live
    p.set_nodes(addrs[:M], w[:M])
    keys = oracle.synth_keys(n, 11)
    assert (p.assign_ranked_spread(keys, R) == spread_oracle(policy, keys, seeds[:M], w[:M], dom, R)).all()
    # relabel between two calls: racks of 16 -> racks of 64
    dom = (np.arange(M) // 64).astype(np.uint32)
    p.set_node_domains(np.arange(M, dtype=np.uint32), dom)
    assert (p.assign_ranked_spread(keys, R) == spread_oracle(policy, keys, seeds[:M], w[:M], dom, R)).all()
    # a partial relabel (a batch of some indices) and labels kept across membership calls
    dom[10:20] = 900
    p.set_node_domains(np.arange(10, 20, dtype=np.uint32), dom[10:20])
    p.node_set_active(12, False)
    p.node_set_active(12, True)
    p.node_upsert(addrs[13], int(w[13]))
    p.set_nodes(addrs[:M], w[:M])
    assert [p.node_domain(j) for j in (0, 12, 13, 19, 20)] == [0, 900, 900, 900, 0]
    assert (p.assign_ranked_spread(keys, R) == spread_oracle(policy, keys, seeds[:M], w[:M], dom, R)).all()
    # a node interned after the labels were set is a domain of its own
    assert p.node_upsert(addrs[M], int(w[M])) == M
    assert p.node_domain(M) == NONE
    dom2 = np.append(dom, np.uint32(NONE))
    assert (p.assign_ranked_spread(keys, R) == spread_oracle(policy, keys, seeds, w, dom2, R)).all()
    # cleared back to RIO_NONE: the ranked lists again
    p.set_node_domains(np.arange(M, dtype=np.uint32), np.full(M, NONE, dtype=np.uint32))
    assert (p.assign_ranked_spread(keys, R) == p.assign_ranked(keys, R)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_labels_leave_existing_calls_alone(gp, oracle, policy):
    """Two handles over the same nodes, one with racks labelled (and its spread side table built): assign_batch, assign_ranked, a ranked
    resident set through a change set, and a directory through rebalance_changes give the same results on both."""
    M, n, R = 512, 30_000, 3
    addrs, seeds, w = oracle.synth_nodes(M)
    keys = oracle.synth_keys(n, 13)
    ps = [provider(gp, policy) for _ in range(2)]
    for p in ps:
        p.set_nodes(addrs, w)
    ps[1].set_node_domains(np.arange(M, dtype=np.uint32), (np.arange(M) // 32).astype(np.uint32))
    ps[1].assign_ranked_spread(keys, R)
    sets = []
    for p in ps:
        p.update_many(keys, p.assign_batch(keys))
        s = p.new_set(n)
        s.load_keys(keys)
        s.assign_ranked(R)
        sets.append(s)
    assert (ps[0].assign_batch(keys) == ps[1].assign_batch(keys)).all()
    assert (ps[0].assign_ranked(keys, R) == ps[1].assign_ranked(keys, R)).all()
    changes = {3: 0, 40: 0, 41: 0, 100: 2}
    results = []
    for p, s in zip(ps, sets):
        idx = np.array(sorted(changes), dtype=np.uint32)
        prev = np.array([w[j] for j in idx], dtype=np.uint32)
        for j, nw in changes.items():
            if nw:
                p.node_upsert(addrs[j], nw)
            else:
                p.node_set_active(j, False)
        mc = s.rebalance_changes_ranked(idx, prev)
        md = p.rebalance_changes(idx, prev)
        results.append((mc, md, s.read_ranked(), s.read(), s.counters(), p.lookup_many(keys), p.assign_ranked(keys, R)))
    a, b = results
    assert a[0] == b[0] and a[1] == b[1]
    for x, y in zip(a[2:], b[2:]):
        assert (x == y).all()


FLAT_MAX_STAGED = max(m for m in range(FLAT_STAGED[1] // 16 + 1) if m * 16 + (m * 4 + 15) // 16 * 16 <= FLAT_STAGED[1])


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("side", [0, 1])
def test_both_sides_of_the_staging_threshold(gp, oracle, policy, side):
    """Flat: 16-byte records plus the 4-byte domain array against the 96 KB shared-memory limit.  HRW2: the blob plus the part of
    the side table the walk stages (the subtree weights and per-node {bucket, weight}: the bytes of the ranked walk's side table)
    against the 200 KB budget.  M sits on the last staged node count (side 0) or one past it (side 1)."""
    import test_gpu_boundaries as TB

    if policy == "hrw":
        M = FLAT_MAX_STAGED + side
    else:
        assert TB.T("rank_smem_budget") == TRIE_STAGED[1]
        M = TB.largest_staged_ranked_trie(oracle, 12, 8000) + side
    p = provider(gp, policy)
    addrs, seeds, w = oracle.synth_nodes(M)
    p.set_nodes(addrs, w)
    dom = (np.arange(M) // 32).astype(np.uint32)
    p.set_node_domains(np.arange(M, dtype=np.uint32), dom)
    keys = oracle.synth_keys(2000, 17)
    got = p.assign_ranked_spread(keys, 3)
    assert (got == spread_oracle(policy, keys, seeds, w, dom, 3)).all()
    check_shape(got, w, dom)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_extreme_weights(gp, oracle, policy):
    """Weights near 2^32 - 1, whose subtree sums need 64 bits, with one domain holding most of the weight; weight 1 beside them."""
    M, n = 96, 20_000
    p = provider(gp, policy)
    addrs, seeds, w = oracle.synth_nodes(M)
    w = w.astype(np.uint32)
    w[:12] = 0xFFFFFFFF - np.arange(12, dtype=np.uint32)    # domain 0: most of the weight
    w[40:44] = 0xFFFFFFF0                                     # heavy nodes inside another rack
    w[60:64] = 1
    p.set_nodes(addrs, w)
    dom = np.where(np.arange(M) < 12, 0, 1 + np.arange(M) // 8).astype(np.uint32)
    p.set_node_domains(np.arange(M, dtype=np.uint32), dom)
    keys = oracle.synth_keys(n, 19)
    for R in (2, 8):
        got = p.assign_ranked_spread(keys, R)
        assert (got == spread_oracle(policy, keys, seeds, w, dom, R)).all(), R
        check_shape(got, w, dom)
    assert np.isin(got[:, 0], np.arange(12)).mean() > 0.5


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_device_variant_and_bad_arguments(gp, oracle, policy):
    p = provider(gp, policy)
    L, h = p.L, p.h
    M = 256
    addrs, seeds, w = oracle.synth_nodes(M)
    p.set_nodes(addrs, w)
    dom = (np.arange(M) // 32).astype(np.uint32)
    p.set_node_domains(np.arange(M, dtype=np.uint32), dom)
    n, R = 30_001, 5
    keys = oracle.synth_keys(n, 6)
    want = p.assign_ranked_spread(keys, R)
    dk, di = C.c_void_p(), C.c_void_p()
    p._ck(L.rio_cuda_dev_alloc(h, n * 8, C.byref(dk)))
    p._ck(L.rio_cuda_dev_alloc(h, n * R * 4, C.byref(di)))
    p._ck(L.rio_cuda_memcpy_h2d(h, dk, keys.ctypes.data_as(C.c_void_p), n * 8))
    p._ck(L.rio_cuda_assign_ranked_spread_batch_dev(h, dk, n, R, di))
    got = np.empty((n, R), dtype=np.uint32)
    p._ck(L.rio_cuda_memcpy_d2h(h, got.ctypes.data_as(C.c_void_p), di, n * R * 4))
    p.sync()
    assert (got == want).all()
    out = np.empty((n, 9), dtype=np.uint32)
    for ranks in (0, 9):
        for call, kp, op in ((L.rio_cuda_assign_ranked_spread_batch, keys.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)),
                             (L.rio_cuda_assign_ranked_spread_batch_dev, dk, di)):
            assert call(h, kp, n, ranks, op) == -2
            assert b"ranks" in L.rio_cuda_last_error(h)
    for call in (L.rio_cuda_assign_ranked_spread_batch, L.rio_cuda_assign_ranked_spread_batch_dev):
        assert call(h, None, n, 2, di) == -2 and L.rio_cuda_last_error(h)
        assert call(h, dk, n, 2, None) == -2 and L.rio_cuda_last_error(h)
        assert call(h, None, 0, 2, None) == 0
    assert L.rio_cuda_assign_ranked_spread_batch(h, None, 2**62, 8, None) == -2 and b"overflow" in L.rio_cuda_last_error(h)
    with pytest.raises(gp.Unknown):
        p.assign_ranked_spread(keys, 0)
    assert p.assign_ranked_spread(np.empty(0, np.uint64), 4).shape == (0, 4)
    p._ck(L.rio_cuda_dev_free(h, dk))
    p._ck(L.rio_cuda_dev_free(h, di))
    # labels: index out of range, duplicate index, NULL arrays with k > 0; k = 0 does nothing, even with NULL arrays
    idx = np.array([1, 2], dtype=np.uint32)
    lab = np.array([5, 6], dtype=np.uint32)
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    for bad_idx in (np.array([1, M], dtype=np.uint32), np.array([3, 3], dtype=np.uint32)):
        assert L.rio_cuda_node_set_domains(h, ptr(bad_idx), ptr(lab), 2) == -2 and L.rio_cuda_last_error(h)
    assert p.node_domain(3) == 0 and p.node_domain(1) == 0   # a refused batch changes nothing
    assert L.rio_cuda_node_set_domains(h, None, ptr(lab), 2) == -2
    assert L.rio_cuda_node_set_domains(h, ptr(idx), None, 2) == -2
    assert L.rio_cuda_node_set_domains(h, None, None, 0) == 0
    d = C.c_uint32(0)
    assert L.rio_cuda_node_domain(h, M, C.byref(d)) == -2 and b"range" in L.rio_cuda_last_error(h)
    assert L.rio_cuda_node_domain(h, 0, None) == -2
    with pytest.raises(gp.Unknown):
        p.set_node_domains([1, 2], [5])
    assert (p.assign_ranked_spread(keys, R) == want).all()


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_one_million_objects_in_racks(gp, oracle, policy):
    """1 M objects x 1024 nodes in racks of 32 at R = 4, every list against the oracle on all host cores."""
    if HOSTSIM:
        pytest.skip("sized for the GPU: the host restatements take minutes at this size")
    M, n, R = 1024, 1_000_000, 4
    p = provider(gp, policy)
    addrs, seeds, w = oracle.synth_nodes(M)
    p.set_nodes(addrs, w)
    dom = (np.arange(M) // 32).astype(np.uint32)
    p.set_node_domains(np.arange(M, dtype=np.uint32), dom)
    keys = oracle.synth_keys(n, 23)
    got = p.assign_ranked_spread(keys, R)
    want = spread_oracle(policy, keys, seeds, w, dom, R)
    assert (got == want).all(), int((got != want).any(axis=1).sum())
    check_shape(got, w, dom)
    plain = p.assign_ranked(keys, 2)
    assert (dom[plain[:, 0]] == dom[plain[:, 1]]).any()   # the plain rank 2 shares rank 1's rack for some objects, the spread one never


# ---- CPU ---------------------------------------------------------------------------------------------------------------------------
SPREAD_DOUBLES = os.path.join(ROOT, "tests", "cpp", "hostsim", "spread_launchers.cpp")
RANKED_DOUBLES = [os.path.join(ROOT, "tests", "cpp", "hostsim", f) for f in ("ranked_launchers.cpp", "change_launchers.cpp",
                                                                               "ranked_change_launchers.cpp")]


def test_staging_thresholds_are_where_the_launchers_define_them():
    src = open(os.path.join(CSRC, "k_spread.cu")).read()
    assert FLAT_STAGED[0] in src and TRIE_STAGED[0] in src and SPREAD_BUDGET[0] in src and SPREAD_BUDGET[1] == TRIE_STAGED[1]
    assert FLAT_MAX_STAGED == 4915


def test_the_spread_doubles_cover_every_spread_launcher():
    decl = set(re.findall(r"\b(launch_[a-z0-9_]+)\s*\(", open(os.path.join(CSRC, "k_spread.cuh")).read()))
    have = set(re.findall(r"^void\s+([a-z0-9_]+)\s*\(", open(SPREAD_DOUBLES).read(), flags=re.M))
    assert len(decl) == 2 and decl <= have, decl - have


def _hostsim_library(HS, name, doubles):
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, name)
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + doubles + ["-o", so, "-ldl", "-lpthread"])
    return so


def test_spread_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + the ranked, change-set,
    ranked-set and spread doubles)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_spread.so", RANKED_DOUBLES + [SPREAD_DOUBLES])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=3000, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 84 and "failed" not in r.stdout, tail


def test_spread_calls_report_an_error_where_the_kernels_are_not_linked():
    """The engine's host code built with the ranked launchers but WITHOUT the spread ones loads, refuses the spread call with
    RIO_ERR_UPSTREAM and a message, and still serves the labels and assign_ranked."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_nospread.so", RANKED_DOUBLES)
    code = (
        "import sys, numpy as np\n"
        "from rio_rs_b200 import _native as N\n"
        "N.library_path = lambda: sys.argv[1]\n"
        "import rio_rs_b200 as R\n"
        "p = R.GpuObjectPlacement()\n"
        "p.set_nodes(['10.0.0.%d:5000' % j for j in range(8)])\n"
        "p.set_node_domains(np.arange(8), np.arange(8) // 2)\n"
        "assert p.node_domain(5) == 2\n"
        "keys = np.arange(100, dtype=np.uint64)\n"
        "lists = p.assign_ranked(keys, 3)\n"
        "assert (lists[:, 0] == p.assign_batch(keys)).all()\n"
        "try:\n"
        "    p.assign_ranked_spread(keys, 2)\n"
        "except R.Upstream as e:\n"
        "    assert 'spread kernels' in str(e), e\n"
        "    print('refused ok')\n"
    )
    r = subprocess.run([sys.executable, "-c", code, so], capture_output=True, text=True, timeout=300, cwd=HS.ROOT)
    assert r.returncode == 0 and "refused ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

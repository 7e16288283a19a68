"""Ranked placement (DESIGN.md 3.9): each object's first R distinct nodes under the handle's policy, through the C ABI, compared
list for list with the CPU oracle (tests/ranked_oracle.c: repeated masked assignment per object, the definition itself) under
both policies: rank 1 is assign_batch bit for bit, the lists are distinct and padded with RIO_NONE past the live set, and rank 2
is where a LEAVE of rank 1 sends the object.

The last test runs this module's GPU bodies, unchanged, against the engine's host logic compiled with g++ (the host-sim library
of tests/test_engine_host_sim.py): argument checks, the lazy side-table build and the table changes between ranked calls are
exercised on a box without a GPU; the kernels themselves are proven only on the GPU."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import ranked_oracle as RO

NONE = 0xFFFFFFFF
POLICIES = ["hrw", "hrw2"]


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


def oracle_lists(policy, keys, seeds, w, ranks, bits=12):
    return RO.assign_ranked(policy, keys, seeds, w, ranks, bits=bits, threads=os.cpu_count() or 8)


def assert_distinct(lists):
    for a in range(lists.shape[1]):
        for b in range(a + 1, lists.shape[1]):
            assert ((lists[:, a] != lists[:, b]) | (lists[:, a] == NONE)).all(), (a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("M,n,bits,uniform", [(1, 1000, 12, False), (3, 5001, 12, False), (64, 20_000, 1, False), (200, 50_001, 5, False),
                                              (1024, 50_000, 12, False), (1024, 50_000, 12, True), (500, 30_000, 14, False),
                                              (5000, 20_000, 12, False)])
def test_rank_one_is_assign_batch(gp, oracle, policy, M, n, bits, uniform):
    """The shapes of test_gpu_hrw2.py::test_assign_matches_oracle: bits 1 and 5 put many nodes in one bucket (long chains), 14 is the
    deepest trie, M = 5000 has a chain in most buckets; a weight-0 node and an inactive node are not live."""
    p = provider(gp, policy, bits)
    addrs, seeds, w = oracle.synth_nodes(M, uniform=uniform)
    if M > 10:
        w[5] = 0
    p.set_nodes(addrs, w)
    if M > 10:
        p.node_set_active(7, False)
        w[7] = 0
    keys = oracle.synth_keys(n, 1 + (M % 3))
    got = p.assign_ranked(keys, 3)
    assert got.shape == (n, 3) and got.dtype == np.uint32
    assert (got[:, 0] == p.assign_batch(keys)).all()
    assert (got == oracle_lists(policy, keys, seeds, w, 3, bits or 12)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_table_too_large_for_shared_memory(gp, oracle, policy):
    """70 000 live nodes: the tables are read through the read-only path instead of shared memory."""
    M = 70_000
    p = provider(gp, policy)
    addrs, seeds, w = oracle.synth_nodes(M)
    p.set_nodes(addrs, w)
    keys = oracle.synth_keys(4000, 2)
    got = p.assign_ranked(keys, 3)
    assert (got[:, 0] == p.assign_batch(keys)).all()
    assert (got == oracle_lists(policy, keys, seeds, w, 3)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("ranks", [1, 2, 3, 8])
def test_full_lists_equal_the_oracle(gp, oracle, policy, ranks):
    M, n = 1024, 200_000
    p = provider(gp, policy)
    addrs, seeds, w = oracle.synth_nodes(M)
    p.set_nodes(addrs, w)
    keys = oracle.synth_keys(n, 3)
    got = p.assign_ranked(keys, ranks)
    assert (got == oracle_lists(policy, keys, seeds, w, ranks)).all()
    assert (got[:, 0] == p.assign_batch(keys)).all()
    assert (got != NONE).all()
    assert_distinct(got)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("M", [0, 1, 3])
def test_lists_longer_than_the_live_set_are_padded(gp, oracle, policy, M):
    p = provider(gp, policy)
    addrs, seeds, w = oracle.synth_nodes(max(M, 1))
    if M:
        p.set_nodes(addrs[:M], w[:M])
    keys = oracle.synth_keys(5000, 4)
    got = p.assign_ranked(keys, 8)
    assert (got[:, M:] == NONE).all()
    assert (np.sort(got[:, :M], axis=1) == np.arange(M, dtype=np.uint32)).all()   # every live node once, in some order
    if M:
        assert (got == oracle_lists(policy, keys, seeds[:M], w[:M], 8)).all()


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_rank_two_is_where_a_leave_sends_the_object(gp, oracle, policy):
    """Three nodes leave one after another.  Before each leave the lists are read over the live set of that moment; after it, every
    object that was recorded on the leaving node is recorded on its rank-2 node."""
    M, n = 64, 100_000
    p = provider(gp, policy)
    addrs, seeds, w = oracle.synth_nodes(M)
    p.set_nodes(addrs, w)
    keys = oracle.synth_keys(n, 5)
    p.update_many(keys, p.assign_batch(keys))
    for x in (17, 3, 40):
        lists = p.assign_ranked(keys, 2)
        assert (lists == oracle_lists(policy, keys, seeds, w, 2)).all(), x
        on_x = p.lookup_many(keys) == x
        assert on_x.sum() > 0 and (lists[on_x, 0] == x).all()
        p.node_set_active(x, False)
        w[x] = 0
        p.rebalance("leave", x)
        after = p.lookup_many(keys)
        assert (after[on_x] == lists[on_x, 1]).all(), x
        assert (after != x).all()


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("split_classes", [False, True])
def test_twin_seeds_are_ordered_like_the_oracle(gp, oracle, policy, split_classes):
    """Nodes that share a seed hash every object alike: under the flat policy their u ties exactly (and with equal weights their
    scores), so the list order comes from the tie rule alone -- inside one weight class, and across classes when the table is built
    with one class per node."""
    from rio_rs_b200 import _native as N

    M = 150
    p = provider(gp, policy)
    addrs, seeds, w = oracle.synth_nodes(M, uniform=True)
    seeds = seeds.copy()
    p.set_nodes(addrs, w)
    for a, b in [(3, 44), (10, 11), (100, 149), (0, M - 1)]:
        seeds[b] = seeds[a]
        p.dev_set_node_seed(b, int(seeds[a]))
    seeds[7] = seeds[5] = seeds[6]
    p.dev_set_node_seed(5, int(seeds[6]))
    p.dev_set_node_seed(7, int(seeds[6]))
    if split_classes:
        p.dev_set_table_options(N.DEV_SPLIT_CLASSES)
    keys = oracle.synth_keys(60_000, 7)
    got = p.assign_ranked(keys, 4)
    assert (got == oracle_lists(policy, keys, seeds, w, 4)).all()
    assert (got[:, 0] == p.assign_batch(keys)).all()
    assert_distinct(got)
    if policy == "hrw":   # the twins really met: the triple 5, 6, 7 fills three ranks in a row whenever one of them is first
        first = np.isin(got[:, 0], [5, 6, 7])
        assert first.sum() > 0 and (got[first, 0] == 5).all() and (got[first, 1] == 6).all() and (got[first, 2] == 7).all()


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_device_variant_and_bad_arguments(gp, oracle, policy):
    p = provider(gp, policy)
    L, h = p.L, p.h
    addrs, seeds, w = oracle.synth_nodes(256)
    p.set_nodes(addrs, w)
    n, R = 30_001, 5
    keys = oracle.synth_keys(n, 6)
    want = p.assign_ranked(keys, R)
    dk, di = C.c_void_p(), C.c_void_p()
    p._ck(L.rio_cuda_dev_alloc(h, n * 8, C.byref(dk)))
    p._ck(L.rio_cuda_dev_alloc(h, n * R * 4, C.byref(di)))
    p._ck(L.rio_cuda_memcpy_h2d(h, dk, keys.ctypes.data_as(C.c_void_p), n * 8))
    p._ck(L.rio_cuda_assign_ranked_batch_dev(h, dk, n, R, di))
    got = np.empty((n, R), dtype=np.uint32)
    p._ck(L.rio_cuda_memcpy_d2h(h, got.ctypes.data_as(C.c_void_p), di, n * R * 4))
    p.sync()
    assert (got == want).all()
    # a table change between two ranked calls: the side table follows it
    p.node_set_active(9, False)
    w[9] = 0
    p._ck(L.rio_cuda_assign_ranked_batch_dev(h, dk, n, R, di))
    p._ck(L.rio_cuda_memcpy_d2h(h, got.ctypes.data_as(C.c_void_p), di, n * R * 4))
    p.sync()
    assert (got == oracle_lists(policy, keys, seeds, w, R)).all()
    out = np.empty((n, 9), dtype=np.uint32)
    for ranks in (0, 9):
        for call, kp, op in ((L.rio_cuda_assign_ranked_batch, keys.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p)),
                             (L.rio_cuda_assign_ranked_batch_dev, dk, di)):
            assert call(h, kp, n, ranks, op) == -2
            assert b"ranks" in L.rio_cuda_last_error(h)
    for call in (L.rio_cuda_assign_ranked_batch, L.rio_cuda_assign_ranked_batch_dev):
        assert call(h, None, n, 2, di) == -2 and L.rio_cuda_last_error(h)
        assert call(h, dk, n, 2, None) == -2 and L.rio_cuda_last_error(h)
    assert L.rio_cuda_assign_ranked_batch(h, None, 2**62, 8, None) == -2 and b"overflow" in L.rio_cuda_last_error(h)
    with pytest.raises(gp.Unknown):
        p.assign_ranked(keys, 0)
    assert p.assign_ranked(np.empty(0, np.uint64), 4).shape == (0, 4)
    p._ck(L.rio_cuda_dev_free(h, dk))
    p._ck(L.rio_cuda_dev_free(h, di))


RANKED_DOUBLES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "hostsim", "ranked_launchers.cpp")


def test_the_ranked_doubles_cover_every_ranked_launcher():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    decl = set(re.findall(r"\b(launch_[a-z0-9_]+)\s*\(", open(os.path.join(root, "rio_rs_b200", "csrc", "k_ranked.cuh")).read()))
    have = set(re.findall(r"^void\s+([a-z0-9_]+)\s*\(", open(RANKED_DOUBLES).read(), flags=re.M))
    assert decl and decl <= have, decl - have


def test_ranked_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + the ranked doubles)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, "librio_cuda_hostsim_ranked.so")
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + [RANKED_DOUBLES, "-o", so, "-ldl", "-lpthread"])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1200, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 40 and "failed" not in r.stdout, tail


def test_ranked_calls_report_an_error_where_the_kernels_are_not_linked():
    """The engine's host code built WITHOUT the ranked launchers (the host-sim library of tests/test_engine_host_sim.py) still loads,
    every other call works, and the ranked entry points answer RIO_ERR_UPSTREAM with a message instead of computing anything."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, "librio_cuda_hostsim_unranked.so")
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + ["-o", so, "-ldl", "-lpthread"])
    code = (
        "import sys, numpy as np\n"
        "from rio_rs_b200 import _native as N\n"
        "N.library_path = lambda: sys.argv[1]\n"
        "import rio_rs_b200 as R\n"
        "p = R.GpuObjectPlacement()\n"
        "p.set_nodes(['10.0.0.%d:5000' % j for j in range(8)])\n"
        "keys = np.arange(100, dtype=np.uint64)\n"
        "assert (p.assign_batch(keys) < 8).all()\n"
        "try:\n"
        "    p.assign_ranked(keys, 2)\n"
        "except R.Upstream as e:\n"
        "    assert 'ranked kernels' in str(e), e\n"
        "    print('refused ok')\n"
    )
    r = subprocess.run([sys.executable, "-c", code, so], capture_output=True, text=True, timeout=300, cwd=HS.ROOT)
    assert r.returncode == 0 and "refused ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

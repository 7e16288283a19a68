"""Failure-domain ranked placement under the affinity cost (DESIGN.md 3.14): each object's R lowest-cost live nodes in R distinct
domains, through the C ABI, on the tensor-core path (k_affinity_wgmma_spread + k_affinity_resolve_spread) and on the CUDA-core path
(k_assign_affinity_ranked with SPREAD).  Rank 1 is assign_batch(obj_feats) bit for bit; the whole list is checked with the conditioned
fp64 rule of tests/affinity_spread_oracle.py; rank 2 is where the object goes when rank 1's whole domain leaves.

The CPU-only tests at the end run this module's GPU bodies, unchanged, against the engine's host logic compiled with g++ (the
host-sim library of tests/test_engine_host_sim.py plus tests/cpp/hostsim/affinity_ranked_launchers.cpp and
affinity_spread_launchers.cpp).  There the tensor-core path is never selected; the kernels themselves are proven only on the GPU."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import affinity_ranked_oracle as AO
import affinity_spread_oracle as SO

NONE = SO.NONE
VARIANTS = ["umma", "ffma"]


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


def feats(n, M, K, seed=0):
    return (np.random.default_rng(11 + seed).uniform(-1, 1, (n, K)).astype(np.float32),
            np.random.default_rng(13 + seed).uniform(-1, 1, (M, K)).astype(np.float32))


def handle(gp, oracle, fn, w=None, labels=None):
    p = gp.GpuObjectPlacement()
    addrs, _, _ = oracle.synth_nodes(max(len(fn), 1))
    p.set_nodes(addrs[:len(fn)], w, fn)
    if labels is not None:
        p.set_node_domains(np.arange(len(fn), dtype=np.uint32), labels)
    return p


def layout(name, M):
    """racks: 32 contiguous racks (fewer when M < 32); zones: 4 zones, nodes dealt round robin."""
    j = np.arange(M, dtype=np.uint32)
    if name == "racks":
        return j // max(1, -(-M // 32))
    return j % 4


def host_sim(p):
    return p.device_info()["name"].startswith("host-sim")


def tensor_cores(p, var, K, n_live):
    padded = 64 if n_live <= 64 else (n_live + 255) // 256 * 256
    return var == "umma" and K == 16 and 0 < padded <= 2304 and not host_sim(p)


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
@pytest.mark.parametrize("lay", ["racks", "zones"])
@pytest.mark.parametrize("K,M,n", [(16, 1024, 20000), (16, 66, 3001), (16, 67, 3001), (16, 258, 3001), (16, 259, 3001), (16, 2306, 3001),
                                   (16, 2307, 3001), (8, 64, 3000), (5, 9, 1000)])
def test_rank_one_is_assign_batch(gp, oracle, K, M, n, lay, var):
    """Node 3 has weight 0 and node M - 2 is inactive: 64 / 65, 256 / 257 and 2304 / 2305 live nodes sit on either side of a padding
    step of the tensor-core path.  R = 3 (a list of 4 on the tensor cores) under racks, R = 8 under 4 zones (NONE past rank 4)."""
    fo, fn = feats(n, M, K)
    w = np.ones(M, dtype=np.uint32)
    w[3] = 0
    labels = layout(lay, M)
    p = handle(gp, oracle, fn, w, labels)
    p.node_set_active(M - 2, False)
    live = w > 0
    live[M - 2] = False
    R = 3 if lay == "racks" else 8
    with variant(var):
        got = p.assign_ranked_affinity_spread(fo, R)
        one = p.assign_batch(obj_feats=fo)
    assert got.shape == (n, R) and got.dtype == np.uint32
    assert (got[:, 0] == one).all()
    SO.check(got, fo, fn, live, labels)


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
@pytest.mark.parametrize("labels", ["none", "unique"])
@pytest.mark.parametrize("M,R", [(1024, 1), (1024, 2), (1024, 3), (1024, 8), (64, 5)])
def test_without_shared_domains_it_is_the_ranked_list(gp, oracle, M, R, labels, var):
    """No labels, or every label distinct: the CUDA-core list is assign_ranked_affinity's bit for bit.  On the tensor cores the
    candidates differ (RT columns instead of RT groups of 8), so the lists agree but for near-ties."""
    fo, fn = feats(100_000 if M == 1024 else 20_000, M, 16)
    p = handle(gp, oracle, fn, labels=None if labels == "none" else np.arange(M, dtype=np.uint32) * 7 + 1)
    with variant(var):
        got = p.assign_ranked_affinity_spread(fo, R)
        want = p.assign_ranked_affinity(fo, R)
    if tensor_cores(p, var, 16, M):
        SO.check(got[:20000], fo[:20000], fn, np.ones(M, bool), None)
        assert (got == want).all(axis=1).mean() >= 0.9999
        assert (got[:, 0] == want[:, 0]).all()
    else:
        assert (got == want).all()


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
def test_lists_past_the_live_domains_are_padded(gp, oracle, var):
    M, n = 256, 5000
    fo, fn = feats(n, M, 16)
    live = np.ones(M, bool)
    cases = {
        "one domain": (np.full(M, 5, np.uint32), 1),
        "three domains": (np.arange(M, dtype=np.uint32) % 3 + 10, 3),
        # RIO_NONE: every such node is a domain of its own (two of them here, beside two labelled domains)
        "unlabelled nodes": (np.where(np.arange(M) < 2, NONE, np.arange(M) % 2 + 100).astype(np.uint32), 4),
    }
    for name, (labels, n_dom) in cases.items():
        p = handle(gp, oracle, fn, labels=labels)
        with variant(var):
            got = p.assign_ranked_affinity_spread(fo, 8)
            one = p.assign_batch(obj_feats=fo)
        assert (got[:, n_dom:] == NONE).all(), name
        assert (got[:, :n_dom] != NONE).all(), name
        assert (got[:, 0] == one).all(), name
        SO.check(got, fo, fn, live, labels)
    # the labels of nodes that are not live are ignored: node 7 alone in domain 9, then inactive; weight-0 node 8 alone in domain 10
    labels = np.zeros(M, np.uint32)
    labels[7], labels[8] = 9, 10
    w = np.ones(M, np.uint32)
    w[8] = 0
    p = handle(gp, oracle, fn, w, labels)
    p.node_set_active(7, False)
    with variant(var):
        got = p.assign_ranked_affinity_spread(fo, 4)
    assert (got[:, 1:] == NONE).all() and (got[:, 0] != NONE).all()
    live = w > 0
    live[7] = False
    SO.check(got, fo, fn, live, labels)


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
def test_rank_two_is_where_a_rack_leave_sends_the_object(gp, oracle, var):
    """The most frequent rank-1 rack leaves as a whole.  assign_batch(obj_feats) then sends its objects to their old rank 2, and keeps
    every other object, wherever the fp64 order over the new live set is clear."""
    M, n = 1024, 100_000
    fo, fn = feats(n, M, 16)
    labels = layout("racks", M)
    p = handle(gp, oracle, fn, labels=labels)
    with variant(var):
        lists = p.assign_ranked_affinity_spread(fo, 2)
        before = p.assign_batch(obj_feats=fo)
        assert (lists[:, 0] == before).all()
        rack = int(np.bincount(labels[before]).argmax())
        on_rack = labels[before] == rack
        for j in np.flatnonzero(labels == rack):
            p.node_set_active(int(j), False)
        after = p.assign_batch(obj_feats=fo)
    live = labels != rack
    assert live[after].all()
    want_idx, want_cost = AO.ranked(fo, fn, live, 2)
    AO.check(after[:, None], fo, fn, live, (want_idx, want_cost))
    tol = AO.tau(fo, fn, after[:, None])[:, 0] + AO.tau(fo, fn, want_idx[:, :1])[:, 0]
    clear = want_cost[:, 1] - want_cost[:, 0] > tol
    assert clear[on_rack].mean() > 0.99
    assert (after[on_rack & clear] == lists[on_rack & clear, 1]).all()
    assert (after[~on_rack & clear] == before[~on_rack & clear]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
def test_exact_ties(gp, oracle, var):
    """Identical feature rows have identical fp32 costs.  Twins in one domain: the lower index is listed and its twin never is.  Twins
    in two domains: the lower index first and the twin right after it.  Pairs inside one group of 8 (10, 11 / 20, 21) and across groups
    (3, 44 / 5, 50)."""
    M, n, R = 64, 60_000, 4
    fo, fn = feats(n, M, 16)
    labels = np.arange(M, dtype=np.uint32) // 4 + 100   # 16 racks of 4
    same, apart = [(10, 11), (3, 44)], [(20, 21), (5, 50)]
    for a, b in same + apart:
        fn[b] = fn[a]
    for a, b in same:
        labels[b] = labels[a]
    for a, b in apart:   # each alone in its domain, so that a listed twin is never hidden by a better rack mate
        labels[a], labels[b] = 800 + a, 900 + b
    p = handle(gp, oracle, fn, labels=labels)
    with variant(var):
        got = p.assign_ranked_affinity_spread(fo, R)
        assert (got[:, 0] == p.assign_batch(obj_feats=fo)).all()
    SO.check(got, fo, fn, np.ones(M, bool), labels)
    for a, b in same:
        assert not (got == b).any(), (a, b)
        assert (got[:, 0] == a).sum() > 100, (a, b)   # the ties really met
    for a, b in apart:
        ra, rb = got == a, got == b
        assert (ra[:, :-1] == rb[:, 1:]).all(), (a, b)
        assert not rb[:, 0].any(), (a, b)
        assert (got[:, 0] == a).sum() > 100, (a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
def test_relabel_between_calls(gp, oracle, var):
    """Labels do not change the table; a relabel between two calls is still honoured by the next one."""
    M, n, R = 512, 30_000, 4
    fo, fn = feats(n, M, 16)
    labels = layout("racks", M)
    p = handle(gp, oracle, fn, labels=labels)
    with variant(var):
        first = p.assign_ranked_affinity_spread(fo, R)
        SO.check(first, fo, fn, np.ones(M, bool), labels)
        labels = layout("zones", M)
        p.set_node_domains(np.arange(M, dtype=np.uint32), labels)
        second = p.assign_ranked_affinity_spread(fo, R)
        one = p.assign_batch(obj_feats=fo)
    assert (second[:, 0] == one).all() and (first[:, 0] == one).all()
    SO.check(second, fo, fn, np.ones(M, bool), labels)
    assert (first != second).any()


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
def test_labels_change_no_other_call(gp, oracle, var):
    M, n = 1024, 50_000
    fo, fn = feats(n, M, 16)
    p = handle(gp, oracle, fn)
    with variant(var):
        a0, r0 = p.assign_batch(obj_feats=fo), p.assign_ranked_affinity(fo, 4)
        p.set_node_domains(np.arange(M, dtype=np.uint32), layout("racks", M))
        p.assign_ranked_affinity_spread(fo, 4)
        a1, r1 = p.assign_batch(obj_feats=fo), p.assign_ranked_affinity(fo, 4)
    assert a0.tobytes() == a1.tobytes() and r0.tobytes() == r1.tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
@pytest.mark.parametrize("K,M", [(16, 1024), (16, 64), (16, 2400), (8, 64)])
def test_which_kernels_ran(gp, oracle, K, M, var):
    """The tensor-core path is two launches (k_affinity_wgmma_spread + k_affinity_resolve_spread), the CUDA-core path one."""
    fo, fn = feats(2000, M, K)
    p = handle(gp, oracle, fn, labels=layout("racks", M))
    with variant(var):
        p.assign_ranked_affinity_spread(fo, 2)   # the table and domain uploads happen here, not in the counted call
        l0 = p.launch_count()
        p.assign_ranked_affinity_spread(fo, 2)
        launches = p.launch_count() - l0
    assert launches == (2 if tensor_cores(p, var, K, M) else 1), launches


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
def test_device_variant_and_bad_arguments(gp, oracle, var):
    M, n, R = 256, 30_001, 5
    fo, fn = feats(n, M, 16)
    labels = layout("racks", M)
    p = handle(gp, oracle, fn, labels=labels)
    L, h = p.L, p.h
    with variant(var):
        want = p.assign_ranked_affinity_spread(fo, R)
        df, di = C.c_void_p(), C.c_void_p()
        p._ck(L.rio_cuda_dev_alloc(h, n * 16 * 4, C.byref(df)))
        p._ck(L.rio_cuda_dev_alloc(h, n * R * 4, C.byref(di)))
        p._ck(L.rio_cuda_memcpy_h2d(h, df, fo.ctypes.data_as(C.c_void_p), n * 16 * 4))
        got = np.empty((n, R), dtype=np.uint32)
        for _ in range(2):   # two calls: identical bytes
            p._ck(L.rio_cuda_assign_ranked_affinity_spread_batch_dev(h, df, n, R, di))
            p._ck(L.rio_cuda_memcpy_d2h(h, got.ctypes.data_as(C.c_void_p), di, n * R * 4))
            p.sync()
            assert (got == want).all()
        # a table change between two calls: the lists follow it
        p.node_set_active(9, False)
        live = np.ones(M, bool)
        live[9] = False
        p._ck(L.rio_cuda_assign_ranked_affinity_spread_batch_dev(h, df, n, R, di))
        p._ck(L.rio_cuda_memcpy_d2h(h, got.ctypes.data_as(C.c_void_p), di, n * R * 4))
        p.sync()
        assert (got != 9).all() and (got[:, 0] == p.assign_batch(obj_feats=fo)).all()
        SO.check(got, fo, fn, live, labels)
        out = np.empty((n, 9), dtype=np.uint32)
        fp = fo.ctypes.data_as(C.c_void_p)
        for ranks in (0, 9):
            for call, f, o in ((L.rio_cuda_assign_ranked_affinity_spread_batch, fp, out.ctypes.data_as(C.c_void_p)),
                               (L.rio_cuda_assign_ranked_affinity_spread_batch_dev, df, di)):
                assert call(h, f, n, ranks, o) == -2
                assert b"ranks" in L.rio_cuda_last_error(h)
        for call in (L.rio_cuda_assign_ranked_affinity_spread_batch, L.rio_cuda_assign_ranked_affinity_spread_batch_dev):
            assert call(h, None, n, 2, di) == -2 and L.rio_cuda_last_error(h)
            assert call(h, df, n, 2, None) == -2 and L.rio_cuda_last_error(h)
            assert call(h, None, 0, 2, None) == 0
        assert L.rio_cuda_assign_ranked_affinity_spread_batch(h, None, 2**62, 8, None) == -2 and b"overflow" in L.rio_cuda_last_error(h)
        with pytest.raises(gp.Unknown):
            p.assign_ranked_affinity_spread(fo, 0)
        assert p.assign_ranked_affinity_spread(np.empty((0, 16), np.float32), 4).shape == (0, 4)
        p._ck(L.rio_cuda_dev_free(h, df))
        p._ck(L.rio_cuda_dev_free(h, di))
    # a handle without node features
    q = gp.GpuObjectPlacement()
    addrs, _, _ = oracle.synth_nodes(8)
    q.set_nodes(addrs)
    for call in (q.L.rio_cuda_assign_ranked_affinity_spread_batch, q.L.rio_cuda_assign_ranked_affinity_spread_batch_dev):
        assert call(q.h, fp, 100, 2, out.ctypes.data_as(C.c_void_p)) == -2
        assert b"needs node features" in q.L.rio_cuda_last_error(q.h)


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
def test_one_million_objects_in_32_racks(gp, oracle, var):
    """1 M objects x 1024 nodes in 32 racks at R = 8 (50 k objects on the host-sim, whose doubles sort every object's nodes); the
    first 200 k lists are checked with the oracle."""
    M, R = 1024, 8
    p0 = gp.GpuObjectPlacement()
    n = 50_000 if host_sim(p0) else 1_000_000
    fo, fn = feats(n, M, 16, seed=5)
    labels = layout("racks", M)
    p = handle(gp, oracle, fn, labels=labels)
    with variant(var):
        got = p.assign_ranked_affinity_spread(fo, R)
        one = p.assign_batch(obj_feats=fo)
    assert (got[:, 0] == one).all()
    assert (got != NONE).all()
    SO.check(got[:200_000], fo[:200_000], fn, np.ones(M, bool), labels)


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DOUBLES = os.path.join(ROOT, "tests", "cpp", "hostsim", "affinity_spread_launchers.cpp")
RANKED_DOUBLES = os.path.join(ROOT, "tests", "cpp", "hostsim", "affinity_ranked_launchers.cpp")


def test_the_doubles_cover_every_affinity_spread_launcher():
    decl = set(re.findall(r"\b(launch_[a-z0-9_]+)\s*\(", open(os.path.join(ROOT, "rio_rs_b200", "csrc", "k_affinity_spread.cuh")).read()))
    have = set(re.findall(r"^(?:void|cudaError_t)\s+([a-z0-9_]+)\s*\(", open(DOUBLES).read(), flags=re.M))
    assert decl and decl <= have, decl - have


def _hostsim_library(HS, name, doubles):
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, name)
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + doubles + ["-o", so, "-ldl", "-lpthread"])
    return so


def test_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + both affinity doubles)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_affinity_spread.so", [RANKED_DOUBLES, DOUBLES])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 70 and "failed" not in r.stdout, tail


def test_calls_report_an_error_where_the_kernels_are_not_linked():
    """The engine's host code built WITHOUT the failure-domain affinity launchers still loads, assign_ranked_affinity works, and both
    failure-domain affinity entry points answer RIO_ERR_UPSTREAM with a message instead of computing anything."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_no_affinity_spread.so", [RANKED_DOUBLES])
    code = (
        "import sys, ctypes as C, numpy as np\n"
        "from rio_rs_b200 import _native as N\n"
        "N.library_path = lambda: sys.argv[1]\n"
        "import rio_rs_b200 as R\n"
        "p = R.GpuObjectPlacement()\n"
        "fn = np.random.default_rng(1).uniform(-1, 1, (8, 16)).astype(np.float32)\n"
        "fo = np.random.default_rng(2).uniform(-1, 1, (100, 16)).astype(np.float32)\n"
        "p.set_nodes(['10.0.0.%d:5000' % j for j in range(8)], None, fn)\n"
        "p.set_node_domains(np.arange(8, dtype=np.uint32), np.arange(8, dtype=np.uint32) // 2)\n"
        "assert (p.assign_ranked_affinity(fo, 2)[:, 0] == p.assign_batch(obj_feats=fo)).all()\n"
        "try:\n"
        "    p.assign_ranked_affinity_spread(fo, 2)\n"
        "    raise SystemExit('computed without kernels')\n"
        "except R.Upstream as e:\n"
        "    assert 'failure-domain affinity kernels' in str(e), e\n"
        "d = C.c_void_p()\n"
        "p._ck(p.L.rio_cuda_dev_alloc(p.h, 100 * 16 * 4, C.byref(d)))\n"
        "assert p.L.rio_cuda_assign_ranked_affinity_spread_batch_dev(p.h, d, 100, 2, d) == -1\n"
        "assert b'failure-domain affinity kernels' in p.L.rio_cuda_last_error(p.h)\n"
        "print('refused ok')\n"
    )
    r = subprocess.run([sys.executable, "-c", code, so], capture_output=True, text=True, timeout=300, cwd=HS.ROOT)
    assert r.returncode == 0 and "refused ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

"""Ranked placement under the affinity cost (DESIGN.md 3.9): each object's R lowest-cost live nodes, through the C ABI, on the
tensor-core path (k_affinity_wgmma_ranked + k_affinity_resolve_ranked) and on the CUDA-core path (k_assign_affinity_ranked).  Rank 1
is assign_batch(obj_feats) bit for bit; the whole list is compared with the fp64 oracle of tests/affinity_ranked_oracle.py under its
condition-aware tolerance; rank 2 is where a leave of rank 1 sends the object.

The CPU-only tests at the end run this module's GPU bodies, unchanged, against the engine's host logic compiled with g++ (the
host-sim library of tests/test_engine_host_sim.py plus tests/cpp/hostsim/affinity_ranked_launchers.cpp).  There the tensor-core path
is never selected; the kernels themselves are proven only on the GPU."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import affinity_ranked_oracle as AO

NONE = AO.NONE
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


def feats(n, M, K):
    return (np.random.default_rng(11).uniform(-1, 1, (n, K)).astype(np.float32),
            np.random.default_rng(13).uniform(-1, 1, (M, K)).astype(np.float32))


def handle(gp, oracle, fn, w=None):
    p = gp.GpuObjectPlacement()
    addrs, _, _ = oracle.synth_nodes(max(len(fn), 1))
    p.set_nodes(addrs[:len(fn)], w, fn)
    return p


def tensor_cores(p, var, K, n_live):
    padded = 64 if n_live <= 64 else (n_live + 255) // 256 * 256
    # the host-sim build of the engine (tests/test_engine_host_sim.py) restates no tensor-core kernel
    return var == "umma" and K == 16 and 0 < padded <= 2304 and not p.device_info()["name"].startswith("host-sim")


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
@pytest.mark.parametrize("K,M,n", [(16, 1024, 60000), (16, 37, 5001), (16, 64, 999), (16, 65, 7000), (16, 300, 20000), (16, 2000, 4000), (16, 2400, 3000),
                                   (16, 66, 3001), (16, 67, 3001), (16, 258, 3001), (16, 259, 3001), (16, 2306, 3001), (16, 2307, 3001),
                                   (8, 64, 3000), (5, 9, 1000)])
def test_rank_one_is_assign_batch(gp, oracle, K, M, n, var):
    """The shapes of test_gpu_parity.py::test_affinity_cost_argmin; node 3 has weight 0 and node M - 2 is inactive, so neither is
    live: 64 / 65, 256 / 257 and 2304 / 2305 live nodes sit on either side of a padding step of the tensor-core path."""
    fo, fn = feats(n, M, K)
    w = np.ones(M, dtype=np.uint32)
    w[3] = 0
    p = handle(gp, oracle, fn, w)
    p.node_set_active(M - 2, False)
    live = w > 0
    live[M - 2] = False
    with variant(var):
        got = p.assign_ranked_affinity(fo, 4)
        one = p.assign_batch(obj_feats=fo)
    assert got.shape == (n, 4) and got.dtype == np.uint32
    assert (got[:, 0] == one).all()
    AO.check(got, fo, fn, live)


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
@pytest.mark.parametrize("K,M", [(16, 1024), (16, 64), (16, 2400), (8, 64)])
def test_which_kernels_ran(gp, oracle, K, M, var):
    """The tensor-core path is two launches (k_affinity_wgmma_ranked + k_affinity_resolve_ranked), the CUDA-core path one."""
    fo, fn = feats(2000, M, K)
    p = handle(gp, oracle, fn)
    with variant(var):
        p.assign_ranked_affinity(fo, 2)   # the table upload happens here, not in the counted call
        l0 = p.launch_count()
        p.assign_ranked_affinity(fo, 2)
        launches = p.launch_count() - l0
    assert launches == (2 if tensor_cores(p, var, K, M) else 1), launches


_FULL = {}


def full_case(gp, oracle, M, var):
    if (M, var) not in _FULL:
        fo, fn = feats(100_000, M, 16)
        _FULL[(M, var)] = (fo, fn, AO.ranked(fo, fn, np.ones(M, bool), 9))
    return _FULL[(M, var)]


@pytest.mark.gpu
@pytest.mark.parametrize("M,var", [(1024, "umma"), (1024, "ffma"), (2400, "umma")])
@pytest.mark.parametrize("ranks", [1, 2, 3, 8])
def test_full_lists(gp, oracle, M, var, ranks):
    """100 k objects: 1024 nodes on the tensor cores and on the CUDA cores, 2400 nodes (more than shared memory holds) on the
    CUDA cores by size."""
    fo, fn, want = full_case(gp, oracle, M, var)
    p = handle(gp, oracle, fn)
    with variant(var):
        got = p.assign_ranked_affinity(fo, ranks)
        one = p.assign_batch(obj_feats=fo)
    assert (got[:, 0] == one).all()
    assert (got != NONE).all()
    AO.check(got, fo, fn, np.ones(M, bool), want)


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
@pytest.mark.parametrize("M", [0, 1, 3])
def test_lists_longer_than_the_live_set_are_padded(gp, oracle, M, var):
    """M live nodes and R = 8; with M < 2 the table holds two nodes, the ones past M of weight 0."""
    fo, fn = feats(5000, max(M, 2), 16)
    w = np.ones(len(fn), dtype=np.uint32)
    w[M:] = 0
    p = handle(gp, oracle, fn, w)
    with variant(var):
        got = p.assign_ranked_affinity(fo, 8)
        one = p.assign_batch(obj_feats=fo)
    assert (got[:, M:] == NONE).all()
    assert (np.sort(got[:, :M], axis=1) == np.arange(M, dtype=np.uint32)).all()   # every live node once
    assert (got[:, 0] == one).all()
    AO.check(got, fo, fn, w > 0)


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
def test_rank_two_is_where_a_leave_sends_the_object(gp, oracle, var):
    """Three nodes leave one after another, each the most frequent rank 1 of the moment.  After each leave, assign_batch(obj_feats)
    sends the objects of the leaving node to their old rank 2, and every other object keeps its node, wherever the fp64 order is
    clear (rule (c) of the oracle module); both answers are accepted placements over the new live set in every case."""
    M, n = 64, 100_000
    fo, fn = feats(n, M, 16)
    p = handle(gp, oracle, fn)
    live = np.ones(M, bool)
    with variant(var):
        for _ in range(3):
            lists = p.assign_ranked_affinity(fo, 2)
            before = p.assign_batch(obj_feats=fo)
            assert (lists[:, 0] == before).all()
            x = int(np.bincount(before, minlength=M).argmax())
            on_x = before == x
            p.node_set_active(x, False)
            live[x] = False
            after = p.assign_batch(obj_feats=fo)
            assert (after != x).all()
            want_idx, want_cost = AO.ranked(fo, fn, live, 2)
            AO.check(after[:, None], fo, fn, live, (want_idx, want_cost))
            AO.check(lists[on_x, 1:2], fo[on_x], fn, live, (want_idx[on_x], want_cost[on_x]))
            tol = AO.tau(fo, fn, after[:, None])[:, 0] + AO.tau(fo, fn, want_idx[:, :1])[:, 0]
            clear = want_cost[:, 1] - want_cost[:, 0] > tol
            assert clear[on_x].mean() > 0.99
            assert (after[on_x & clear] == lists[on_x & clear, 1]).all()
            assert (after[~on_x & clear] == before[~on_x & clear]).all()


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
def test_exact_ties_rank_the_lower_index_first(gp, oracle, var):
    """Nodes with identical feature rows have identical fp32 costs: twins inside one group of 8 (10, 11), in different groups (3, 44),
    and a triple across groups (5, 29, 50).  The lower index ranks first and the twins fill consecutive ranks."""
    M, n, R = 64, 60_000, 4
    fo, fn = feats(n, M, 16)
    sets = [(10, 11), (3, 44), (5, 29, 50)]
    for s in sets:
        fn[list(s[1:])] = fn[s[0]]
    p = handle(gp, oracle, fn)
    with variant(var):
        got = p.assign_ranked_affinity(fo, R)
        assert (got[:, 0] == p.assign_batch(obj_feats=fo)).all()
    AO.check(got, fo, fn, np.ones(M, bool))
    for s in sets:
        for a, b in zip(s, s[1:]):
            ra, rb = got == a, got == b
            # wherever the later twin is listed, the earlier one is right before it; the earlier one is followed by the later one
            assert (ra[:, :-1] == rb[:, 1:]).all(), (a, b)
            assert not rb[:, 0].any(), (a, b)
        assert (got[:, 0] == s[0]).sum() > 100, s   # the ties really met


@pytest.mark.gpu
def test_bf16_exact_inputs_agree_across_paths(gp, oracle):
    """bf16-representable features: every product is exact in fp32, the two paths differ only in the order of the 16 additions, so
    their lists agree in all but a few rows, and where they differ both are accepted placements (the difference is a near-tie)."""
    rng = np.random.default_rng(3)

    def bf16_round(x):
        u = x.astype(np.float32).view(np.uint32)
        return ((u + 0x8000) & 0xFFFF0000).astype(np.uint32).view(np.float32)

    fo = bf16_round(rng.uniform(-1, 1, (30000, 16)))
    fn = bf16_round(rng.uniform(-1, 1, (512, 16)))
    p = handle(gp, oracle, fn)
    res = {}
    for v in VARIANTS:
        with variant(v):
            res[v] = p.assign_ranked_affinity(fo, 4)
    want = AO.ranked(fo, fn, np.ones(512, bool), 5)
    for v in VARIANTS:
        AO.check(res[v], fo, fn, np.ones(512, bool), want)
    assert (res["umma"] == res["ffma"]).all(axis=1).mean() > 0.9999


@pytest.mark.gpu
@pytest.mark.parametrize("var", VARIANTS)
def test_device_variant_and_bad_arguments(gp, oracle, var):
    M, n, R = 256, 30_001, 5
    fo, fn = feats(n, M, 16)
    p = handle(gp, oracle, fn)
    L, h = p.L, p.h
    with variant(var):
        want = p.assign_ranked_affinity(fo, R)
        df, di = C.c_void_p(), C.c_void_p()
        p._ck(L.rio_cuda_dev_alloc(h, n * 16 * 4, C.byref(df)))
        p._ck(L.rio_cuda_dev_alloc(h, n * R * 4, C.byref(di)))
        p._ck(L.rio_cuda_memcpy_h2d(h, df, fo.ctypes.data_as(C.c_void_p), n * 16 * 4))
        got = np.empty((n, R), dtype=np.uint32)
        for _ in range(2):   # two calls: identical bytes
            p._ck(L.rio_cuda_assign_ranked_affinity_batch_dev(h, df, n, R, di))
            p._ck(L.rio_cuda_memcpy_d2h(h, got.ctypes.data_as(C.c_void_p), di, n * R * 4))
            p.sync()
            assert (got == want).all()
        # a table change between two calls: the lists follow it
        p.node_set_active(9, False)
        live = np.ones(M, bool)
        live[9] = False
        p._ck(L.rio_cuda_assign_ranked_affinity_batch_dev(h, df, n, R, di))
        p._ck(L.rio_cuda_memcpy_d2h(h, got.ctypes.data_as(C.c_void_p), di, n * R * 4))
        p.sync()
        assert (got != 9).all() and (got[:, 0] == p.assign_batch(obj_feats=fo)).all()
        AO.check(got, fo, fn, live)
        out = np.empty((n, 9), dtype=np.uint32)
        fp = fo.ctypes.data_as(C.c_void_p)
        for ranks in (0, 9):
            for call, f, o in ((L.rio_cuda_assign_ranked_affinity_batch, fp, out.ctypes.data_as(C.c_void_p)),
                               (L.rio_cuda_assign_ranked_affinity_batch_dev, df, di)):
                assert call(h, f, n, ranks, o) == -2
                assert b"ranks" in L.rio_cuda_last_error(h)
        for call in (L.rio_cuda_assign_ranked_affinity_batch, L.rio_cuda_assign_ranked_affinity_batch_dev):
            assert call(h, None, n, 2, di) == -2 and L.rio_cuda_last_error(h)
            assert call(h, df, n, 2, None) == -2 and L.rio_cuda_last_error(h)
        assert L.rio_cuda_assign_ranked_affinity_batch(h, None, 2**62, 8, None) == -2 and b"overflow" in L.rio_cuda_last_error(h)
        with pytest.raises(gp.Unknown):
            p.assign_ranked_affinity(fo, 0)
        assert p.assign_ranked_affinity(np.empty((0, 16), np.float32), 4).shape == (0, 4)
        p._ck(L.rio_cuda_dev_free(h, df))
        p._ck(L.rio_cuda_dev_free(h, di))
    # a handle without node features
    q = gp.GpuObjectPlacement()
    addrs, _, _ = oracle.synth_nodes(8)
    q.set_nodes(addrs)
    for call in (q.L.rio_cuda_assign_ranked_affinity_batch, q.L.rio_cuda_assign_ranked_affinity_batch_dev):
        assert call(q.h, fp, 100, 2, out.ctypes.data_as(C.c_void_p)) == -2
        assert b"needs node features" in q.L.rio_cuda_last_error(q.h)


DOUBLES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "hostsim", "affinity_ranked_launchers.cpp")


def test_the_doubles_cover_every_ranked_affinity_launcher():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    decl = set(re.findall(r"\b(launch_[a-z0-9_]+)\s*\(", open(os.path.join(root, "rio_rs_b200", "csrc", "k_affinity_ranked.cuh")).read()))
    have = set(re.findall(r"^(?:void|cudaError_t)\s+([a-z0-9_]+)\s*\(", open(DOUBLES).read(), flags=re.M))
    assert decl and decl <= have, decl - have


def test_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + the doubles above)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, "librio_cuda_hostsim_affinity_ranked.so")
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + [DOUBLES, "-o", so, "-ldl", "-lpthread"])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 50 and "failed" not in r.stdout, tail


def test_calls_report_an_error_where_the_kernels_are_not_linked():
    """The engine's host code built WITHOUT the ranked affinity launchers still loads, assign_batch(obj_feats) works, and both ranked
    affinity entry points answer RIO_ERR_UPSTREAM with a message instead of computing anything."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, "librio_cuda_hostsim_no_affinity_ranked.so")
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + ["-o", so, "-ldl", "-lpthread"])
    code = (
        "import sys, ctypes as C, numpy as np\n"
        "from rio_rs_b200 import _native as N\n"
        "N.library_path = lambda: sys.argv[1]\n"
        "import rio_rs_b200 as R\n"
        "p = R.GpuObjectPlacement()\n"
        "fn = np.random.default_rng(1).uniform(-1, 1, (8, 16)).astype(np.float32)\n"
        "fo = np.random.default_rng(2).uniform(-1, 1, (100, 16)).astype(np.float32)\n"
        "p.set_nodes(['10.0.0.%d:5000' % j for j in range(8)], None, fn)\n"
        "assert (p.assign_batch(obj_feats=fo) < 8).all()\n"
        "try:\n"
        "    p.assign_ranked_affinity(fo, 2)\n"
        "    raise SystemExit('computed without kernels')\n"
        "except R.Upstream as e:\n"
        "    assert 'ranked affinity kernels' in str(e), e\n"
        "d = C.c_void_p()\n"
        "p._ck(p.L.rio_cuda_dev_alloc(p.h, 100 * 16 * 4, C.byref(d)))\n"
        "assert p.L.rio_cuda_assign_ranked_affinity_batch_dev(p.h, d, 100, 2, d) == -1\n"
        "assert b'ranked affinity kernels' in p.L.rio_cuda_last_error(p.h)\n"
        "print('refused ok')\n"
    )
    r = subprocess.run([sys.executable, "-c", code, so], capture_output=True, text=True, timeout=300, cwd=HS.ROOT)
    assert r.returncode == 0 and "refused ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

"""Bounded-load placement under the affinity cost (DESIGN.md 3.16): ObjectSet.assign_bounded_affinity and
GpuObjectPlacement.assign_bounded_affinity_batch against tests/affinity_bounded_oracle.py, the round loop of 3.5 with the affinity
argmin in place of the rendezvous hash.

* CUDA cores: idx, counters and passes equal the oracle over the exact c32 argmin bit for bit.
* Tensor cores, small-integer features (every product and sum exact): the same oracle, bit for bit, exact cost ties included.
* Tensor cores, U(-1, 1) features: the oracle over an argmin built from the engine itself, a twin handle whose closed nodes are
  inactive; two identical calls give identical results.
* Every run also checks: pass 0 is set_assign(use_affinity = 1), the counters are the histogram of the result, an object that moved
  left a closed node, the batch form equals the set form, and ranked lists are dropped.

The CPU tests at the end run this module's GPU bodies, unchanged, against the engine's host logic compiled with g++ (the host-sim
library of tests/test_engine_host_sim.py) with a plain restatement of the new launcher, and check that a build without it refuses
both calls while the other bounded and affinity calls keep working.  There the tensor-core path is never selected."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import affinity_bounded_oracle as BO

NONE = 0xFFFFFFFF
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPS = [(5, 4), (101, 100), (1, 1)]
ROUNDS = [1, 2, 4, 16]


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


def tensor_cores(p, var, K, n_live):
    padded = 64 if n_live <= 64 else (n_live + 255) // 256 * 256
    return var == "umma" and K == 16 and 0 < padded <= 2304 and not host_sim(p)


def addresses(M):
    return ["10.1.%d.%d:7000" % (j >> 8, j & 255) for j in range(M)]


class Cluster:
    """A handle with M nodes (weights, feature rows, some inactive, optionally some active with weight 0) and a set of n objects with
    keys and features, mirrored here for the oracle."""

    def __init__(self, gp, M, n, K, seed=0, fo=None, fn=None, dead=(), zero_weight=(), wmax=16):
        rng = np.random.default_rng(1000 + seed)
        self.gp, self.M, self.n, self.K = gp, M, n, K
        self.fo = rng.uniform(-1, 1, (n, K)).astype(np.float32) if fo is None else np.asarray(fo, np.float32)
        self.fn = rng.uniform(-1, 1, (M, K)).astype(np.float32) if fn is None else np.asarray(fn, np.float32)
        self.w = rng.integers(1, wmax + 1, M).astype(np.uint32)
        self.w[list(zero_weight)] = 0
        self.active = np.ones(M, bool)
        self.active[list(dead)] = False
        self.live = self.active & (self.w > 0)
        self.keys = rng.integers(0, 2**63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)
        self.p = self.handle(self.active)
        self.s = self.p.new_set(n)
        self.s.load_keys(self.keys)
        self.s.load_feats(self.fo)

    def handle(self, mask):
        """A handle with this cluster's nodes, those outside `mask` inactive."""
        p = self.gp.GpuObjectPlacement()
        p.set_nodes(addresses(self.M), self.w, self.fn)
        for j in np.flatnonzero(~np.asarray(mask, bool)):
            p.node_set_active(int(j), False)
        return p

    def oracle(self, cap, rounds, argmin=None, n_total=0):
        return BO.assign_bounded(self.keys, argmin or BO.c32_argmin(self.fo, self.fn), self.w, self.live, self.active, n_total, cap[0], cap[1], rounds)

    def engine_argmin(self):
        """The engine as its own primitive: the objects `rows` placed by assign_batch(obj_feats) on a twin handle whose nodes outside
        `mask` are inactive (the operands a spill round compacts over live minus closed)."""
        def argmin(rows, mask):
            return self.handle(mask).assign_batch(obj_feats=self.fo[rows])
        return argmin

    def run(self, cap, rounds, var, want=None):
        """The set call and the batch call under `var`, checked against `want` (the oracle's tuple) and the invariants of 3.16."""
        with variant(var):
            self.s.assign(True)
            plain = self.s.read()
            self.s.assign_ranked_affinity(2)
            passes = self.s.assign_bounded_affinity(0, cap[0], cap[1], rounds)
            got, cnt = self.s.read(), self.s.counters()
            bidx, bpasses = self.p.assign_bounded_affinity_batch(self.keys, self.fo, 0, cap[0], cap[1], rounds)
        with pytest.raises(self.gp.Unknown):
            self.s.read_ranked()
        assert (cnt == BO.counts(got, self.M)).all()
        assert bidx.tobytes() == got.tobytes() and bpasses == passes
        if want is not None:
            widx, wcnt, wpasses, wpass0, wclosed, _ = want
            assert plain.tobytes() == wpass0.tobytes()
            assert passes == wpasses, (passes, wpasses)
            assert (cnt == wcnt).all()
            assert got.tobytes() == widx.tobytes(), int((got != widx).sum())
            moved = got != plain
            assert wclosed[plain[moved]].all()   # an object leaves its pass-0 node only by spilling from it
        return got, cnt, passes


@pytest.mark.gpu
@pytest.mark.parametrize("K", [8, 16, 24])
@pytest.mark.parametrize("cap", CAPS)
def test_cuda_cores_equal_the_oracle(gp, K, cap):
    """RIO_AFFINITY_VARIANT=ffma (and K = 8 / 24, where no tensor path exists): bit for bit the oracle over c32, at every max_rounds,
    weights 1..16, two dead nodes and one active node of weight 0."""
    c = Cluster(gp, 48, 20000, K, seed=K + cap[0], dead=(5, 17), zero_weight=(30,))
    fired = 0
    for rounds in ROUNDS:
        want = c.oracle(cap, rounds)
        _, _, passes = c.run(cap, rounds, "ffma", want)
        fired += passes > 1
    assert fired >= 2   # the inputs are imbalanced enough for spill rounds to run


@pytest.mark.gpu
def test_stops_when_no_node_is_open(gp):
    """Every object prefers node 0, then 1, then 2, then 3: at cap 1/1 the spills cascade down the order until the last node goes
    over too, and the rounds stop with nothing open (the seed is the first whose oracle run ends that way)."""
    K, M, n = 8, 4, 4000
    fn = np.zeros((M, K), np.float32)
    fn[:, 0] = [4, 3, 2, 1]
    for seed in range(40):
        rng = np.random.default_rng(seed)
        fo = np.zeros((n, K), np.float32)
        fo[:, 0] = rng.uniform(0.5, 1, n)
        c = Cluster(gp, M, n, K, seed=seed, fo=fo, fn=fn, wmax=1)
        want = c.oracle((1, 1), 16)
        if want[5] == "closed":
            break
    else:
        pytest.fail("no seed closes every node")
    _, _, passes = c.run((1, 1), 16, "ffma", want)
    assert 1 < passes < 16


def int_feats(rng, shape):
    return rng.integers(-4, 5, shape).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [48, 64, 65, 257])
@pytest.mark.parametrize("cap", CAPS)
def test_tensor_cores_equal_the_oracle_on_integer_features(gp, M, cap):
    """Features in [-4, 4]: the bf16 split, the wgmma accumulation and c32 are all exact, so the tensor path must give the c32 oracle's
    answer bit for bit, exact ties to the lower index included.  65 and 257 live nodes sit one past a padding step; their closed sets
    take the compacted count back across it."""
    rng = np.random.default_rng(M + cap[0])
    c = Cluster(gp, M, 20000, 16, seed=M, fo=int_feats(rng, (20000, 16)), fn=int_feats(rng, (M, 16)))
    fired = 0
    for rounds in ROUNDS:
        want = c.oracle(cap, rounds)
        _, _, passes = c.run(cap, rounds, "umma", want)
        fired += passes > 1
        if M in (65, 257) and rounds == 16 and passes > 1:
            assert want[4].sum() >= 1   # 64 | 256 open nodes or fewer: the round ran on the smaller tile
    assert fired >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("M", [2304, 2305])
def test_live_count_at_the_tensor_core_limit(gp, M):
    """2304 live nodes are the tensor path's largest padded set; at 2305 pass 0 and every round take the CUDA cores.  Integer features
    make both equal the c32 oracle."""
    rng = np.random.default_rng(M)
    n = 6000
    c = Cluster(gp, M, n, 16, seed=M, fo=int_feats(rng, (n, 16)), fn=int_feats(rng, (M, 16)))
    for cap, rounds in [((5, 4), 4), ((1, 1), 16)]:
        c.run(cap, rounds, "umma", c.oracle(cap, rounds))


@pytest.mark.gpu
@pytest.mark.parametrize("M", [48, 200, 700])
def test_tensor_cores_equal_the_engine_restatement(gp, M):
    """U(-1, 1) features on the tensor cores: each round's re-placement is what a twin handle with the closed nodes inactive returns
    from assign_batch for the spilled rows.  Two identical calls agree, so a row's answer does not depend on its place in the batch."""
    c = Cluster(gp, M, 60000, 16, seed=M, dead=(3,))
    with variant("umma"):
        assert tensor_cores(c.p, "umma", 16, int(c.live.sum())) or host_sim(c.p)
        fired = 0
        for cap in CAPS:
            want = c.oracle(cap, 8, argmin=c.engine_argmin())
            first = c.run(cap, 8, "umma", want)
            again = c.run(cap, 8, "umma", want)
            assert first[0].tobytes() == again[0].tobytes() and first[2] == again[2]
            fired += first[2] > 1
    assert fired >= 2


@pytest.mark.gpu
def test_errors(gp):
    R = gp
    fo = np.random.default_rng(3).uniform(-1, 1, (100, 16)).astype(np.float32)
    keys = np.arange(100, dtype=np.uint64)
    # a handle without node features
    p = R.GpuObjectPlacement()
    p.set_nodes(addresses(8))
    s = p.new_set(100)
    s.load_keys(keys)
    s.load_feats(fo)
    with pytest.raises(R.Unknown):
        s.assign_bounded_affinity()
    with pytest.raises(R.Unknown):
        p.assign_bounded_affinity_batch(keys, fo)
    # set features missing, then of another K
    p = R.GpuObjectPlacement()
    p.set_nodes(addresses(8), None, np.ones((8, 16), np.float32))
    s = p.new_set(100)
    s.load_keys(keys)
    with pytest.raises(R.Unknown):
        s.assign_bounded_affinity()
    s.load_feats(fo[:, :8])
    with pytest.raises(R.Unknown):
        s.assign_bounded_affinity()
    s.load_feats(fo)
    # bad factor / rounds
    for bad in [dict(cap_den=0), dict(max_rounds=0)]:
        with pytest.raises(R.Unknown):
            s.assign_bounded_affinity(**bad)
        with pytest.raises(R.Unknown):
            p.assign_bounded_affinity_batch(keys, fo, **bad)
    # a bounded call in flight on the set
    s.assign_bounded_begin(0, 5, 4, 4)
    with pytest.raises(R.Unknown):
        s.assign_bounded_affinity()
    s.assign_bounded_end()
    assert s.assign_bounded_affinity() >= 1
    # NULL buffers
    out = np.empty(100, np.uint32)
    for k, f, o in [(None, fo, out), (keys, None, out), (keys, fo, None)]:
        st = p.L.rio_cuda_assign_bounded_affinity_batch(p.h, None if k is None else k.ctypes.data, None if f is None else f.ctypes.data, 100, 0, 5, 4, 4,
                                                        None if o is None else o.ctypes.data, None)
        assert st != 0
    assert p.L.rio_cuda_set_assign_bounded_affinity(None, 0, 5, 4, 4, None) != 0
    # n = 0 answers OK with no pass
    assert p.assign_bounded_affinity_batch(keys[:0], fo[:0])[1] == 0


def _worker(rank, world, port, n, M, q, comm):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["RIO_COMM"] = comm
    import torch.distributed as dist

    import rio_rs_b200 as R
    from rio_rs_b200 import parallel

    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)  # bootstrap only
    rng = np.random.default_rng(77)
    fo = rng.uniform(-1, 1, (n, 16)).astype(np.float32)
    fn = rng.uniform(-1, 1, (M, 16)).astype(np.float32)
    w = rng.integers(1, 17, M).astype(np.uint32)
    keys = rng.integers(0, 2**63, n, dtype=np.uint64)
    p = R.GpuObjectPlacement(device=rank)
    parallel.init_comm(p, dist)
    p.set_nodes(addresses(M), w, fn)
    lo, hi = parallel.shard_range(n, rank, world)
    s = p.new_set(hi - lo)
    s.load_keys(keys[lo:hi])
    s.load_feats(fo[lo:hi])
    out = {}
    for var in ("umma", "ffma"):
        os.environ["RIO_AFFINITY_VARIANT"] = var
        for cap in CAPS:
            passes = s.assign_bounded_affinity(n, cap[0], cap[1], 4)
            out[var, cap] = (passes, s.read().tolist(), s.counters().tolist())
    q.put((rank, lo, hi, out))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("comm", ["p2p", "nccl"])
def test_two_ranks_equal_one_rank_on_the_global_set(gp, comm):
    """Two ranks, each with one shard: every shard equals the one-rank call on the global set, and every rank holds the global
    counters.  Skipped with fewer than two GPUs."""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    n, M, world = 200_000, 96, 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + os.getpid() % 500 + (11 if comm == "nccl" else 0)
    procs = [ctx.Process(target=_worker, args=(r, world, port, n, M, q, comm)) for r in range(world)]
    for pr in procs:
        pr.start()
    res = sorted(q.get(timeout=600) for _ in range(world))
    for pr in procs:
        pr.join(timeout=120)
        assert pr.exitcode == 0
    rng = np.random.default_rng(77)
    fo = rng.uniform(-1, 1, (n, 16)).astype(np.float32)
    fn = rng.uniform(-1, 1, (M, 16)).astype(np.float32)
    w = rng.integers(1, 17, M).astype(np.uint32)
    keys = rng.integers(0, 2**63, n, dtype=np.uint64)
    p = gp.GpuObjectPlacement()
    p.set_nodes(addresses(M), w, fn)
    for var in ("umma", "ffma"):
        for cap in CAPS:
            with variant(var):
                widx, wpasses = p.assign_bounded_affinity_batch(keys, fo, n, cap[0], cap[1], 4)
            got = np.empty(n, dtype=np.uint32)
            for rank, lo, hi, out in res:
                passes, idx, cnt = out[var, cap]
                got[lo:hi] = idx
                assert passes == wpasses and cnt == BO.counts(widx, M).tolist()
            assert got.tobytes() == widx.tobytes(), (var, cap)


DOUBLES = os.path.join(ROOT, "tests", "cpp", "hostsim", "affinity_bounded_launchers.cpp")
OTHER_DOUBLES = [os.path.join(ROOT, "tests", "cpp", "hostsim", f) for f in ("ranked_launchers.cpp", "change_launchers.cpp", "ranked_change_launchers.cpp",
                                                                              "spread_launchers.cpp", "spread_change_launchers.cpp",
                                                                              "affinity_ranked_launchers.cpp", "affinity_spread_launchers.cpp",
                                                                              "affinity_set_launchers.cpp")]


def test_the_doubles_cover_the_bounded_affinity_launcher():
    decl = set(re.findall(r"\b(launch_[a-z0-9_]+)\s*\(", open(os.path.join(ROOT, "rio_rs_b200", "csrc", "k_affinity_bounded.cuh")).read()))
    have = set(re.findall(r"^void\s+([a-z0-9_]+)\s*\(", open(DOUBLES).read(), flags=re.M))
    assert len(decl) == 1 and decl <= have, decl - have


def _hostsim_library(HS, name, doubles):
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, name)
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + doubles + ["-o", so, "-ldl", "-lpthread"])
    return so


def test_bounded_affinity_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + every ranked, set, affinity
    and bounded-affinity double); the two-rank test skips there."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_bounded_affinity.so", OTHER_DOUBLES + [DOUBLES])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=3000, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 22 and "failed" not in r.stdout, tail


def test_bounded_affinity_reports_an_error_where_the_kernel_is_not_linked():
    """The engine's host code built WITHOUT the bounded-affinity launcher loads, refuses both new calls with RIO_ERR_UPSTREAM and a
    message, and still serves set_assign_bounded and set_assign(use_affinity = 1)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_no_bounded_affinity.so", OTHER_DOUBLES)
    code = (
        "import sys, numpy as np\n"
        "from rio_rs_b200 import _native as N\n"
        "N.library_path = lambda: sys.argv[1]\n"
        "import rio_rs_b200 as R\n"
        "p = R.GpuObjectPlacement()\n"
        "fn = np.random.default_rng(1).uniform(-1, 1, (8, 16)).astype(np.float32)\n"
        "fo = np.random.default_rng(2).uniform(-1, 1, (100, 16)).astype(np.float32)\n"
        "keys = np.arange(100, dtype=np.uint64)\n"
        "p.set_nodes(['10.0.0.%d:5000' % j for j in range(8)], None, fn)\n"
        "s = p.new_set(100); s.load_keys(keys); s.load_feats(fo)\n"
        "for call in (lambda: s.assign_bounded_affinity(), lambda: p.assign_bounded_affinity_batch(keys, fo)):\n"
        "    try:\n"
        "        call()\n"
        "        raise SystemExit('computed without kernels')\n"
        "    except R.Upstream as e:\n"
        "        assert 'bounded affinity kernels' in str(e), e\n"
        "s.assign(True)\n"
        "assert (s.read() == p.assign_batch(obj_feats=fo)).all()\n"
        "assert s.assign_bounded(0, 5, 4, 4) >= 1\n"
        "assert (s.read() == p.assign_bounded_batch(keys, 0, 5, 4, 4)[0]).all()\n"
        "print('refused ok')\n"
    )
    r = subprocess.run([sys.executable, "-c", code, so], capture_output=True, text=True, timeout=300, cwd=HS.ROOT)
    assert r.returncode == 0 and "refused ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

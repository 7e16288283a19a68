"""Bounded-load affinity sets kept within capacity through membership changes (DESIGN.md 3.17): ObjectSet.rebalance_changes_bounded_affinity
against tests/affinity_set_bounded_oracle.py, after every change set of a sequence that starts from assign_bounded_affinity.

* CUDA cores (K = 8, 16 with RIO_AFFINITY_VARIANT=ffma, 24): idx, counters, passes and moved equal the oracle over the exact c32
  argmin bit for bit.
* Tensor cores, small-integer features (every product and sum exact): the same oracle, bit for bit.
* Tensor cores, U(-1, 1) features: the oracle over an argmin built from the engine itself (a twin handle whose nodes outside the mask
  are inactive, the pattern of tests/test_gpu_bounded_affinity.py); the S2 merge is c32 on both paths.
* After every call: the counters are the histogram of idx, and every object that moved was S1, was taken by a candidate, or sat on a
  node that was over capacity in some round.

The CPU tests at the end run this module's GPU bodies, unchanged, against the engine's host logic compiled with g++ (the host-sim
library of tests/test_engine_host_sim.py) with a plain restatement of the new launchers, and check that a build without them refuses
the new call while set_assign_bounded_affinity and set_rebalance_changes_ranked keep working.  There the tensor path is never taken."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import affinity_bounded_oracle as BO
import affinity_set_bounded_oracle as SB

NONE = 0xFFFFFFFF
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPS = [(5, 4), (101, 100), (1, 1)]
ROUNDS = [16, 1, 4, 2, 8]


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
    return ["10.2.%d.%d:7000" % (j >> 8, j & 255) for j in range(M)]


def int_feats(rng, shape):
    return rng.integers(-4, 5, shape).astype(np.float32)


class BCluster:
    """A handle whose node table is mirrored here (feature rows as the kernels see them, weights, active flags of every interned node),
    a set of n objects assigned by assign_bounded_affinity, and the mirror of the set's record (the feature rows of the last call)."""

    def __init__(self, gp, M, n, K, var, cap, seed=0, ints=False, engine=False, dead=(), spare=8):
        rng = np.random.default_rng(500 + seed)
        self.gp, self.K, self.var, self.cap, self.ints, self.engine = gp, K, var, cap, ints, engine
        self.rng = rng
        self.fo = int_feats(rng, (n, K)) if ints else rng.uniform(-1, 1, (n, K)).astype(np.float32)
        self.fn = self.feats(M)
        self.w = rng.integers(1, 17, M).astype(np.uint32)
        self.active = np.ones(M, bool)
        self.active[list(dead)] = False
        self.addrs = addresses(M + spare)
        self.keys = rng.integers(0, 2**63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)
        self.p = self.handle(self.active)
        self.s = self.p.new_set(n)
        self.s.load_keys(self.keys)
        self.s.load_feats(self.fo)
        with variant(var):
            passes = self.s.assign_bounded_affinity(0, cap[0], cap[1], 16)
        self.idx = self.s.read()
        want = BO.assign_bounded(self.keys, self.argmin(), self.w, self.live, self.active, 0, cap[0], cap[1], 16)
        assert passes == want[2] and self.idx.tobytes() == want[0].tobytes()
        self.snap = self.fn.copy()
        self.tensor = tensor_cores(self.p, var, K, int(self.live.sum()))
        self.steps = self.n_beaten = self.n_spilled = 0

    @property
    def live(self):
        return self.active & (self.w > 0)

    def feats(self, m):
        return int_feats(self.rng, (m, self.K)) if self.ints else self.rng.uniform(-1, 1, (m, self.K)).astype(np.float32)

    def handle(self, mask):
        """A handle with this cluster's nodes, those outside `mask` inactive."""
        p = self.gp.GpuObjectPlacement()
        M = len(self.fn)
        p.set_nodes(self.addrs[:M], self.w, self.fn)
        for j in np.flatnonzero(~np.asarray(mask, bool)):
            p.node_set_active(int(j), False)
        return p

    def argmin(self):
        if not self.engine:
            return BO.c32_argmin(self.fo, self.fn)

        def argmin(rows, mask):
            return self.handle(mask).assign_batch(obj_feats=self.fo[rows])
        return argmin

    # ---- node-table changes, mirrored; each returns the change set (idx, prev_weight) -----------------------------------------
    def prev_of(self, js):
        return [int(self.w[j]) if self.live[j] else 0 for j in js]

    def leave(self, js):
        prev = self.prev_of(js)
        for j in js:
            self.p.node_set_active(int(j), False)
            self.active[j] = False
        return list(js), prev

    def join(self, js):
        """re-activates interned nodes (features kept) or interns the next spare (fresh features)"""
        prev = []
        for j in js:
            if j >= len(self.fn):
                assert j == len(self.fn)
                f = self.feats(1)[0]
                self.fn = np.vstack([self.fn, f[None]])
                self.w = np.append(self.w, np.uint32(self.rng.integers(1, 17)))
                self.active = np.append(self.active, False)
                prev.append(0)
                assert self.p.node_upsert(self.addrs[j], int(self.w[j]), f) == j
            else:
                prev.append(self.prev_of([j])[0])
                if self.w[j] == 0:
                    self.w[j] = 1
                self.p.node_upsert(self.addrs[j], int(self.w[j]))
            self.active[j] = True
        return list(js), prev

    def reweight(self, js, w):
        prev = self.prev_of(js)
        for j, wj in zip(js, w):
            self.w[j] = wj
            self.p.node_upsert(self.addrs[j], int(wj))
            self.active[j] = True
        return list(js), prev

    def refeature(self, js):
        f = self.feats(len(js))
        for q, j in enumerate(js):
            self.fn[j] = f[q]
            self.p.node_upsert(self.addrs[j], int(self.w[j]), self.fn[j])
            self.active[j] = True   # node_upsert activates
        return [], []

    def set_nodes_refeatured(self, js):
        """set_nodes over the active nodes with new features for js; the inactive nodes lose theirs (zeros), as set_nodes does"""
        f = self.feats(len(js))
        for q, j in enumerate(js):
            self.fn[j] = f[q]
        on = np.flatnonzero(self.active)
        self.fn[~self.active] = 0
        self.p.set_nodes([self.addrs[j] for j in on], self.w[on], self.fn[on])
        return [], []

    # ---- one call of the new entry point against the oracle -----------------------------------------------------------------
    def step(self, change, tag, rounds=None, cap=None):
        idx, prev = change
        cap = cap or self.cap
        rounds = rounds or ROUNDS[self.steps % len(ROUNDS)]
        self.steps += 1
        M = len(self.fn)
        live = self.live
        snap = np.zeros((M, self.K), np.float32)
        snap[: len(self.snap)] = self.snap
        refeat = live & ((np.arange(M) >= len(self.snap)) | (snap.view(np.uint32) != self.fn.view(np.uint32)).any(axis=1))
        replace = ~live | refeat
        cand = [j for j, pw in zip(idx, prev) if live[j] and pw == 0] + [int(j) for j in np.flatnonzero(refeat)]
        want = SB.rebalance(self.keys, self.idx, self.fo, self.fn, self.argmin(), replace, sorted(set(cand)), self.w, live, self.active, 0, cap[0],
                            cap[1], rounds)
        with variant(self.var):
            moved, passes = self.s.rebalance_changes_bounded_affinity(idx, prev, 0, cap[0], cap[1], rounds)
        got, cnt = self.s.read(), self.s.counters()
        assert (cnt == BO.counts(got, M)).all(), tag
        assert got.tobytes() == want["idx"].tobytes(), (tag, int((got != want["idx"]).sum()))
        assert (cnt == want["counters"]).all(), tag
        assert (passes, moved) == (want["passes"], want["moved"]), (tag, passes, moved, want["passes"], want["moved"])
        assert moved == int((got != self.idx).sum()), tag
        # the movement contract: S1, taken by a candidate, or spilled from a node that was over capacity in some round
        ch = got != self.idx
        rest = ch & ~want["s1"] & ~want["beaten"]
        assert want["over"][self.idx[rest]].all() and want["spilled"][rest].all(), tag
        self.n_beaten += int(want["beaten"].sum())
        self.n_spilled += int(want["spilled"].sum())
        self.idx = got
        self.snap = self.fn.copy()
        self.tensor = tensor_cores(self.p, self.var, self.K, int(live.sum()))
        return want


def busiest(c):
    i = c.idx[c.idx != NONE].astype(np.int64)
    return int(np.bincount(i, minlength=len(c.fn)).argmax())


def sequence(c):
    """the change sets of DESIGN.md 3.17's tests, one after the other"""
    M0 = len(c.fn)
    b = busiest(c)
    c.step(c.leave([b]), "one leave")
    c.step(c.join([b]), "one join")
    c.step(c.leave(list(range(8, 16))), "a rack leaves")
    c.step(c.join(list(range(8, 16))), "the rack rejoins")
    c.step(c.join([len(c.fn)]), "a node interned after the assign joins")
    c.step(c.reweight([1, 2, 3, 4], [max(1, int(c.w[j]) // 4) for j in (1, 2, 3, 4)]), "weight decrease", rounds=16)
    # a weight increase only adds headroom: from a state within capacity nothing moves
    before = c.idx
    js = [5, 6]
    want = c.step(c.reweight(js, [int(c.w[j]) * 2 for j in js]), "weight increase", rounds=16)
    if (BO.counts(before, len(c.fn)) <= want["cap"]).all():
        assert want["moved"] == 0 and want["passes"] == 2
    c.step(c.refeature([0, M0 // 2]), "node_upsert refeature")
    c.step(c.set_nodes_refeatured([3, M0 - 1]), "set_nodes refeature")
    c.step(c.reweight([7], [0]), "an active node set to weight 0")
    c.step(([], []), "k = 0")
    c.step(c.refeature([9]), "k = 0 with a refeature")
    everyone = [int(j) for j in np.flatnonzero(c.active)]
    c.step(c.leave(everyone), "everyone leaves")
    assert (c.idx == NONE).all()
    c.step(c.join(everyone), "everyone rejoins")
    assert (c.idx != NONE).all()
    assert c.n_beaten > 0 and c.n_spilled > 0   # candidates took objects, and the rounds spilled some


@pytest.mark.gpu
@pytest.mark.parametrize("K", [8, 16, 24])
@pytest.mark.parametrize("cap", CAPS)
def test_cuda_cores_equal_the_oracle(gp, K, cap):
    """RIO_AFFINITY_VARIANT=ffma (and K = 8 / 24, where no tensor path exists): bit for bit the c32 oracle after every change set."""
    c = BCluster(gp, 48, 20000, K, "ffma", cap, seed=K + cap[0], dead=(40,))
    assert not c.tensor
    sequence(c)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [48, 65, 257])
@pytest.mark.parametrize("cap", CAPS)
def test_tensor_cores_equal_the_oracle_on_integer_features(gp, M, cap):
    """Features in [-4, 4] on the tensor cores: every cost is exact, so the c32 oracle holds bit for bit.  65 and 257 live nodes are
    one past a padding step; the first leave takes the live count back across it."""
    c = BCluster(gp, M, 20000, 16, "umma", cap, seed=M + cap[0], ints=True)
    assert c.tensor or host_sim(c.p)
    sequence(c)


@pytest.mark.gpu
def test_live_counts_at_the_launcher_thresholds(gp):
    """64 | 65 and 256 | 257 live nodes crossed both ways by joins and leaves, on both paths, integer features."""
    for var in ("umma", "ffma"):
        for M in (65, 257):
            c = BCluster(gp, M, 8000, 16, var, (5, 4), seed=M, ints=True, dead=(M - 1,))
            c.step(c.join([M - 1]), "join to %d" % M)
            c.step(c.leave([M - 1, M - 2]), "leave to %d" % (M - 2))
            c.step(c.join([M - 2]), "join to %d" % (M - 1))


@pytest.mark.gpu
def test_a_tensor_core_set_crossing_the_tensor_limit(gp):
    """2304 live nodes are the tensor path's largest padded set: a join takes the set to 2305 (the CUDA cores), a leave back.  Integer
    features make both paths equal the c32 oracle."""
    M = 2305
    c = BCluster(gp, M, 6000, 16, "umma", (5, 4), seed=M, ints=True, dead=(M - 1,))
    assert c.tensor or host_sim(c.p)
    c.step(c.join([M - 1]), "2305 live")
    assert not c.tensor
    c.step(c.leave([M - 1]), "2304 live", cap=(1, 1))
    assert c.tensor or host_sim(c.p)
    c.step(c.join([M]), "a new node: 2305 live", cap=(101, 100))


@pytest.mark.gpu
@pytest.mark.parametrize("M", [48, 200])
def test_tensor_cores_equal_the_engine_restatement(gp, M):
    """U(-1, 1) features on the tensor cores: S1 objects and spilled objects go where a twin handle with the same open nodes puts
    them; S2 objects follow c32."""
    for cap in ((5, 4), (1, 1)):
        c = BCluster(gp, M, 30000, 16, "umma", cap, seed=M + cap[0], engine=True, dead=(3,))
        assert c.tensor or host_sim(c.p)
        sequence(c)


def _fresh(gp, M=16, n=2000, K=16):
    rng = np.random.default_rng(9)
    p = gp.GpuObjectPlacement()
    p.set_nodes(addresses(M), rng.integers(1, 9, M).astype(np.uint32), rng.uniform(-1, 1, (M, K)).astype(np.float32))
    s = p.new_set(n)
    s.load_keys(rng.integers(0, 2**63, n, dtype=np.uint64))
    s.load_feats(rng.uniform(-1, 1, (n, K)).astype(np.float32))
    return p, s


@pytest.mark.gpu
def test_errors_change_nothing(gp):
    R = gp
    p, s = _fresh(gp)
    # no record yet
    with pytest.raises(R.Unknown):
        s.rebalance_changes_bounded_affinity([], [])
    assert p.L.rio_cuda_set_rebalance_changes_bounded_affinity(None, None, None, 0, 0, 5, 4, 4, None, None) != 0
    s.assign_bounded_affinity(0, 5, 4, 8)
    p.node_set_active(2, False)
    idx0, cnt0 = s.read(), s.counters()
    bad = [dict(idx=[99], prev_weight=[1]), dict(idx=[2, 2], prev_weight=[1, 1]), dict(idx=[2], prev_weight=[1], cap_den=0),
           dict(idx=[2], prev_weight=[1], max_rounds=0)]
    for b in bad:
        with pytest.raises(R.Unknown):
            s.rebalance_changes_bounded_affinity(**b)
        assert s.read().tobytes() == idx0.tobytes() and (s.counters() == cnt0).all()
    st = p.L.rio_cuda_set_rebalance_changes_bounded_affinity(s.s, None, None, 1, 0, 5, 4, 4, None, None)
    assert st != 0
    # a handle K other than the recorded one
    q, t = _fresh(gp)
    t.assign_bounded_affinity()
    q.set_nodes(addresses(16), None, np.ones((16, 8), np.float32))
    with pytest.raises(R.Unknown):
        t.rebalance_changes_bounded_affinity([], [])
    # the refused calls left the record: the change set still applies
    moved, passes = s.rebalance_changes_bounded_affinity([2], [int(1)])
    assert moved >= (idx0 == 2).sum() and passes >= 1


@pytest.mark.gpu
def test_every_dropping_call_removes_the_record(gp):
    R = gp
    rng = np.random.default_rng(4)
    calls = {
        "load_keys": lambda p, s: s.load_keys(rng.integers(0, 2**63, 2000, dtype=np.uint64)),
        "synth_keys": lambda p, s: s.synth_keys(0, 2000, 3),
        "load_feats": lambda p, s: s.load_feats(rng.uniform(-1, 1, (2000, 16)).astype(np.float32)),
        "assign": lambda p, s: s.assign(False),
        "assign_affinity": lambda p, s: s.assign(True),
        "assign_bounded": lambda p, s: s.assign_bounded(),
        "assign_bounded_begin_end": lambda p, s: (s.assign_bounded_begin(), s.assign_bounded_end()),
        "rebalance": lambda p, s: s.rebalance("join", 0),
        "rebalance_changes": lambda p, s: s.rebalance_changes([], []),
        "assign_ranked": lambda p, s: s.assign_ranked(2),
        "assign_ranked_spread": lambda p, s: s.assign_ranked_spread(2),
        "assign_ranked_affinity": lambda p, s: s.assign_ranked_affinity(2),
        "assign_ranked_affinity_spread": lambda p, s: s.assign_ranked_affinity_spread(2),
    }
    for name, call in calls.items():
        p, s = _fresh(gp)
        s.assign_bounded_affinity()
        assert s.rebalance_changes_bounded_affinity([], [])[1] >= 1
        call(p, s)
        with pytest.raises(R.Unknown):
            s.rebalance_changes_bounded_affinity([], [])
        s.assign_bounded_affinity()   # a new record
        s.rebalance_changes_bounded_affinity([], [])


def _worker(rank, world, port, n, M, q, comm):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["RIO_COMM"] = comm
    import torch.distributed as dist

    import rio_rs_b200 as R
    from rio_rs_b200 import parallel

    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)  # bootstrap only
    fo, fn, w, keys = _two_rank_inputs(n, M)
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
        s.assign_bounded_affinity(n, 5, 4, 8)
        out[var] = [_two_rank_events(p, s, n)]
    q.put((rank, lo, hi, out))
    dist.barrier()
    dist.destroy_process_group()


def _two_rank_inputs(n, M):
    rng = np.random.default_rng(78)
    return (rng.uniform(-1, 1, (n, 16)).astype(np.float32), rng.uniform(-1, 1, (M, 16)).astype(np.float32), rng.integers(1, 17, M).astype(np.uint32),
            rng.integers(0, 2**63, n, dtype=np.uint64))


def _two_rank_events(p, s, n):
    """a leave, a refeature and a k = 0 call; -> [(moved, passes, idx, counters)] after each"""
    res = []
    p.node_set_active(1, False)
    for ch in (([1], [3]), ([], [])):
        moved, passes = s.rebalance_changes_bounded_affinity(ch[0], ch[1], n, 5, 4, 8)
        res.append((moved, passes, s.read().tolist(), s.counters().tolist()))
    p.node_set_active(1, True)
    return res


@pytest.mark.gpu
@pytest.mark.parametrize("comm", ["p2p", "nccl"])
def test_two_ranks_equal_one_rank_on_the_global_set(gp, comm):
    """Two ranks, each with one shard: after every change set each shard equals the one-rank call on the global set, every rank holds
    the global counters and the same passes, and the moved counts add up to the one-rank count.  Skipped with fewer than two GPUs."""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    n, M, world = 200_000, 96, 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 30500 + os.getpid() % 500 + (11 if comm == "nccl" else 0)
    procs = [ctx.Process(target=_worker, args=(r, world, port, n, M, q, comm)) for r in range(world)]
    for pr in procs:
        pr.start()
    res = sorted(q.get(timeout=600) for _ in range(world))
    for pr in procs:
        pr.join(timeout=120)
        assert pr.exitcode == 0
    fo, fn, w, keys = _two_rank_inputs(n, M)
    p = gp.GpuObjectPlacement()
    p.set_nodes(addresses(M), w, fn)
    s = p.new_set(n)
    s.load_keys(keys)
    s.load_feats(fo)
    for var in ("umma", "ffma"):
        with variant(var):
            s.assign_bounded_affinity(n, 5, 4, 8)
            want = _two_rank_events(p, s, n)
        for e, (wmoved, wpasses, widx, wcnt) in enumerate(want):
            got = np.empty(n, dtype=np.uint32)
            moved = 0
            for rank, lo, hi, out in res:
                m, passes, idx, cnt = out[var][0][e]
                got[lo:hi] = idx
                moved += m
                assert passes == wpasses and cnt == wcnt
            assert got.tolist() == widx and moved == wmoved, (var, e)


DOUBLES = os.path.join(ROOT, "tests", "cpp", "hostsim", "set_bounded_affinity_launchers.cpp")
OTHER_DOUBLES = [os.path.join(ROOT, "tests", "cpp", "hostsim", f) for f in ("ranked_launchers.cpp", "change_launchers.cpp", "ranked_change_launchers.cpp",
                                                                              "spread_launchers.cpp", "spread_change_launchers.cpp",
                                                                              "affinity_ranked_launchers.cpp", "affinity_spread_launchers.cpp",
                                                                              "affinity_set_launchers.cpp", "affinity_bounded_launchers.cpp")]


def test_the_doubles_cover_the_new_launchers():
    decl = set(re.findall(r"\b(launch_[a-z0-9_]+)\s*\(", open(os.path.join(ROOT, "rio_rs_b200", "csrc", "k_set_bounded_affinity.cuh")).read()))
    have = set(re.findall(r"^void\s+([a-z0-9_]+)\s*\(", open(DOUBLES).read(), flags=re.M))
    assert len(decl) == 2 and decl <= have, decl - have


def _hostsim_library(HS, name, doubles):
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, name)
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + doubles + ["-o", so, "-ldl", "-lpthread"])
    return so


def test_set_bounded_affinity_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + every double, the new one
    included); the two-rank test skips there."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_set_bounded_affinity.so", OTHER_DOUBLES + [DOUBLES])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=3000, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 24 and "failed" not in r.stdout, tail


def test_the_new_call_reports_an_error_where_its_kernels_are_not_linked():
    """The engine's host code built WITHOUT the new launchers loads, refuses the new call with RIO_ERR_UPSTREAM and a message, and still
    serves set_assign_bounded_affinity and set_rebalance_changes_ranked."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_no_set_bounded_affinity.so", OTHER_DOUBLES)
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
        "assert s.assign_bounded_affinity(0, 5, 4, 4) >= 1\n"
        "assert (s.read() == p.assign_bounded_affinity_batch(keys, fo, 0, 5, 4, 4)[0]).all()\n"
        "try:\n"
        "    s.rebalance_changes_bounded_affinity([], [])\n"
        "    raise SystemExit('computed without kernels')\n"
        "except R.Upstream as e:\n"
        "    assert 'bounded affinity change-set kernels' in str(e), e\n"
        "s.assign_ranked_affinity(2)\n"
        "p.node_set_active(3, False)\n"
        "s.rebalance_changes_ranked([3], [1])\n"
        "assert (s.read_ranked() == p.assign_ranked_affinity(fo, 2)).all()\n"
        "print('refused ok')\n"
    )
    r = subprocess.run([sys.executable, "-c", code, so], capture_output=True, text=True, timeout=300, cwd=HS.ROOT)
    assert r.returncode == 0 and "refused ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

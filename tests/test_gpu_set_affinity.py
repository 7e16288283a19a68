"""Affinity resident sets (DESIGN.md 3.15): a set keeps each object's R lowest-cost nodes under the affinity cost of its features (or
its R lowest-cost nodes in R distinct domains), and one change-set call brings every list up to date over the current live set, node
features and labels.  Every state is compared with a fresh assign_ranked_affinity(_spread) of the set's features and with the fp64
oracles of tests/affinity_ranked_oracle.py and tests/affinity_spread_oracle.py: the lists, the set's primary index (column 0), its
counters against a histogram of column 0, and out_moved / out_changed against the row diff from the previous read-back.  On the CUDA
cores the lists equal a fresh CUDA-core call byte for byte; on the tensor cores they pass the oracle and rows no change can reach stay
as they were.

The CPU tests at the end run this module's GPU bodies, unchanged, against the engine's host logic compiled with g++ (the host-sim
library of tests/test_engine_host_sim.py) with plain restatements of the affinity-set launchers, and check that a build without those
launchers refuses the affinity-set calls while the other sets and the batch calls keep working.  There the tensor-core path is never
selected."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import affinity_ranked_oracle as AO
import affinity_spread_oracle as SO

NONE = 0xFFFFFFFF
KINDS = ["ranked", "spread"]
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rio_rs_b200", "csrc")


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


def racks(M):
    return np.arange(M, dtype=np.uint32) // max(1, -(-M // 32))


class AffCluster:
    """A provider whose node table is mirrored here (feature rows, live mask, weights, labels of every interned node) and a resident
    set holding affinity lists of its objects' features."""

    def __init__(self, gp, oracle, M, n, K, R, kind, var, seed=0, live=None, spare=8):
        self.gp, self.oracle, self.K, self.R, self.kind, self.var = gp, oracle, K, R, kind, var
        rng = np.random.default_rng(100 + seed)
        self.fo = rng.uniform(-1, 1, (n, K)).astype(np.float32)
        self.addrs = oracle.synth_nodes(M + spare)[0]   # the spares are interned by joins
        self.fn = rng.uniform(-1, 1, (M, K)).astype(np.float32)
        self.w = rng.integers(1, 5, M).astype(np.uint32)
        self.live = np.ones(M, bool) if live is None else np.asarray(live, bool).copy()
        self.dom = racks(M)
        self.p = gp.GpuObjectPlacement()
        self.p.set_nodes(self.addrs[:M], self.w, self.fn)
        self.p.set_node_domains(np.arange(M, dtype=np.uint32), self.dom)
        for j in np.flatnonzero(~self.live):
            self.p.node_set_active(int(j), False)
        self.s = self.p.new_set(n)
        self.s.synth_keys(0, n, 5)
        self.s.load_feats(self.fo)
        with variant(var):
            self.assign()
        self.tensor = tensor_cores(self.p, var, K, int(self.live.sum()))
        self.cur = self.s.read_ranked()
        self.check(self.cur, None, "assign")

    def assign(self):
        if self.kind == "spread":
            self.s.assign_ranked_affinity_spread(self.R)
        else:
            self.s.assign_ranked_affinity(self.R)

    def fresh(self, var):
        with variant(var):
            if self.kind == "spread":
                return self.p.assign_ranked_affinity_spread(self.fo, self.R)
            return self.p.assign_ranked_affinity(self.fo, self.R)

    def oracle_check(self, got):
        if self.kind == "spread":
            SO.check(got, self.fo, self.fn, self.live, self.dom)
        else:
            AO.check(got, self.fo, self.fn, self.live)

    def check(self, prev, counts, tag):
        got = self.s.read_ranked()
        assert got.shape == (len(self.fo), self.R)
        if not self.tensor:
            want = self.fresh("ffma")
            assert got.tobytes() == want.tobytes(), (tag, int((got != want).any(axis=1).sum()))
        self.oracle_check(got)
        assert (self.s.read() == got[:, 0]).all(), tag
        c0 = got[:, 0]
        hist = np.bincount(c0[c0 != NONE].astype(np.int64), minlength=len(self.fn))
        assert (self.s.counters() == hist[: len(self.fn)]).all(), tag
        if counts is not None:
            want_counts = (int((prev[:, 0] != got[:, 0]).sum()), int((prev != got).any(axis=1).sum()))
            assert tuple(counts) == want_counts, (tag, counts, want_counts)
        return got

    # ---- node-table changes, mirrored; each returns the change set (idx, prev_weight) -------------------------------------------
    def prev_of(self, js):
        return [int(self.w[j]) if self.live[j] else 0 for j in js]

    def leave(self, js):
        prev = self.prev_of(js)
        for j in js:
            self.p.node_set_active(int(j), False)
            self.live[j] = False
        return list(js), prev

    def join(self, js):
        """re-activates interned nodes (their features are kept) or interns the spares (fresh features, label of their own)"""
        prev = []
        for j in js:
            if j >= len(self.fn):
                assert j == len(self.fn)
                f = np.random.default_rng(900 + j).uniform(-1, 1, self.K).astype(np.float32)
                self.fn = np.vstack([self.fn, f[None]])
                self.w = np.append(self.w, np.uint32(1))
                self.live = np.append(self.live, False)
                self.dom = np.append(self.dom, np.uint32(NONE))
                prev.append(0)
                assert self.p.node_upsert(self.addrs[j], 1, f) == j
            else:
                prev.append(self.prev_of([j])[0])
                self.p.node_upsert(self.addrs[j], int(self.w[j]))
            self.live[j] = True
        return list(js), prev

    def reweight(self, js, factor=0.5):
        prev = self.prev_of(js)
        for j in js:
            self.w[j] = max(1, int(self.w[j] * factor))
            self.p.node_upsert(self.addrs[j], int(self.w[j]))
        return list(js), prev

    def refeature(self, js, seed=1):
        rng = np.random.default_rng(700 + seed)
        for j in js:
            self.fn[j] = rng.uniform(-1, 1, self.K).astype(np.float32)
            self.p.node_upsert(self.addrs[j], int(self.w[j]), self.fn[j])
        return [], []

    def set_nodes_refeatured(self, js, seed=2):
        """set_nodes over the live nodes with new features for js; the other interned nodes lose theirs (zeros), as set_nodes does"""
        rng = np.random.default_rng(800 + seed)
        for j in js:
            self.fn[j] = rng.uniform(-1, 1, self.K).astype(np.float32)
        on = np.flatnonzero(self.live)
        self.fn[~self.live] = 0
        self.p.set_nodes([self.addrs[j] for j in on], self.w[on], self.fn[on])
        return [], []

    def relabel(self, js, label):
        self.dom[js] = label
        self.p.set_node_domains(np.asarray(js, dtype=np.uint32), np.full(len(js), label, dtype=np.uint32))
        return [], []

    def step(self, change, tag):
        idx, prev = change
        l0 = self.p.launch_count()
        counts = self.s.rebalance_changes_ranked(idx, prev)
        self.launches = self.p.launch_count() - l0   # kernels the change set launched
        old, self.cur = self.cur, self.check(self.cur, counts, tag)
        return old, counts


def sequence(c, spread):
    """the change sets of the issue, applied one after the other; returns the number of steps"""
    M = len(c.fn)
    c0 = c.cur[:, 0]
    busy = int(np.bincount(c0[c0 != NONE].astype(np.int64)).argmax())
    steps = [
        ("one leave", lambda: c.leave([busy])),
        ("one join", lambda: c.join([busy])),
        ("a rack leaves", lambda: c.leave([int(j) for j in np.flatnonzero(c.dom[:M] == c.dom[1])][:32])),
        ("joins and leaves", lambda: (lambda a, b: (a[0] + b[0], a[1] + b[1]))(c.join([int(j) for j in np.flatnonzero(c.dom[:M] == c.dom[1])][:32]),
                                                                               c.leave([M - 2, M - 1]))),
        ("a spare joins", lambda: c.join([len(c.fn)])),
        ("node_upsert features", lambda: c.refeature([0, 5])),
        ("set_nodes features", lambda: c.set_nodes_refeatured([3, 4, M // 2])),
    ]
    if spread:
        steps.append(("relabel", lambda: c.relabel([6, 7, 8], 4242)))
    for tag, f in steps:
        c.step(f(), tag)
    # a weight-only change: nothing moves, and only the pass runs
    live_js = [int(j) for j in np.flatnonzero(c.live)[:8]]
    old, counts = c.step(c.reweight(live_js), "weights")
    assert tuple(counts) == (0, 0) and c.launches == 1
    # identical features upserted again: k = 0 finds nothing and launches nothing
    for j in live_js[:3]:
        c.p.node_upsert(c.addrs[j], int(c.w[j]), c.fn[j])
    old, counts = c.step(([], []), "same features")
    assert tuple(counts) == (0, 0) and c.launches == 0
    # every node leaves, then some rejoin
    c.step(c.leave([int(j) for j in np.flatnonzero(c.live)]), "all leave")
    assert (c.cur == NONE).all()
    c.step(c.join(list(range(0, len(c.fn), 2))), "rejoin")
    return len(steps) + 4


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("K,M,n", [(16, 9, 2000), (16, 66, 3000), (16, 1024, 5000), (16, 2307, 3000), (8, 66, 3000), (5, 9, 2000), (5, 1024, 3000)])
def test_cuda_cores_are_bit_exact(gp, oracle, K, M, n, kind):
    """RIO_AFFINITY_VARIANT=ffma: after every change set the lists equal a fresh CUDA-core call byte for byte and pass the fp64 oracle."""
    with variant("ffma"):
        c = AffCluster(gp, oracle, M, n, K, 4 if kind == "ranked" else 3, kind, "ffma", seed=M + K)
        assert not c.tensor
        sequence(c, kind == "spread")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("M", [66, 259, 1024, 2306])
def test_tensor_cores_are_within_tolerance(gp, oracle, M, kind):
    """The default path at K = 16: every state passes the oracle, and a row that holds no REPLACE member and that no candidate reaches
    within the tolerance is left byte for byte as it was.  At M = 2306 nodes 3 and M - 2 are not live: 2304 live nodes fill the
    tensor path, and the spare's join takes the S1 rows to the CUDA cores."""
    live = np.ones(M, bool)
    if M == 2306:
        live[[3, M - 2]] = False
    c = AffCluster(gp, oracle, M, 4000, 16, 4, kind, "umma", seed=M, live=live)
    assert c.tensor == (not host_sim(c.p))
    # a join of one spare: no REPLACE member anywhere; rows the new node cannot reach stay
    before = c.cur.copy()
    old, _ = c.step(c.join([len(c.fn)]), "spare joins")
    j = len(c.fn) - 1
    last = np.where(before[:, -1] == NONE, 0, before[:, -1])
    cl = AO.cost_of(c.fo, c.fn, last[:, None])[:, 0]
    cj = AO.cost_of(c.fo, c.fn, np.full((len(c.fo), 1), j, np.uint32))[:, 0]
    tol = AO.tau(c.fo, c.fn, last[:, None])[:, 0] + AO.tau(c.fo, c.fn, np.full((len(c.fo), 1), j, np.uint32))[:, 0]
    far = (before[:, -1] != NONE) & (cj > cl + tol)
    assert far.any()
    assert (c.cur[far] == before[far]).all()
    # a leave: rows without the node are S2 with no candidate, so they are untouched
    busy = int(np.bincount(c.cur[:, 0].astype(np.int64)).argmax())
    before = c.cur.copy()
    c.step(c.leave([busy]), "leave")
    untouched = ~(before == busy).any(axis=1)
    assert (c.cur[untouched] == before[untouched]).all()
    # a refeature and (spread) a relabel
    c.step(c.refeature([int(np.flatnonzero(c.live)[5])]), "refeature")
    if kind == "spread":
        c.step(c.relabel([10, 11], 777), "relabel")
    # rows agree with a fresh tensor-core call but for near-ties
    fresh = c.fresh("umma")
    assert (c.cur == fresh).all(axis=1).mean() >= 0.999


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_path_crossing(gp, oracle, kind):
    """A tensor-core set whose joins push the padded live count past 2304 recomputes on the CUDA cores and still passes the oracle; a
    CUDA-core set (2307 live) stays on the CUDA cores after leaves bring it under 2304, and stays bit-exact against ffma."""
    c = AffCluster(gp, oracle, 2300, 3000, 16, 3, kind, "umma", seed=1, spare=8)
    for _ in range(6):
        c.step(c.join([len(c.fn)]), "spare joins")
    assert not tensor_cores(c.p, "umma", 16, int(c.live.sum()))
    busy = int(np.bincount(c.cur[:, 0].astype(np.int64)).argmax())
    c.step(c.leave([busy]), "leave past the tensor-core limit")
    d = AffCluster(gp, oracle, 2307, 3000, 16, 3, kind, "umma", seed=2)
    assert not d.tensor
    c0 = d.cur[:, 0]
    top = [int(j) for j in np.argsort(-np.bincount(c0.astype(np.int64), minlength=2307))[:4]]
    d.step(d.leave(top), "leaves under 2304")   # check() compares with ffma byte for byte
    d.step(d.join([top[0]]), "rejoin")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_launch_counts(gp, oracle, kind):
    with variant("ffma"):
        c = AffCluster(gp, oracle, 256, 4000, 16, 2, kind, "ffma", seed=3)
        c.step(c.reweight([1, 2]), "no candidate")
        assert c.launches == 1
        busy = int(np.bincount(c.cur[:, 0].astype(np.int64)).argmax())
        c.step(c.leave([busy]), "leave")
        assert c.launches == 4   # pass, gather, list kernel, scatter
        c.step(([], []), "nothing")
        assert c.launches == 0


@pytest.mark.gpu
def test_interaction_and_errors(gp, oracle):
    with variant("ffma"):
        c = AffCluster(gp, oracle, 128, 3000, 16, 3, "ranked", "ffma", seed=4)
        p, s = c.p, c.s
        # a solver change is accepted: the affinity lists do not depend on it
        p.set_solver("hrw2", 0)
        c.step(c.leave([7]), "solver changed")
        p.set_solver("hrw", 0)
        # commit writes column 0
        s.commit()
        keys, idx = s.read(want_keys=True)
        assert (p.lookup_many(keys) == c.cur[:, 0]).all() and (idx == c.cur[:, 0]).all()
        # argument errors
        for r in (0, 9):
            with pytest.raises(gp.Unknown):
                s.assign_ranked_affinity(r)
            with pytest.raises(gp.Unknown):
                s.assign_ranked_affinity_spread(r)
        with pytest.raises(gp.Unknown):
            s.rebalance_changes_ranked([10**6], [0])
        with pytest.raises(gp.Unknown):
            s.rebalance_changes_ranked([7, 7], [0, 0])
        assert (s.read_ranked() == c.cur).all()
        # hash sets of the same handle, plain and failure-domain, next to it
        h1, h2 = p.new_set(2000), p.new_set(2000)
        for h in (h1, h2):
            h.synth_keys(0, 2000, 9)
        h1.assign_ranked(3)
        h2.assign_ranked_spread(3)
        hk = h1.read(want_keys=True)[0]
        c.step(c.join([7]), "join beside hash sets")
        for h, call in ((h1, p.assign_ranked), (h2, p.assign_ranked_spread)):
            h.rebalance_changes_ranked([7], [0])
            assert (h.read_ranked() == call(hk, 3)).all()
        # set_load_feats drops affinity lists, not hash lists
        h1.load_feats(c.fo[:2000])
        assert (h1.read_ranked() == p.assign_ranked(hk, 3)).all()
        s.load_feats(c.fo)
        with pytest.raises(gp.Unknown):
            s.read_ranked()
        # kinds switch either way
        s.assign_ranked(3)
        assert (s.read_ranked() == p.assign_ranked(s.read(want_keys=True)[0], 3)).all()
        s.assign_ranked_affinity_spread(3)
        c.kind = "spread"
        c.cur = c.check(c.cur, None, "switched to spread")
        c.step(c.leave([8]), "spread leave")
        # a K change between assign and change set is refused; the lists stay
        keep = s.read_ranked()
        on = np.flatnonzero(c.live)
        p.set_nodes([c.addrs[j] for j in on], c.w[on], np.ones((len(on), 8), np.float32))
        with pytest.raises(gp.Unknown, match="assign the lists again"):
            s.rebalance_changes_ranked([], [])
        assert (s.read_ranked() == keep).all()
        # set features of another K than the handle's, and a handle without node features
        with pytest.raises(gp.Unknown, match="different K"):
            s.assign_ranked_affinity(2)
        q = gp.GpuObjectPlacement()
        q.set_nodes(c.addrs[:8])
        t = q.new_set(10)
        t.synth_keys(0, 10, 1)
        t.load_feats(np.ones((10, 16), np.float32))
        with pytest.raises(gp.Unknown, match="needs node features"):
            t.assign_ranked_affinity(2)
        u = p.new_set(10)
        u.synth_keys(0, 10, 1)
        with pytest.raises(gp.Unknown, match="missing"):
            u.assign_ranked_affinity_spread(2)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_one_million_objects(gp, oracle, kind):
    """1 M objects x 1024 nodes x K = 16 at R = 4 in 32 racks (20 k objects on the host-sim): one rack leaves and one node is
    refeatured, on the default path; the first 200 k lists are checked with the oracle."""
    p0 = gp.GpuObjectPlacement()
    n = 20_000 if host_sim(p0) else 1_000_000
    c = AffCluster.__new__(AffCluster)
    c.gp, c.oracle, c.K, c.R, c.kind, c.var = gp, oracle, 16, 4, kind, "umma"
    rng = np.random.default_rng(77)
    c.fo = rng.uniform(-1, 1, (n, 16)).astype(np.float32)
    c.fn = rng.uniform(-1, 1, (1024, 16)).astype(np.float32)
    c.addrs = oracle.synth_nodes(1024)[0]
    c.w = np.ones(1024, np.uint32)
    c.live = np.ones(1024, bool)
    c.dom = racks(1024)
    c.p = gp.GpuObjectPlacement()
    c.p.set_nodes(c.addrs, c.w, c.fn)
    c.p.set_node_domains(np.arange(1024, dtype=np.uint32), c.dom)
    c.s = c.p.new_set(n)
    c.s.synth_keys(0, n, 5)
    c.s.load_feats(c.fo)
    c.assign()
    c.tensor = tensor_cores(c.p, "umma", 16, 1024)
    c.cur = c.s.read_ranked()
    c.refeature([500])
    idx, prev = c.leave([int(j) for j in np.flatnonzero(c.dom == 3)])
    moved, changed = c.s.rebalance_changes_ranked(idx, prev)
    got = c.s.read_ranked()
    assert (moved, changed) == (int((got[:, 0] != c.cur[:, 0]).sum()), int((got != c.cur).any(axis=1).sum()))
    assert (c.s.read() == got[:, 0]).all() and (got != NONE).all() and not np.isin(got, idx).any()
    m = min(n, 200_000)
    if kind == "spread":
        SO.check(got[:m], c.fo[:m], c.fn, c.live, c.dom)
    else:
        AO.check(got[:m], c.fo[:m], c.fn, c.live)
    if not c.tensor:
        assert got.tobytes() == c.fresh("ffma").tobytes()


DOUBLES = os.path.join(ROOT, "tests", "cpp", "hostsim", "affinity_set_launchers.cpp")
OTHER_DOUBLES = [os.path.join(ROOT, "tests", "cpp", "hostsim", f) for f in ("ranked_launchers.cpp", "change_launchers.cpp", "ranked_change_launchers.cpp",
                                                                              "spread_launchers.cpp", "spread_change_launchers.cpp",
                                                                              "affinity_ranked_launchers.cpp", "affinity_spread_launchers.cpp")]


def test_the_doubles_cover_every_affinity_set_launcher():
    decl = set(re.findall(r"\b(launch_[a-z0-9_]+)\s*\(", open(os.path.join(CSRC, "k_affinity_set.cuh")).read()))
    have = set(re.findall(r"^void\s+([a-z0-9_]+)\s*\(", open(DOUBLES).read(), flags=re.M))
    assert len(decl) == 2 and decl <= have, decl - have


def _hostsim_library(HS, name, doubles):
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, name)
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + doubles + ["-o", so, "-ldl", "-lpthread"])
    return so


def test_affinity_set_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + every ranked, set and
    affinity double)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_set_affinity.so", OTHER_DOUBLES + [DOUBLES])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=3000, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 29 and "failed" not in r.stdout, tail


def test_affinity_sets_report_an_error_where_the_kernels_are_not_linked():
    """The engine's host code built WITHOUT the affinity-set launchers loads, refuses both affinity-set calls with RIO_ERR_UPSTREAM and a
    message, and still serves the batch affinity calls and hash-policy ranked sets."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_no_affinity_sets.so", OTHER_DOUBLES)
    code = (
        "import sys, numpy as np\n"
        "from rio_rs_b200 import _native as N\n"
        "N.library_path = lambda: sys.argv[1]\n"
        "import rio_rs_b200 as R\n"
        "p = R.GpuObjectPlacement()\n"
        "fn = np.random.default_rng(1).uniform(-1, 1, (8, 16)).astype(np.float32)\n"
        "fo = np.random.default_rng(2).uniform(-1, 1, (100, 16)).astype(np.float32)\n"
        "p.set_nodes(['10.0.0.%d:5000' % j for j in range(8)], None, fn)\n"
        "s = p.new_set(100); s.synth_keys(0, 100, 1); s.load_feats(fo)\n"
        "for call in (s.assign_ranked_affinity, s.assign_ranked_affinity_spread):\n"
        "    try:\n"
        "        call(2)\n"
        "        raise SystemExit('computed without kernels')\n"
        "    except R.Upstream as e:\n"
        "        assert 'affinity-set kernels' in str(e), e\n"
        "assert (p.assign_ranked_affinity(fo, 2)[:, 0] == p.assign_batch(obj_feats=fo)).all()\n"
        "s.assign_ranked(2)\n"
        "keys = s.read(want_keys=True)[0]\n"
        "p.node_set_active(3, False)\n"
        "s.rebalance_changes_ranked([3], [1])\n"
        "assert (s.read_ranked() == p.assign_ranked(keys, 2)).all()\n"
        "print('refused ok')\n"
    )
    r = subprocess.run([sys.executable, "-c", code, so], capture_output=True, text=True, timeout=300, cwd=HS.ROOT)
    assert r.returncode == 0 and "refused ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

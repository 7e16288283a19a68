"""Object churn in resident sets (DESIGN.md 3.18): ObjectSet.insert and ObjectSet.erase against tests/set_churn_oracle.py.

* After every call of a seeded sequence of inserts and erases, for every kind a set can hold (unassigned; plain hash under HRW and
  HRW2 at 12 and 5 trie bits; plain affinity on the CUDA cores at K = 8, 16, 24 and on the tensor cores; ranked and failure-domain
  lists under both policies; ranked and failure-domain affinity lists on both paths; bounded hash; bounded affinity), the set's keys,
  idx, lists, counters and size and the calls' out_first / out_erased equal the oracle bit for bit.  The oracle places a new row with
  the handle's own batch call of the set's kind.
* The movement contract is checked directly: an insert leaves rows [0, n) byte for byte, an erase keeps every surviving row's (key,
  node, list) and only moves rows.
* Fixed point: for the history-free kinds, churn then a change set equals a twin set loaded with the final rows and assigned afresh.
* Bounded affinity: after inserts, the k = 0 change-set call equals tests/affinity_set_bounded_oracle.py from that state.
* Every refusal leaves the set byte for byte as it was.

The CPU tests at the end run this module's GPU bodies, unchanged, against the engine's host logic compiled with g++ (the host-sim
library of tests/test_engine_host_sim.py) with a plain restatement of the new launchers, and check that a build without them refuses
both calls while every other call keeps working.  There the tensor path is never taken."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import affinity_bounded_oracle as BO
import affinity_set_bounded_oracle as SB
import set_churn_oracle as O

NONE = 0xFFFFFFFF
SENTINEL = 0xFFFFFFFFFFFFFFFF
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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


def addresses(M):
    return ["10.3.%d.%d:7000" % (j >> 8, j & 255) for j in range(M)]


LIST_KINDS = ("ranked", "spread", "ranked_affinity", "spread_affinity")


class Churn:
    """A handle, a set of `kind` on it and the set's shadow.  `dead` nodes start inactive."""

    def __init__(self, gp, kind, M=48, K=0, solver="hrw", bits=12, var="umma", R=3, cap=3000, n0=1001, seed=0, dead=()):
        self.gp, self.kind, self.K, self.var, self.R, self.cap = gp, kind, K, var, R, cap
        self.rng = np.random.default_rng(700 + seed)
        self.M = M
        self.fn = self.rng.uniform(-1, 1, (M, K)).astype(np.float32) if K else None
        self.w = self.rng.integers(1, 17, M).astype(np.uint32)
        self.p = gp.GpuObjectPlacement()
        self.p.set_solver(solver, bits)
        self.p.set_nodes(addresses(M), self.w, self.fn)
        for j in dead:
            self.p.node_set_active(int(j), False)
        if kind in ("spread", "spread_affinity"):
            self.p.set_node_domains(np.arange(M), np.arange(M) // 4)
        self.s = self.p.new_set(cap)
        keys = self.keys(n0)
        self.s.load_keys(keys)
        fo = self.feats(n0) if K else None
        if K:
            self.s.load_feats(fo)
        with variant(var):
            {
                "none": lambda: None,
                "hash": lambda: self.s.assign(False),
                "affinity": lambda: self.s.assign(True),
                "ranked": lambda: self.s.assign_ranked(R),
                "spread": lambda: self.s.assign_ranked_spread(R),
                "ranked_affinity": lambda: self.s.assign_ranked_affinity(R),
                "spread_affinity": lambda: self.s.assign_ranked_affinity_spread(R),
                "bounded": lambda: self.s.assign_bounded(0, 5, 4, 4),
                "bounded_affinity": lambda: self.s.assign_bounded_affinity(0, 5, 4, 4),
            }[kind]()
        k, idx = self.s.read(want_keys=True)
        assert k.tobytes() == keys.tobytes()
        lists = self.s.read_ranked() if kind in LIST_KINDS else None
        cnt = self.s.counters() if kind != "none" else np.zeros(M, np.int64)
        self.sh = O.Shadow(keys, idx, lists, fo, cnt, kind != "none")

    def keys(self, m):
        return self.rng.integers(0, 2**63, m, dtype=np.uint64) * np.uint64(2) + self.rng.integers(0, 2, m, dtype=np.uint64)

    def feats(self, m):
        return self.rng.uniform(-1, 1, (m, self.K)).astype(np.float32)

    def place(self, keys, feats):
        """the batch call of the set's kind for fresh rows, over the handle's current table"""
        p, R = self.p, self.R
        with variant(self.var):
            if self.kind in ("hash", "bounded"):
                return p.assign_batch(keys), None
            if self.kind in ("affinity", "bounded_affinity"):
                return p.assign_batch(obj_feats=feats), None
            lists = {
                "ranked": lambda: p.assign_ranked(keys, R),
                "spread": lambda: p.assign_ranked_spread(keys, R),
                "ranked_affinity": lambda: p.assign_ranked_affinity(feats, R),
                "spread_affinity": lambda: p.assign_ranked_affinity_spread(feats, R),
            }[self.kind]()
            return lists[:, 0].copy(), lists

    def state(self):
        """everything the set shows: keys, idx, lists, counters, size"""
        n = self.s.size()
        k, idx = self.s.read(want_keys=True)
        lists = self.s.read_ranked() if self.kind in LIST_KINDS else None
        return n, k, idx, lists, self.s.counters()

    def check(self, tag):
        n, k, idx, lists, cnt = self.state()
        sh = self.sh
        assert n == sh.n, (tag, n, sh.n)
        assert k.tobytes() == sh.keys.tobytes(), tag
        assert idx.tobytes() == sh.idx.tobytes(), (tag, int((idx != sh.idx).sum()))
        if lists is not None:
            assert lists.tobytes() == sh.lists.tobytes(), tag
        sh.grow_counters(len(cnt))
        assert (cnt.astype(np.int64) == sh.counters).all(), tag
        if self.kind != "none":
            assert (cnt.astype(np.int64) == O.counts(idx, len(cnt))).all(), tag

    def resync(self):
        """the shadow takes the set's nodes, lists and counters after a call it does not model (a change set)"""
        _, _, self.sh.idx, self.sh.lists, cnt = self.state()
        self.sh.counters = cnt.astype(np.int64)

    # ---- the two calls, each against the oracle, with the movement contract checked directly -------------------------------
    def insert(self, keys, tag, feats=None):
        keys = np.asarray(keys, dtype=np.uint64)
        if self.K and feats is None:
            feats = self.feats(len(keys))
        before = self.state()
        first = self.s.insert(keys, feats)   # outside variant(): the set's recorded path decides, not the environment
        want = self.sh.insert(keys, feats, self.place, self.p.node_count()[0])
        assert first == want == before[0], tag
        after = self.state()
        n0 = before[0]
        assert after[1][:n0].tobytes() == before[1].tobytes() and after[2][:n0].tobytes() == before[2].tobytes(), tag
        if before[3] is not None:
            assert after[3][:n0].tobytes() == before[3].tobytes(), tag
        self.check(tag)

    def erase(self, keys, tag):
        keys = np.asarray(keys, dtype=np.uint64)
        before = self.state()
        got = self.s.erase(keys)
        want = self.sh.erase(keys, self.p.node_count()[0])
        assert got == want, (tag, got, want)
        after = self.state()
        # every surviving row keeps its key, node and list; only its position may change
        keep = ~np.isin(before[1], keys)
        assert rows(before[1][keep], before[2][keep], None if before[3] is None else before[3][keep]) == rows(*after[1:4]), tag
        self.check(tag)

    def present(self, m):
        return self.rng.choice(self.sh.keys, size=min(m, self.sh.n), replace=False) if self.sh.n else np.zeros(0, np.uint64)


def rows(keys, idx, lists):
    """the set's rows as a sorted list of (key, node, list): what an erase must keep, whatever it moves"""
    lists = [()] * len(keys) if lists is None else [tuple(r) for r in lists.tolist()]
    return sorted(zip(keys.tolist(), idx.tolist(), lists))


def sequence(c):
    """the churn of DESIGN.md 3.18's tests, one call after the other; the set starts at an odd n"""
    c.insert(c.keys(37), "insert at odd n")
    c.insert(c.keys(1), "insert one row")
    c.insert([], "insert nothing")
    c.erase([], "erase nothing")
    c.erase(np.concatenate([c.present(120), c.keys(30)]), "erase present and absent keys")
    dup = c.present(5)
    c.insert(np.concatenate([dup, dup[:2]]), "insert keys already in the set")
    c.erase(np.concatenate([dup[:3], dup[:3], dup[3:4]]), "erase duplicated keys, listed twice")
    c.erase(c.keys(50), "erase keys not present")
    c.insert([SENTINEL, 7], "insert the hash set's empty key")
    c.erase([SENTINEL], "erase the hash set's empty key")
    c.erase([SENTINEL, 7], "erase the empty key when it is absent")
    if c.kind != "none":
        busy = int(np.bincount(c.sh.idx[c.sh.idx != NONE].astype(np.int64)).argmax())
        c.erase(c.sh.keys[c.sh.idx == busy], "erase all the objects of one node")
    c.erase(c.present(c.sh.n // 3)[::2], "erase a sixth")
    c.insert(c.keys(c.cap - c.sh.n), "insert up to exactly capacity")
    assert c.s.size() == c.cap
    with pytest.raises(c.gp.Unknown):
        c.s.insert(c.keys(1), c.feats(1) if c.K else None)
    c.check("a refused insert past capacity")
    c.erase(c.sh.keys, "erase all")
    assert c.s.size() == 0
    c.erase(c.keys(3), "erase from an empty set")
    c.insert(c.keys(65), "insert into the emptied set")


KINDS = [
    ("none", {}),
    ("none", dict(K=8)),
    ("hash", dict(solver="hrw")),
    ("hash", dict(solver="hrw2", bits=12)),
    ("hash", dict(solver="hrw2", bits=5)),
    ("affinity", dict(K=8, var="ffma")),
    ("affinity", dict(K=16, var="ffma")),
    ("affinity", dict(K=24, var="ffma")),
    ("affinity", dict(K=16, var="umma")),
    ("ranked", dict(solver="hrw")),
    ("ranked", dict(solver="hrw2", bits=5)),
    ("spread", dict(solver="hrw")),
    ("spread", dict(solver="hrw2", bits=12)),
    ("ranked_affinity", dict(K=16, var="umma")),
    ("ranked_affinity", dict(K=16, var="ffma")),
    ("ranked_affinity", dict(K=8, var="ffma")),
    ("spread_affinity", dict(K=16, var="umma")),
    ("spread_affinity", dict(K=16, var="ffma")),
    ("bounded", dict(solver="hrw")),
    ("bounded", dict(solver="hrw2", bits=12)),
    ("bounded_affinity", dict(K=16, var="umma")),
    ("bounded_affinity", dict(K=8, var="ffma")),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,opts", KINDS, ids=["%s-%s" % (k, "-".join("%s%s" % kv for kv in o.items())) for k, o in KINDS])
def test_churn_equals_the_oracle(gp, kind, opts):
    c = Churn(gp, kind, seed=len(kind) + opts.get("K", 0) + opts.get("bits", 0), dead=(3,), **opts)
    sequence(c)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["affinity", "ranked_affinity", "spread_affinity", "bounded_affinity"])
@pytest.mark.parametrize("M", [65, 257, 2305])
def test_live_counts_across_the_launcher_thresholds(gp, kind, M):
    """A tensor-core set with 64 / 256 / 2304 live nodes: a node joins (65 / 257 / 2305 live: a padding step, or the CUDA cores for
    2305), then two leave; the inserts between are placed over the table of the moment, as the batch call places them."""
    c = Churn(gp, kind, M=M, K=16, var="umma", cap=1200, n0=301, seed=M, dead=(M - 1,))
    c.insert(c.keys(41), "%d live" % (M - 1))
    c.p.node_set_active(M - 1, True)
    c.insert(c.keys(41), "%d live" % M)
    c.erase(c.present(60), "erase at %d live" % M)
    c.p.node_set_active(M - 1, False)
    c.p.node_set_active(M - 2, False)
    c.insert(c.keys(41), "%d live" % (M - 2))
    c.erase(c.present(60), "erase at %d live" % (M - 2))


def _churn(c):
    c.insert(c.keys(57), "insert")
    c.erase(np.concatenate([c.present(200), c.keys(10)]), "erase")
    c.insert(c.keys(3), "insert at odd n")


FIXED = [
    ("hash", dict(solver="hrw")),
    ("hash", dict(solver="hrw2", bits=12)),
    ("ranked", dict(solver="hrw")),
    ("ranked", dict(solver="hrw2", bits=12)),
    ("spread", dict(solver="hrw")),
    ("spread", dict(solver="hrw2", bits=5)),
    ("ranked_affinity", dict(K=16, var="ffma")),
    ("ranked_affinity", dict(K=24, var="ffma")),
    ("spread_affinity", dict(K=8, var="ffma")),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,opts", FIXED, ids=["%s-%s" % (k, "-".join("%s%s" % kv for kv in o.items())) for k, o in FIXED])
def test_churn_then_a_change_set_equals_a_fresh_assign(gp, kind, opts):
    """History-free kinds: after churn and a change set (a leave, a join, a weight change), the set equals a twin loaded with the
    final rows in the final order and assigned from scratch: the new rows were fresh rows, and the erase moved feature rows along."""
    c = Churn(gp, kind, seed=31 + len(kind), dead=(5,), **opts)
    _churn(c)
    prev = [int(c.w[j]) for j in (2, 5, 9)]
    c.p.node_set_active(2, False)
    c.p.node_upsert(addresses(c.M)[5], int(c.w[5]))
    c.p.node_upsert(addresses(c.M)[9], int(c.w[9]) * 3)
    change = ([2, 5, 9], [prev[0], 0, prev[2]])
    with variant(c.var):
        if kind == "hash":
            c.s.rebalance_changes(*change)
        else:
            c.s.rebalance_changes_ranked(*change)
    c.resync()
    _churn(c)
    twin = c.p.new_set(c.cap)
    k, idx = c.s.read(want_keys=True)
    twin.load_keys(k)
    if c.K:
        twin.load_feats(c.sh.feats)
    with variant(c.var):
        {"hash": lambda: twin.assign(False), "ranked": lambda: twin.assign_ranked(c.R), "spread": lambda: twin.assign_ranked_spread(c.R),
         "ranked_affinity": lambda: twin.assign_ranked_affinity(c.R), "spread_affinity": lambda: twin.assign_ranked_affinity_spread(c.R)}[kind]()
    assert twin.read().tobytes() == idx.tobytes()
    if kind in LIST_KINDS:
        assert twin.read_ranked().tobytes() == c.s.read_ranked().tobytes()
    assert (twin.counters() == c.s.counters()).all()


@pytest.mark.gpu
@pytest.mark.parametrize("K", [8, 16])
def test_bounded_affinity_after_inserts_is_brought_back_by_k0(gp, K):
    """Inserts onto a bounded affinity set are plain argmin rows; the k = 0 change-set call then runs the capacity rounds from that
    state, as tests/affinity_set_bounded_oracle.py does (the CUDA cores: exact c32)."""
    c = Churn(gp, "bounded_affinity", K=K, var="ffma", n0=2001, cap=6000, seed=K)
    fn = c.fn
    live = np.ones(c.M, bool)
    for r in range(3):
        hot = np.repeat(fn[r][None], 400, axis=0)   # 400 objects that all prefer one node: it goes over capacity
        c.insert(c.keys(400), "insert onto node %d" % r, feats=hot)
        c.erase(c.present(150), "erase")
        want = SB.rebalance(c.sh.keys, c.sh.idx, c.sh.feats, fn, BO.c32_argmin(c.sh.feats, fn), ~live, [], c.w, live, live, 0, 5, 4, 16)
        moved, passes = c.s.rebalance_changes_bounded_affinity([], [], 0, 5, 4, 16)
        got = c.s.read()
        assert got.tobytes() == want["idx"].tobytes(), r
        assert (moved, passes) == (want["moved"], want["passes"]) and passes > 1, r
        assert (c.s.counters() == want["counters"]).all()
        c.sh.idx, c.sh.counters = got.copy(), want["counters"].astype(np.int64)


@pytest.mark.gpu
def test_records_survive_churn(gp):
    """The lists' and the bounded record's change-set calls still accept a set after inserts and erases."""
    for kind, opts in (("ranked", {}), ("spread_affinity", dict(K=16)), ("bounded_affinity", dict(K=16))):
        c = Churn(gp, kind, seed=5, **opts)
        _churn(c)
        c.p.node_set_active(1, False)
        if kind == "bounded_affinity":
            c.s.rebalance_changes_bounded_affinity([1], [int(c.w[1])])
        else:
            c.s.rebalance_changes_ranked([1], [int(c.w[1])])
        assert not (c.s.read() == 1).any()
        c.resync()
        _churn(c)


@pytest.mark.gpu
def test_errors_change_nothing(gp):
    R = gp
    L = gp.GpuObjectPlacement().L
    assert L.rio_cuda_set_insert(None, None, None, 0, None) != 0
    assert L.rio_cuda_set_erase(None, None, 0, None) != 0

    def refused(c, call, tag):
        before = c.state()
        with pytest.raises(R.Unknown):
            call()
        after = c.state()
        assert before[0] == after[0] and all(a.tobytes() == b.tobytes() for a, b in zip(before[1:4], after[1:4]) if a is not None), tag
        assert (before[4] == after[4]).all(), tag

    c = Churn(gp, "ranked", K=8, seed=1)
    s = c.s
    refused(c, lambda: c.s._ck(L.rio_cuda_set_insert(s.s, None, None, 3, None)), "insert: null keys")
    refused(c, lambda: c.s._ck(L.rio_cuda_set_erase(s.s, None, 3, None)), "erase: null keys")
    refused(c, lambda: s.insert(c.keys(3)), "features missing")
    refused(c, lambda: s.insert(c.keys(c.cap - c.sh.n + 1), c.feats(c.cap - c.sh.n + 1)), "past capacity")
    c.p.set_solver("hrw2", 12)
    refused(c, lambda: s.insert(c.keys(3), c.feats(3)), "lists under another solver")
    c.p.set_solver("hrw", 12)
    c.insert(c.keys(3), "the solver is back: the insert goes through")
    # a set without features refuses features
    h = Churn(gp, "hash", seed=2)
    refused(h, lambda: h.s.insert(h.keys(2), np.zeros((2, 4), np.float32)), "features given to a set without them")
    # a bounded call in flight
    b = Churn(gp, "bounded", seed=3)
    b.s.assign_bounded_begin(0, 5, 4, 4)
    refused(b, lambda: b.s.insert(b.keys(2)), "insert during a bounded call")
    refused(b, lambda: b.s.erase(b.present(2)), "erase during a bounded call")
    b.s.assign_bounded_end()
    # an affinity kind, a bounded record and a plain affinity set under another handle K
    for kind in ("ranked_affinity", "bounded_affinity", "affinity"):
        a = Churn(gp, kind, K=16, seed=4)
        a.p.set_nodes(addresses(a.M), a.w, np.ones((a.M, 8), np.float32))
        refused(a, lambda: a.s.insert(a.keys(2), a.feats(2)), kind + " under another K")
        a.erase(a.present(20), kind + ": erase needs no placement")
    # m = 0 does nothing, whatever the arguments
    assert c.s.insert(np.zeros(0, np.uint64)) == c.sh.n and c.s.erase(np.zeros(0, np.uint64)) == 0
    c.check("m = 0")


# ---- host-sim --------------------------------------------------------------------------------------------------------------------
DOUBLES = os.path.join(ROOT, "tests", "cpp", "hostsim", "set_churn_launchers.cpp")
OTHER_DOUBLES = [os.path.join(ROOT, "tests", "cpp", "hostsim", f) for f in ("ranked_launchers.cpp", "change_launchers.cpp", "ranked_change_launchers.cpp",
                                                                              "spread_launchers.cpp", "spread_change_launchers.cpp",
                                                                              "affinity_ranked_launchers.cpp", "affinity_spread_launchers.cpp",
                                                                              "affinity_set_launchers.cpp", "affinity_bounded_launchers.cpp",
                                                                              "set_bounded_affinity_launchers.cpp")]


def test_the_doubles_cover_the_new_launchers():
    decl = set(re.findall(r"\b(launch_[a-z0-9_]+)\s*\(", open(os.path.join(ROOT, "rio_rs_b200", "csrc", "k_set_churn.cuh")).read()))
    have = set(re.findall(r"^void\s+([a-z0-9_]+)\s*\(", open(DOUBLES).read(), flags=re.M))
    assert len(decl) == 4 and decl <= have, decl - have


def _hostsim_library(HS, name, doubles):
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, name)
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + doubles + ["-o", so, "-ldl", "-lpthread"])
    return so


def test_set_churn_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + every double, the new one
    included)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_set_churn.so", OTHER_DOUBLES + [DOUBLES])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=3000, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 47 and "failed" not in r.stdout, tail


def test_the_new_calls_report_an_error_where_their_kernels_are_not_linked():
    """The engine's host code built WITHOUT the new launchers loads, refuses insert and erase with RIO_ERR_UPSTREAM and a message, and
    still serves the set's other calls."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_no_set_churn.so", OTHER_DOUBLES)
    code = (
        "import sys, numpy as np\n"
        "from rio_rs_b200 import _native as N\n"
        "N.library_path = lambda: sys.argv[1]\n"
        "import rio_rs_b200 as R\n"
        "p = R.GpuObjectPlacement()\n"
        "p.set_nodes(['10.0.0.%d:5000' % j for j in range(8)])\n"
        "keys = np.arange(100, dtype=np.uint64)\n"
        "s = p.new_set(200); s.load_keys(keys); s.assign_ranked(2)\n"
        "for call in (lambda: s.insert(keys[:3] + 1000), lambda: s.erase(keys[:3])):\n"
        "    try:\n"
        "        call()\n"
        "        raise SystemExit('ran without kernels')\n"
        "    except R.Upstream as e:\n"
        "        assert 'set churn kernels' in str(e), e\n"
        "assert s.size() == 100 and (s.read_ranked() == p.assign_ranked(keys, 2)).all()\n"
        "p.node_set_active(3, False)\n"
        "s.rebalance_changes_ranked([3], [1])\n"
        "assert (s.read_ranked() == p.assign_ranked(keys, 2)).all()\n"
        "print('refused ok')\n"
    )
    r = subprocess.run([sys.executable, "-c", code, so], capture_output=True, text=True, timeout=300, cwd=HS.ROOT)
    assert r.returncode == 0 and "refused ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

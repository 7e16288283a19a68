"""Delta commit of a resident set (DESIGN.md 3.20): ObjectSet.commit_changes against tests/set_commit_oracle.py.

* Every call's manifest (rows, keys, from, to) and out_n equal the oracle bit for bit, the oracle reading the directory with
  lookup_many before the call.  After every call the directory answers for every key the test ever wrote (set keys, erased keys, keys
  of other writers) and for foreign keys as the oracle's model does, and its placed count is the model's.
* Scenarios: the first commit into an empty directory; a call with nothing changed; change sets under flat HRW and HRW2 (a leave, a
  join, a rack, a weight decrease); every node inactive; bounded rounds at cap 101/100; a bounded affinity change set on the CUDA
  cores; weighted bounded rounds with hot objects; a ranked set's change set; churn; other writers between commits; duplicate keys,
  the directory's reserved key beside its neighbour, and a directory that grows during the call.
* Equivalence: a twin handle with the same history running set_commit ends with the same lookups and placed count.
* Dry run: the manifest equals the real call that follows, and the directory is unchanged.  Refusals change nothing.
* On the GPU, 2 M objects x 1024 nodes: after one leave the manifest is the numpy diff of set_read before and after the event.

The CPU tests at the end run this module's GPU bodies, unchanged, against the engine's host logic compiled with g++ (the host-sim
library of tests/test_engine_host_sim.py) with a plain restatement of the new launchers, and check that a build without them refuses
the call while set_commit keeps working."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import set_commit_oracle as O

NONE = 0xFFFFFFFF
EMPTY = 0xFFFFFFFFFFFFFFFF
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gp():
    from rio_rs_b200 import build

    build.build()
    import rio_rs_b200 as R

    return R


def host_sim(p):
    return p.device_info()["name"].startswith("host-sim")


def addresses(M):
    return ["10.4.%d.%d:7000" % (j >> 8, j & 255) for j in range(M)]


class Rig:
    """A handle, a set on it, and every key the test has put anywhere in the directory."""

    def __init__(self, gp, M=48, solver="hrw", bits=12, K=0, n=3001, cap=6000, seed=0, keys=None, dir_cap=0):
        self.gp, self.M, self.K = gp, M, K
        self.rng = np.random.default_rng(900 + seed)
        self.w = self.rng.integers(1, 17, M).astype(np.uint32)
        self.fn = self.rng.uniform(-1, 1, (M, K)).astype(np.float32) if K else None
        self.p = gp.GpuObjectPlacement(directory_capacity=dir_cap)
        self.p.set_solver(solver, bits)
        self.p.set_nodes(addresses(M), self.w, self.fn)
        self.s = self.p.new_set(cap)
        keys = self.keys(n) if keys is None else np.asarray(keys, np.uint64)
        self.s.load_keys(keys)
        if K:
            self.feats = self.rng.uniform(-1, 1, (len(keys), K)).astype(np.float32)
            self.s.load_feats(self.feats)
        self.seen = keys.copy()
        self.foreign = self.keys(64)

    def keys(self, m):
        return self.rng.integers(0, 2**63, m, dtype=np.uint64) * np.uint64(2) + self.rng.integers(0, 2, m, dtype=np.uint64)

    def saw(self, keys):
        self.seen = np.concatenate([self.seen, np.asarray(keys, np.uint64)])

    def probe(self):
        return np.concatenate([self.seen, self.foreign])

    def model(self):
        pr = self.probe()
        return O.Directory(pr, self.p.lookup_many(pr))

    def placed(self, model):
        return sum(1 for v in model.d.values() if v != NONE)

    def commit(self, tag, dry_run=False):
        """commit_changes against the oracle; returns the manifest"""
        keys, idx = self.s.read(want_keys=True)
        self.saw(keys)
        model = self.model()
        assert self.p.directory_len()[0] == self.placed(model), tag
        before = self.p.lookup_many(self.probe()), self.p.directory_len()
        want = model.commit(keys, idx, dry_run)
        got = self.s.commit_changes(dry_run=dry_run)
        for g, w_, name in zip(got, want, ("rows", "keys", "from", "to")):
            assert g.dtype == w_.dtype and g.tobytes() == w_.tobytes(), (tag, name, len(g), len(w_))
        after = self.p.lookup_many(self.probe())
        assert after.tobytes() == model.answer(self.probe()).tobytes(), (tag, int((after != model.answer(self.probe())).sum()))
        assert self.p.directory_len()[0] == self.placed(model), tag
        if dry_run:
            assert after.tobytes() == before[0].tobytes() and self.p.directory_len() == before[1], tag
        return got

    def commit_dry_then_real(self, tag):
        dry = self.commit(tag + " (dry run)", dry_run=True)
        real = self.commit(tag)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(dry, real)), tag
        return real

    def leave(self, js):
        prev = [int(self.w[j]) for j in js]
        for j in js:
            self.p.node_set_active(int(j), False)
        return list(js), prev


def _history(r, commit):
    """a first commit, then change sets of every kind under the handle's policy, each followed by a commit"""
    commit("first commit")
    commit("nothing changed")
    r.s.rebalance_changes(*r.leave([3]))
    commit("a leave")
    r.p.node_set_active(3, True)
    r.s.rebalance_changes([3], [0])
    commit("the node joins back")
    j = r.p.node_upsert("10.9.0.1:7000", 9)
    r.s.rebalance_changes([j], [0])
    commit("a new node joins")
    r.s.rebalance_changes(*r.leave(range(8, 16)))
    commit("a rack of 8 leaves")
    prev = int(r.w[20])
    r.p.node_upsert(addresses(r.M)[20], max(1, prev // 4))
    r.s.rebalance_changes([20], [prev])
    commit("a weight decrease")


POLICIES = [dict(solver="hrw"), dict(solver="hrw2", bits=12), dict(solver="hrw2", bits=5)]


@pytest.mark.gpu
@pytest.mark.parametrize("opts", POLICIES, ids=["hrw", "hrw2-12", "hrw2-5"])
def test_change_sets_equal_the_oracle(gp, opts):
    r = Rig(gp, seed=1, **opts)
    r.s.assign(False)
    m = r.commit_dry_then_real("first commit into an empty directory")
    n = r.s.size()
    assert len(m[0]) == n and (m[0] == np.arange(n)).all() and (m[2] == NONE).all()
    assert len(r.commit("nothing changed")[0]) == 0
    _history(r, r.commit_dry_then_real)


@pytest.mark.gpu
@pytest.mark.parametrize("opts", POLICIES[:2], ids=["hrw", "hrw2-12"])
def test_every_node_inactive_removes_every_key(gp, opts):
    r = Rig(gp, M=16, seed=2, **opts)
    r.s.assign(False)
    r.commit("first commit")
    r.s.rebalance_changes(*r.leave(range(16)))
    assert (r.s.read() == NONE).all()
    m = r.commit("every node inactive")
    assert len(m[0]) == r.s.size() and (m[3] == NONE).all()
    assert (r.p.lookup_many(r.s.read(want_keys=True)[0]) == NONE).all() and r.p.directory_len()[0] == 0


@pytest.mark.gpu
def test_bounded_rounds(gp):
    r = Rig(gp, seed=3)
    r.s.assign(False)
    r.commit("plain assignment")
    passes = r.s.assign_bounded(0, 101, 100, 8)
    assert passes > 1
    m = r.commit_dry_then_real("bounded at 101/100")
    assert len(m[0]) > 0


@pytest.mark.gpu
def test_bounded_affinity_change_set_on_the_cuda_cores(gp):
    r = Rig(gp, K=8, seed=4)
    r.s.assign_bounded_affinity(0, 5, 4, 8)
    r.commit("bounded affinity")
    r.s.rebalance_changes_bounded_affinity(*r.leave([2, 7]), 0, 5, 4, 8)
    m = r.commit_dry_then_real("bounded affinity change set")
    assert len(m[0]) > 0 and not np.isin(m[3], [2, 7]).any()


@pytest.mark.gpu
def test_weighted_bounded_with_hot_objects(gp):
    r = Rig(gp, seed=5)
    r.s.assign(False)
    r.commit("plain assignment")
    w = np.ones(r.s.size(), np.uint32)
    w[r.rng.choice(len(w), 40, replace=False)] = 200
    r.s.write_weights(w)
    r.s.assign_bounded_weighted(False, 0, 5, 4, 8)
    m = r.commit_dry_then_real("weighted bounded")
    assert len(m[0]) > 0


@pytest.mark.gpu
def test_ranked_set_commits_column_0(gp):
    r = Rig(gp, seed=6)
    r.s.assign_ranked(3)
    m = r.commit("ranked assignment")
    assert (m[3] == r.s.read_ranked()[:, 0]).all()
    r.s.rebalance_changes_ranked(*r.leave([5]))
    r.commit_dry_then_real("ranked change set")


@pytest.mark.gpu
def test_churn(gp):
    r = Rig(gp, seed=7)
    r.s.assign(False)
    r.commit("first commit")
    new = r.keys(77)
    r.s.insert(new)
    m = r.commit("inserted rows")
    assert (m[1] == new).all() and (m[2] == NONE).all()
    keys = r.s.read(want_keys=True)[0]
    gone = r.rng.choice(keys, 300, replace=False)
    before = r.p.lookup_many(gone)
    r.s.erase(gone)
    r.s.rebalance_changes(*r.leave([1]))
    r.commit_dry_then_real("erase, then a leave")
    assert (r.p.lookup_many(gone) == before).all()   # erased keys stay in the directory


@pytest.mark.gpu
def test_other_writers_between_commits(gp):
    r = Rig(gp, seed=8)
    r.s.assign(False)
    r.commit("first commit")
    keys = r.s.read(want_keys=True)[0]
    extra = r.keys(50)
    r.saw(extra)
    r.p.place_batch(np.concatenate([keys[:100], extra]), "hrw")
    r.p.update_many(keys[100:300], (np.arange(200) % r.M).astype(np.uint32))
    r.p.remove_many(keys[300:400])
    r.p.clean_node(11)
    m = r.commit_dry_then_real("after place_batch, update_many, remove_many and clean_node")
    assert len(m[0]) > 0 and (m[2] == NONE).sum() > 0 and (m[2] != NONE).sum() > 0


@pytest.mark.gpu
def test_duplicate_keys_and_the_reserved_key(gp):
    rng = np.random.default_rng(10)
    base = rng.integers(0, 2**62, 1500, dtype=np.uint64)
    keys = np.concatenate([base, base[:200], np.array([EMPTY, EMPTY - 1, 5, EMPTY], np.uint64), base[200:300]])
    keys = keys[rng.permutation(len(keys))]
    r = Rig(gp, seed=9, keys=keys)
    r.s.assign(False)   # duplicate rows share their key, so they share their node
    r.commit_dry_then_real("duplicates, first commit")
    # rows of one key on different nodes: every row is compared with the directory at the start, the last selected row wins
    k, idx = r.s.read(want_keys=True)
    dup = np.flatnonzero(np.isin(k, base[:200]) | (k == EMPTY) | (k == EMPTY - 1))
    r.p.update_many(k[dup], ((idx[dup].astype(np.int64) + 1 + np.arange(len(dup))) % r.M).astype(np.uint32))
    m = r.commit_dry_then_real("duplicates on other nodes in the directory")
    assert len(m[0]) >= len(dup) // 2
    r.s.rebalance_changes(*r.leave([0, 4]))
    r.commit_dry_then_real("duplicates after a change set")


@pytest.mark.gpu
def test_the_reserved_key_beside_its_neighbour_can_differ_from_set_commit(gp):
    """~0 - 1 in row 0 and ~0 in row 1 are two set keys placed apart, but one directory key.  The first commit writes both rows and row
    1 wins, as in set_commit.  A second call then selects row 0 only (row 1 matches the directory), so the directory flips to row 0's
    node, where set_commit keeps row 1's."""
    keys = np.array([EMPTY - 1, EMPTY, 17, 18], np.uint64)
    a, b = Rig(gp, seed=16, keys=keys), Rig(gp, seed=16, keys=keys)
    for r in (a, b):
        r.s.assign(False)
    idx = a.s.read()
    if idx[0] == idx[1]:
        pytest.skip("the seed placed ~0 - 1 and ~0 on one node")
    m = a.commit("first commit")
    assert list(m[0]) == [0, 1, 2, 3]
    b.s.commit()
    assert a.p.lookup_many([EMPTY])[0] == b.p.lookup_many([EMPTY])[0] == idx[1]
    m = a.commit("second commit")
    assert list(m[0]) == [0] and m[2][0] == idx[1] and m[3][0] == idx[0]
    b.s.commit()
    assert a.p.lookup_many([EMPTY - 1])[0] == idx[0] and b.p.lookup_many([EMPTY - 1])[0] == idx[1]


@pytest.mark.gpu
def test_directory_grows_during_the_call(gp):
    r = Rig(gp, seed=12, n=5000, cap=5000, dir_cap=1024)
    r.s.assign(False)
    slots = r.p.directory_len()[1]
    r.commit_dry_then_real("first commit into a small directory")
    assert r.p.directory_len()[1] > slots


@pytest.mark.gpu
@pytest.mark.parametrize("opts", POLICIES[:2], ids=["hrw", "hrw2-12"])
def test_equivalence_with_set_commit(gp, opts):
    a, b = Rig(gp, seed=13, **opts), Rig(gp, seed=13, **opts)
    a.s.assign(False)
    b.s.assign(False)
    _history(a, a.commit)
    _history(b, lambda tag: b.s.commit())
    for r in (a, b):
        r.s.insert(r.keys(30))
        r.s.rebalance_changes(*r.leave([30]))
    a.commit("after churn")
    b.s.commit()
    probe = np.concatenate([a.seen, a.s.read(want_keys=True)[0], a.foreign])
    assert a.p.lookup_many(probe).tobytes() == b.p.lookup_many(probe).tobytes()
    assert a.p.directory_len()[0] == b.p.directory_len()[0]


@pytest.mark.gpu
def test_refusals_change_nothing(gp):
    R = gp
    L = gp.GpuObjectPlacement().L
    n = C.c_uint64(7)
    assert L.rio_cuda_set_commit_changes(None, 0, 0, None, None, None, None, C.byref(n)) != 0 and n.value == 7
    r = Rig(gp, seed=14)

    def refused(call, tag):
        before = r.p.lookup_many(r.probe()), r.p.directory_len()
        with pytest.raises(R.Unknown):
            call()
        assert r.p.lookup_many(r.probe()).tobytes() == before[0].tobytes() and r.p.directory_len() == before[1], tag

    refused(lambda: r.s.commit_changes(), "a set with no assignment")
    r.s.assign(False)
    r.commit("first commit")
    r.s.rebalance_changes(*r.leave([6]))
    want = len(r.model().commit(*r.s.read(want_keys=True), dry_run=True)[0])
    assert want > 1
    for dry in (0, 1):
        bufs = [np.full(want, 0xAB, np.uint64), np.full(want, 0xAB, np.uint64), np.full(want, 0xAB, np.uint32), np.full(want, 0xAB, np.uint32)]
        ptrs = [b.ctypes.data_as(C.c_void_p) for b in bufs]
        for arg in range(4):
            got = C.c_uint64(0)
            only = [p if q == arg else None for q, p in enumerate(ptrs)]
            refused(lambda: r.s._ck(L.rio_cuda_set_commit_changes(r.s.s, dry, want - 1, *only, C.byref(got))), "cap one short")
            assert got.value == want
            assert all((b == 0xAB).all() for b in bufs), "an out array was written"
        # NULL arrays: the count, whatever cap says
        got = C.c_uint64(0)
        r.s._ck(L.rio_cuda_set_commit_changes(r.s.s, 1, 0, None, None, None, None, C.byref(got)))
        assert got.value == want
    r.s.assign_bounded_begin(0, 5, 4, 4)
    refused(lambda: r.s.commit_changes(), "a bounded call in flight")
    refused(lambda: r.s.commit_changes(dry_run=True), "a bounded call in flight, dry run")
    r.s.assign_bounded_end()
    r.commit_dry_then_real("after the bounded call ended")
    # an empty set: nothing to commit
    e = r.p.new_set(10)
    e.load_keys(np.zeros(0, np.uint64))
    e.assign(False)
    assert all(len(a) == 0 for a in e.commit_changes())


@pytest.mark.gpu
def test_a_leave_at_2m_objects_and_1024_nodes(gp):
    p = gp.GpuObjectPlacement()
    if host_sim(p):
        pytest.skip("2 M objects x 1024 nodes is a GPU-sized case")
    M, n = 1024, 2_000_000
    rng = np.random.default_rng(15)
    w = rng.integers(1, 17, M).astype(np.uint32)
    p.set_nodes(addresses(M), w)
    s = p.new_set(n)
    s.synth_keys(0, n, 77)
    s.assign(False)
    s.commit()
    keys, before = s.read(want_keys=True)
    dir_before = p.lookup_many(keys)
    assert (dir_before == before).all()
    j = int(np.argmax(np.bincount(before, minlength=M)))
    p.node_set_active(j, False)
    s.rebalance_changes([j], [int(w[j])])
    after = s.read()
    rows = np.flatnonzero(after != before)
    dry = s.commit_changes(dry_run=True)
    got = s.commit_changes()
    for m in (dry, got):
        assert m[0].tobytes() == rows.astype(np.uint64).tobytes()
        assert m[1].tobytes() == keys[rows].tobytes()
        assert m[2].tobytes() == dir_before[rows].tobytes() and (m[2] == j).all()
        assert m[3].tobytes() == after[rows].tobytes()
    assert (p.lookup_many(keys) == after).all()
    assert len(s.commit_changes()[0]) == 0


# ---- host-sim --------------------------------------------------------------------------------------------------------------------
DOUBLES = os.path.join(ROOT, "tests", "cpp", "hostsim", "set_commit_launchers.cpp")
OTHER_DOUBLES = [os.path.join(ROOT, "tests", "cpp", "hostsim", f) for f in ("ranked_launchers.cpp", "change_launchers.cpp", "ranked_change_launchers.cpp",
                                                                              "spread_launchers.cpp", "spread_change_launchers.cpp",
                                                                              "affinity_ranked_launchers.cpp", "affinity_spread_launchers.cpp",
                                                                              "affinity_set_launchers.cpp", "affinity_bounded_launchers.cpp",
                                                                              "set_bounded_affinity_launchers.cpp", "set_churn_launchers.cpp",
                                                                              "bounded_weighted_launchers.cpp")]


def test_the_doubles_cover_the_new_launchers():
    decl = set(re.findall(r"\b(launch_[a-z0-9_]+)\s*\(", open(os.path.join(ROOT, "rio_rs_b200", "csrc", "k_set_commit.cuh")).read()))
    have = set(re.findall(r"^void\s+([a-z0-9_]+)\s*\(", open(DOUBLES).read(), flags=re.M))
    assert len(decl) == 2 and decl <= have, decl - have


def _hostsim_library(HS, name, doubles):
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, name)
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + doubles + ["-o", so, "-ldl", "-lpthread"])
    return so


def test_set_commit_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + every double, the new one
    included)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_set_commit.so", OTHER_DOUBLES + [DOUBLES])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=3000, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 16 and "failed" not in r.stdout, tail


def test_the_new_call_reports_an_error_where_its_kernels_are_not_linked():
    """The engine's host code built WITHOUT the new launchers loads, refuses the call with RIO_ERR_UPSTREAM and a message, and still
    commits the set with set_commit."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_no_set_commit.so", OTHER_DOUBLES)
    code = (
        "import sys, numpy as np\n"
        "from rio_rs_b200 import _native as N\n"
        "N.library_path = lambda: sys.argv[1]\n"
        "import rio_rs_b200 as R\n"
        "p = R.GpuObjectPlacement()\n"
        "p.set_nodes(['10.0.0.%d:5000' % j for j in range(8)])\n"
        "keys = np.arange(100, dtype=np.uint64)\n"
        "s = p.new_set(200); s.load_keys(keys); s.assign()\n"
        "for dry in (False, True):\n"
        "    try:\n"
        "        s.commit_changes(dry_run=dry)\n"
        "        raise SystemExit('ran without kernels')\n"
        "    except R.Upstream as e:\n"
        "        assert 'set commit kernels' in str(e), e\n"
        "assert p.directory_len()[0] == 0\n"
        "s.commit()\n"
        "assert (p.lookup_many(keys) == s.read()).all()\n"
        "print('refused ok')\n"
    )
    r = subprocess.run([sys.executable, "-c", code, so], capture_output=True, text=True, timeout=300, cwd=HS.ROOT)
    assert r.returncode == 0 and "refused ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

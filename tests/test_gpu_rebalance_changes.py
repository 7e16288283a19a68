"""Change-set rebalance (DESIGN.md 3.10): one call takes a set of node changes -- joins, leaves, weight increases and decreases --
and leaves the directory and a resident set equal to the fresh assignment over the final live set.  Every state is compared with
the CPU oracle (oracle.assign_hrw / assign_hrw2 over the final live weights) under both policies, the directory (after
set.commit()) and the set side by side: placements, the number moved, and the set's counters.

The CPU tests at the end run this module's GPU bodies, unchanged, against the engine's host logic compiled with g++ (the host-sim
library of tests/test_engine_host_sim.py) with plain restatements of the change-set launchers, and check that a build without those
launchers refuses the flat path and still serves HRW2."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

NONE = 0xFFFFFFFF
POLICIES = ["hrw", "hrw2"]
THREADS = os.cpu_count() or 8


@pytest.fixture(scope="module")
def gp():
    from rio_rs_b200 import build

    build.build()
    import rio_rs_b200 as R

    return R


class Cluster:
    """A provider, its node table mirrored as live weights (0 = not live), a resident set and the directory committed from it."""

    def __init__(self, gp, oracle, policy, M, n, live_frac=0.9, key_seed=3, weight_seed=7):
        self.oracle, self.policy = oracle, policy
        self.p = gp.GpuObjectPlacement()
        self.p.set_solver(policy, 0)
        self.addrs, self.seeds, self.w = oracle.synth_nodes(M, weight_seed=weight_seed)
        rng = np.random.default_rng(M + n)
        self.live = self.w.copy()
        self.live[rng.random(M) > live_frac] = 0
        self.p.set_nodes(self.addrs, self.live)
        self.keys = oracle.synth_keys(n, key_seed)
        self.s = self.p.new_set(n)
        self.s.load_keys(self.keys)
        self.s.assign()
        self.s.commit()
        self.cur = self.fresh()
        assert (self.s.read() == self.cur).all()

    def fresh(self, w=None):
        w = self.live if w is None else w
        if self.policy == "hrw2":
            return self.oracle.assign_hrw2(self.keys, self.seeds, w, threads=THREADS)
        return self.oracle.assign_hrw(self.keys, self.seeds, w, threads=THREADS)

    def apply(self, changes):
        """changes: {node: new live weight, 0 = leave}.  Returns (idx, prev_weight) read from the engine before the changes."""
        idx = np.array(sorted(changes), dtype=np.uint32)
        prev = np.empty(len(idx), dtype=np.uint32)
        for q, j in enumerate(idx):
            active, weight, _ = self.p.node_state(int(j))
            prev[q] = weight if active and weight else 0
            assert prev[q] == self.live[j]
        for j, nw in changes.items():
            if nw:
                assert self.p.node_upsert(self.addrs[j], int(nw)) == j
            else:
                self.p.node_set_active(int(j), False)
            self.live[j] = nw
        return idx, prev

    def rebalance_and_check(self, idx, prev, tag=""):
        ms = self.s.rebalance_changes(idx, prev)
        md = self.p.rebalance_changes(idx, prev)
        want = self.fresh()
        got = self.s.read()
        assert (got == want).all(), tag
        assert (self.p.lookup_many(self.keys) == want).all(), tag
        moved = int((self.cur != want).sum())
        assert ms == moved == md, (tag, ms, md, moved)
        cnt = self.s.counters()
        assert (cnt == self.oracle.counts(want, len(self.w))[: len(cnt)]).all(), tag
        old, self.cur = self.cur, want
        return old, want


def random_changes(rng, live, w, k):
    """k distinct nodes, each drawn as a join, leave, weight increase, weight decrease or an unchanged weight."""
    M = len(live)
    out = {}
    for j in rng.choice(M, size=min(k, M), replace=False):
        j = int(j)
        if not live[j]:
            out[j] = int(rng.integers(1, 17)) if rng.random() < 0.8 else 0   # join, or a listed node that stays out
            continue
        kind = rng.integers(0, 4)
        if kind == 0:
            out[j] = 0                                                       # leave
        elif kind == 1:
            out[j] = int(live[j]) + int(rng.integers(1, 9))                  # gains weight
        elif kind == 2:
            out[j] = max(1, int(live[j]) // 2) if live[j] > 1 else int(live[j])   # loses weight (weight 1 stays)
        else:
            out[j] = int(live[j])                                            # r unchanged
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("M", [128, 1024])
@pytest.mark.parametrize("k", [1, 4, 32, "all"])
def test_random_change_sets_equal_a_fresh_assignment(gp, oracle, policy, M, k):
    c = Cluster(gp, oracle, policy, M, 300_000)
    rng = np.random.default_rng(1000 * M + (0 if k == "all" else k))
    for rnd in range(3):
        idx, prev = c.apply(random_changes(rng, c.live, c.w, M if k == "all" else k))
        c.rebalance_and_check(idx, prev, (rnd, len(idx)))
    assert (c.live > 0).sum() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_node_table_larger_than_shared_memory(gp, oracle, policy):
    """7000 interned nodes: the by-index records, the candidates and the flag table are read from global memory."""
    c = Cluster(gp, oracle, policy, 7000, 60_000)
    rng = np.random.default_rng(5)
    for rnd in range(2):
        idx, prev = c.apply(random_changes(rng, c.live, c.w, 48))
        c.rebalance_and_check(idx, prev, rnd)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_c5_events_as_one_change_set(gp, oracle, policy):
    """C5's eight join/leave events: eight single-event calls on one set, one change set on another set and on the directory."""
    M0 = 128
    c = Cluster(gp, oracle, policy, M0 + 4, 300_000, live_frac=2.0)
    for j in range(M0, M0 + 4):                    # the four joiners start outside the cluster
        c.p.node_set_active(j, False)
        c.live[j] = 0
    single = c.p.new_set(len(c.keys))
    single.load_keys(c.keys)
    for s in (single, c.s):
        s.assign()
    c.s.commit()
    c.cur = c.fresh()
    events = [("leave", 17), ("join", M0), ("leave", 3), ("join", M0 + 1), ("leave", 100), ("join", M0 + 2), ("leave", 64), ("join", M0 + 3)]
    idx = np.array([j for _, j in events], dtype=np.uint32)
    prev = np.array([c.live[j] for j in idx], dtype=np.uint32)
    moved_single = 0
    for ev, j in events:
        c.apply({j: 0 if ev == "leave" else int(c.w[j])})
        moved_single += single.rebalance(ev, j)
    c.rebalance_and_check(idx, prev)
    assert (single.read() == c.s.read()).all() and (single.counters() == c.s.counters()).all()
    assert moved_single > 0


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_weight_ramp_of_one_node(gp, oracle, policy):
    """One node goes 16 -> 8 -> 1 -> 0 -> 4 -> 16.  Under the flat policy the movement is minimal: on a decrease every mover was on
    the node, on an increase every mover lands on it."""
    c = Cluster(gp, oracle, policy, 256, 300_000, live_frac=2.0)
    x = 37
    c.apply({x: 16})
    c.s.assign()
    c.s.commit()
    c.cur = c.fresh()
    for nw in (8, 1, 0, 4, 16):
        up = nw > c.live[x]
        idx, prev = c.apply({x: nw})
        old, want = c.rebalance_and_check(idx, prev, nw)
        ch = old != want
        assert ch.sum() > 0, nw
        if policy == "hrw":
            assert (want[ch] == x).all() if up else (old[ch] == x).all(), nw


@pytest.mark.gpu
def test_entries_not_placed_by_the_hash_follow_r1_and_r2(gp, oracle):
    """Directory entries recorded on arbitrary nodes (live, inactive, never live) under the flat policy: an entry on a REPLACE node
    gets the flat placement over the live set, any other one the best node of {its node} u CANDIDATES."""
    M, n = 300, 200_000
    p = gp.GpuObjectPlacement()
    addrs, seeds, w = oracle.synth_nodes(M)
    live = w.copy()
    live[250:] = 0                                              # 250..299: interned, never live
    p.set_nodes(addrs[:250], w[:250])
    for j in range(250, M):
        assert p.node_intern(addrs[j]) == j
    for j in (10, 11):                                          # inactive from the start
        p.node_set_active(j, False)
        live[j] = 0
    keys = oracle.synth_keys(n, 9)
    rng = np.random.default_rng(4)
    y = rng.integers(0, M, size=n).astype(np.uint32)
    p.update_many(keys, y)
    dec = next(j for j in range(21, 40) if w[j] > 1 and j != 30)
    changes = {3: 0, 20: int(w[20]) + 5, dec: int(w[dec]) // 2, 10: 6, 260: 9, 30: int(w[30])}
    idx = np.array(sorted(changes), dtype=np.uint32)
    prev = np.array([live[j] for j in idx], dtype=np.uint32)
    for j, nw in changes.items():
        if nw:
            assert p.node_upsert(addrs[j], nw) == j
        else:
            p.node_set_active(j, False)
        live[j] = nw
    r_prev = {int(j): (0xFFFFFFFF // int(pw) if pw else 0) for j, pw in zip(idx, prev)}
    r_now = lambda j: 0xFFFFFFFF // int(live[j]) if live[j] else 0
    replace = np.array([live[j] == 0 or bool(j in r_prev and r_prev[j] and r_now(j) > r_prev[j]) for j in range(M)], dtype=bool)
    cand = [j for j in r_prev if live[j] and (not r_prev[j] or r_now(j) < r_prev[j])]
    assert sorted(cand) == [10, 20, 260] and replace[[3, 11, dec, 299]].all() and not replace[30]
    want = np.empty(n, dtype=np.uint32)
    r1 = replace[y]
    want[r1] = oracle.assign_hrw(keys[r1], seeds, live, threads=THREADS)
    for node in np.unique(y[~r1]):
        sel = (y == node) & ~r1
        wr = np.zeros(M, dtype=np.uint32)
        wr[cand] = live[cand]
        wr[node] = live[node]
        want[sel] = oracle.assign_hrw(keys[sel], seeds, wr, threads=THREADS)
    moved = p.rebalance_changes(idx, prev)
    got = p.lookup_many(keys)
    assert (got == want).all()
    assert moved == int((y != want).sum())


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_every_node_leaves_then_k_zero(gp, oracle, policy):
    c = Cluster(gp, oracle, policy, 64, 50_000)
    live_nodes = [int(j) for j in np.nonzero(c.live)[0]]
    idx, prev = c.apply({j: 0 for j in live_nodes})
    c.rebalance_and_check(idx, prev)
    assert (c.s.read() == NONE).all() and (c.p.lookup_many(c.keys) == NONE).all() and (c.s.counters() == 0).all()
    # a node comes back: the set re-places its unplaced objects; the directory's unplaced entries stay unplaced (as after a JOIN)
    idx, prev = c.apply({live_nodes[0]: 5})
    assert c.s.rebalance_changes(idx, prev) == len(c.keys) and (c.s.read() == live_nodes[0]).all()
    assert c.p.rebalance_changes(idx, prev) == 0
    before = c.s.read().copy()
    empty = np.empty(0, np.uint32)
    assert c.s.rebalance_changes(empty, empty) == 0 and c.p.rebalance_changes(empty, empty) == 0
    assert (c.s.read() == before).all()


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_bad_arguments(gp, oracle, policy):
    c = Cluster(gp, oracle, policy, 32, 1000)
    L, h, s = c.p.L, c.p.h, c.s.s
    two, prev = np.array([3, 3], np.uint32), np.array([1, 1], np.uint32)
    for call, obj in ((L.rio_cuda_rebalance_changes, h), (L.rio_cuda_set_rebalance_changes, s)):
        assert call(obj, two.ctypes.data_as(C.c_void_p), prev.ctypes.data_as(C.c_void_p), 2, None) == -2
        assert b"duplicate" in L.rio_cuda_last_error(h)
        far = np.array([32], np.uint32)
        assert call(obj, far.ctypes.data_as(C.c_void_p), prev.ctypes.data_as(C.c_void_p), 1, None) == -2
        assert b"range" in L.rio_cuda_last_error(h)
        assert call(obj, None, None, 1, None) == -2 and b"null" in L.rio_cuda_last_error(h)
        assert call(obj, None, None, 0, None) == 0
    with pytest.raises(gp.Unknown):
        c.p.rebalance_changes([1, 2], [1])
    fresh = c.p.new_set(10)
    fresh.load_keys(c.keys[:10])
    with pytest.raises(gp.Unknown, match="no assignment"):
        fresh.rebalance_changes([1], [0])
    assert (c.s.read() == c.cur).all()


CHANGE_DOUBLES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "hostsim", "change_launchers.cpp")


def test_the_change_doubles_cover_every_change_launcher():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    decl = set(re.findall(r"\b(launch_[a-z0-9_]+)\s*\(", open(os.path.join(root, "rio_rs_b200", "csrc", "k_changes.cuh")).read()))
    have = set(re.findall(r"^void\s+([a-z0-9_]+)\s*\(", open(CHANGE_DOUBLES).read(), flags=re.M))
    assert len(decl) == 4 and decl <= have, decl - have


def test_change_set_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + the change-set doubles)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, "librio_cuda_hostsim_changes.so")
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + [CHANGE_DOUBLES, "-o", so, "-ldl", "-lpthread"])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=1800, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 27 and "failed" not in r.stdout, tail


def test_flat_change_sets_report_an_error_where_the_kernels_are_not_linked():
    """The engine's host code built WITHOUT the change-set launchers (the host-sim library of tests/test_engine_host_sim.py) loads,
    refuses the flat path with RIO_ERR_UPSTREAM and a message, and still serves change sets under HRW2 (existing launchers only)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, "librio_cuda_hostsim_nochanges.so")
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + ["-o", so, "-ldl", "-lpthread"])
    code = (
        "import sys, numpy as np\n"
        "from rio_rs_b200 import _native as N\n"
        "N.library_path = lambda: sys.argv[1]\n"
        "import rio_rs_b200 as R\n"
        "from oracle import pyoracle as O\n"
        "O.build()\n"
        "addrs, seeds, w = O.synth_nodes(16)\n"
        "keys = O.synth_keys(5000, 1)\n"
        "for policy in ('hrw', 'hrw2'):\n"
        "    p = R.GpuObjectPlacement()\n"
        "    p.set_solver(policy, 0)\n"
        "    p.set_nodes(addrs, w)\n"
        "    s = p.new_set(len(keys)); s.load_keys(keys); s.assign(); s.commit()\n"
        "    prev = int(w[5])\n"
        "    p.node_set_active(5, False)\n"
        "    w2 = w.copy(); w2[5] = 0\n"
        "    for call in (s.rebalance_changes, p.rebalance_changes):\n"
        "        try:\n"
        "            call([5], [prev])\n"
        "        except R.Upstream as e:\n"
        "            assert policy == 'hrw' and 'change-set kernels' in str(e), e\n"
        "            continue\n"
        "        assert policy == 'hrw2'\n"
        "    if policy == 'hrw2':\n"
        "        want = O.assign_hrw2(keys, seeds, w2)\n"
        "        assert (s.read() == want).all() and (p.lookup_many(keys) == want).all()\n"
        "print('refused ok')\n"
    )
    r = subprocess.run([sys.executable, "-c", code, so], capture_output=True, text=True, timeout=300, cwd=HS.ROOT)
    assert r.returncode == 0 and "refused ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

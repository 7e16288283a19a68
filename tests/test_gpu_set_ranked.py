"""Ranked resident sets (DESIGN.md 3.11): a set keeps each object's first R nodes, and one change-set call brings every list up to
date.  Every state is compared with the ranked CPU oracle (tests/ranked_oracle.c) over the final live weights under both policies:
the lists, the set's primary index (column 0), its counters, out_moved (rows whose rank 1 changed) and out_changed (rows that
changed at any rank).

The CPU tests at the end run this module's GPU bodies, unchanged, against the engine's host logic compiled with g++ (the host-sim
library of tests/test_engine_host_sim.py) with plain restatements of the ranked and ranked-set launchers, and check that a build
without the ranked-set launchers refuses the ranked calls while the unranked change set keeps working."""
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
THREADS = os.cpu_count() or 8


@pytest.fixture(scope="module")
def gp():
    from rio_rs_b200 import build

    build.build()
    import rio_rs_b200 as R

    return R


class RankedCluster:
    """A provider, its node table mirrored as live weights (0 = not live) and seeds, and a resident set holding R-lists."""

    def __init__(self, gp, oracle, policy, M, n, R, live_frac=0.9, key_seed=3, weight_seed=7, twins=()):
        self.oracle, self.policy, self.R = oracle, policy, R
        self.p = gp.GpuObjectPlacement()
        self.p.set_solver(policy, 0)
        self.addrs, self.seeds, self.w = oracle.synth_nodes(M, weight_seed=weight_seed)
        rng = np.random.default_rng(M + n + R)
        self.live = self.w.copy()
        self.live[rng.random(M) > live_frac] = 0
        self.p.set_nodes(self.addrs, self.live)
        for a, b in twins:                       # b gets a's seed: equal pair hashes, ties inside the lists
            self.seeds[b] = self.seeds[a]
            self.p.dev_set_node_seed(b, int(self.seeds[a]))
        self.keys = oracle.synth_keys(n, key_seed)
        self.s = self.p.new_set(n)
        self.s.load_keys(self.keys)
        self.s.assign_ranked(R)
        self.cur = self.fresh()
        self.check_state(self.cur)

    def fresh(self):
        return RO.assign_ranked(self.policy, self.keys, self.seeds, self.live, self.R, threads=THREADS)

    def check_state(self, want, tag=""):
        got = self.s.read_ranked()
        assert got.shape == want.shape and (got == want).all(), (tag, int((got != want).any(axis=1).sum()))
        assert (self.s.read() == want[:, 0]).all(), tag
        cnt = self.s.counters()
        assert (cnt == self.oracle.counts(want[:, 0], len(self.w))[: len(cnt)]).all(), tag

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
        moved, changed = self.s.rebalance_changes_ranked(idx, prev)
        want = self.fresh()
        self.check_state(want, tag)
        want_moved = int((self.cur[:, 0] != want[:, 0]).sum())
        want_changed = int((self.cur != want).any(axis=1).sum())
        assert (moved, changed) == (want_moved, want_changed), (tag, moved, changed, want_moved, want_changed)
        old, self.cur = self.cur, want
        return old, want


def random_changes(rng, live, k):
    """k distinct nodes, each drawn as a join, leave, weight increase, weight decrease or an unchanged weight."""
    M = len(live)
    out = {}
    for j in rng.choice(M, size=min(k, M), replace=False):
        j = int(j)
        if not live[j]:
            out[j] = int(rng.integers(1, 17)) if rng.random() < 0.8 else 0
            continue
        kind = rng.integers(0, 4)
        if kind == 0:
            out[j] = 0
        elif kind == 1:
            out[j] = int(live[j]) + int(rng.integers(1, 9))
        elif kind == 2:
            out[j] = max(1, int(live[j]) // 2) if live[j] > 1 else int(live[j])
        else:
            out[j] = int(live[j])
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("R", [1, 2, 3, 8])
def test_assign_ranked_equals_the_oracle(gp, oracle, policy, R):
    c = RankedCluster(gp, oracle, policy, 300, 20_001, R)
    assert (c.s.read_ranked() == c.p.assign_ranked(c.keys, R)).all()
    assert (c.s.read_ranked(1000, 77) == c.cur[1000:1077]).all()
    assert c.s.read_ranked(5, 0).shape == (0, R)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("M", [128, 1024])
@pytest.mark.parametrize("k", [1, 4, 32, "all"])
@pytest.mark.parametrize("R", [1, 2, 3, 8])
def test_random_change_sets_equal_fresh_lists(gp, oracle, policy, M, k, R):
    c = RankedCluster(gp, oracle, policy, M, 20_000 if M == 128 else 8_000, R)
    rng = np.random.default_rng(1000 * M + 10 * R + (0 if k == "all" else k))
    for rnd in range(3):
        idx, prev = c.apply(random_changes(rng, c.live, M if k == "all" else k))
        c.rebalance_and_check(idx, prev, (rnd, len(idx)))
    assert (c.live > 0).sum() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("M", [6144, 6145])
def test_both_sides_of_the_staging_threshold(gp, oracle, policy, M):
    """Up to 6144 interned nodes the by-index records, candidates and flags are staged in shared memory, above that read from global
    memory."""
    c = RankedCluster(gp, oracle, policy, M, 4_000, 3)
    rng = np.random.default_rng(M)
    for rnd in range(2):
        idx, prev = c.apply(random_changes(rng, c.live, 48))
        c.rebalance_and_check(idx, prev, rnd)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_rank_one_is_the_unranked_change_set(gp, oracle, policy):
    c = RankedCluster(gp, oracle, policy, 256, 50_000, 1)
    twin = c.p.new_set(len(c.keys))
    twin.load_keys(c.keys)
    twin.assign()
    rng = np.random.default_rng(11)
    for k in (1, 8, 64):
        idx, prev = c.apply(random_changes(rng, c.live, k))
        moved_twin = twin.rebalance_changes(idx, prev)
        moved, changed = c.s.rebalance_changes_ranked(idx, prev)
        assert moved == changed == moved_twin
        assert (c.s.read() == twin.read()).all() and (c.s.read_ranked()[:, 0] == twin.read()).all()
        assert (c.s.counters() == twin.counters()).all()


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_list_member_gains_then_loses_weight(gp, oracle, policy):
    """A node that sits at rank > 1 in many lists gains weight (a candidate already in L: counted once), then loses it (S1)."""
    c = RankedCluster(gp, oracle, policy, 64, 30_000, 4, live_frac=2.0)
    x = int(np.bincount(c.cur[:, 2].astype(np.int64), minlength=64).argmax())
    assert (c.cur[:, 1:] == x).sum() > 1000
    for nw in (int(c.live[x]) + 20, max(1, int(c.live[x]) // 4)):
        idx, prev = c.apply({x: nw})
        _, changed = c.s.rebalance_changes_ranked(idx, prev)
        want = c.fresh()
        c.check_state(want, nw)
        assert changed == int((c.cur != want).any(axis=1).sum()) > 0
        c.cur = want


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_weight_ramp_of_one_node(gp, oracle, policy):
    c = RankedCluster(gp, oracle, policy, 256, 40_000, 3, live_frac=2.0)
    x = 37
    for nw in (16, 8, 1, 0, 4, 16):
        if nw == c.live[x]:
            continue
        idx, prev = c.apply({x: nw})
        old, want = c.rebalance_and_check(idx, prev, nw)
        assert (old != want).any(), nw


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_ties_between_twin_seeds_cross_a_change_set(gp, oracle, policy):
    """Nodes with equal seeds and weights tie on the score and the pair hash: the node index decides, in the kernel as in the oracle."""
    M = 200
    twins = [(3, 44), (10, 11), (100, 149), (5, 6), (7, 6)]
    c = RankedCluster(gp, oracle, policy, M, 40_000, 4, live_frac=2.0, weight_seed=1, twins=twins)
    for j in (3, 44, 10, 11, 5, 6, 7, 100, 149):
        c.apply({j: 9})
    c.s.assign_ranked(4)
    c.cur = c.fresh()
    c.check_state(c.cur)
    for changes in ({6: 0, 50: 0}, {6: 9, 11: 0}, {11: 9, 44: 12, 3: 12}, {5: 9, 7: 0, 149: 0, 60: 30}):
        idx, prev = c.apply(changes)
        c.rebalance_and_check(idx, prev, changes)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("R", [3, 8])
def test_padding_fills_and_empties(gp, oracle, policy, R):
    """Two live nodes and R > 2: NONE pads every list; joins fill them; every node leaving leaves only NONE; nodes come back."""
    c = RankedCluster(gp, oracle, policy, 16, 10_000, R, live_frac=2.0)
    idx, prev = c.apply({j: 0 for j in range(2, 16)})
    c.rebalance_and_check(idx, prev, "shrink")
    assert (c.cur[:, 2:] == NONE).all()
    for joins in ({4: 3, 9: 7}, {j: 5 for j in range(10, 16)}):
        idx, prev = c.apply(joins)
        c.rebalance_and_check(idx, prev, joins)
    idx, prev = c.apply({j: 0 for j in np.nonzero(c.live)[0]})
    moved, changed = c.s.rebalance_changes_ranked(idx, prev)
    assert (c.s.read_ranked() == NONE).all() and (c.s.read() == NONE).all() and (c.s.counters() == 0).all()
    assert moved == changed == len(c.keys)
    c.cur = c.fresh()
    for back in ({3: 4}, {1: 2, 12: 16}):
        idx, prev = c.apply(back)
        c.rebalance_and_check(idx, prev, back)
    empty = np.empty(0, np.uint32)
    assert c.s.rebalance_changes_ranked(empty, empty) == (0, 0)
    c.check_state(c.cur)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_calls_that_assign_the_set_drop_the_lists(gp, oracle, policy):
    c = RankedCluster(gp, oracle, policy, 40, 2_000, 2, live_frac=2.0)
    j = 5

    def leave_and_rejoin(s):
        """a real change set on the set: node j leaves, so both the unranked and the ranked call have work to do"""
        idx, prev = c.apply({j: 0})
        s.rebalance_changes(idx, prev)
        c.apply({j: int(c.w[j])})

    def single_event(s):
        c.apply({j: 0})
        s.rebalance("leave", j)
        c.apply({j: int(c.w[j])})
        s.rebalance("join", j)

    drops = [
        ("load_keys", lambda s: s.load_keys(c.keys)),
        ("synth_keys", lambda s: s.synth_keys(0, len(c.keys), 5)),
        ("assign", lambda s: s.assign()),
        ("assign_bounded", lambda s: s.assign_bounded()),
        ("assign_bounded_begin", lambda s: (s.assign_bounded_begin(), s.assign_bounded_end())),
        ("rebalance", single_event),
        ("rebalance_changes", leave_and_rejoin),
    ]
    for name, call in drops:
        c.s.load_keys(c.keys)
        c.s.assign_ranked(2)
        assert c.s.read_ranked().shape == (len(c.keys), 2)
        call(c.s)
        with pytest.raises(gp.Unknown, match="no ranked lists"):
            c.s.read_ranked()
        idx, prev = c.apply({j: 0})
        with pytest.raises(gp.Unknown, match="no ranked lists"):
            c.s.rebalance_changes_ranked(idx, prev)
        c.apply({j: int(c.w[j])})
        assert c.s.read().shape == (len(c.keys),), name   # the set itself still works
    # the lists record their policy: another solver, or another trie depth, is refused and leaves them as they were
    c.s.load_keys(c.keys)
    c.s.assign_ranked(2)
    c.cur = c.fresh()
    other = "hrw2" if policy == "hrw" else "hrw"
    for solver, bits in ((other, 0), (policy, 7)):
        c.p.set_solver(solver, bits)
        idx, prev = c.apply({j: 0})
        with pytest.raises(gp.Unknown, match="another solver"):
            c.s.rebalance_changes_ranked(idx, prev)
        c.apply({j: int(c.w[j])})
        c.p.set_solver(policy, 12)
        c.check_state(c.cur, solver)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_bad_arguments(gp, oracle, policy):
    c = RankedCluster(gp, oracle, policy, 32, 1000, 3)
    L, h, s = c.p.L, c.p.h, c.s.s
    for r in (0, 9):
        assert L.rio_cuda_set_assign_ranked(s, r) == -2 and b"ranks" in L.rio_cuda_last_error(h)
    out = np.empty((1000, 3), np.uint32)
    p = out.ctypes.data_as(C.c_void_p)
    assert L.rio_cuda_set_read_ranked(s, 0, 1001, p) == -2 and b"range" in L.rio_cuda_last_error(h)
    assert L.rio_cuda_set_read_ranked(s, 1001, 0, p) == -2
    assert L.rio_cuda_set_read_ranked(s, 1, 2 ** 64 - 1, p) == -2
    assert L.rio_cuda_set_read_ranked(s, 0, 10, None) == -2 and b"null" in L.rio_cuda_last_error(h)
    assert L.rio_cuda_set_read_ranked(s, 0, 1000, p) == 0 and (out == c.cur).all()
    two, prev = np.array([3, 3], np.uint32), np.array([1, 1], np.uint32)
    call = L.rio_cuda_set_rebalance_changes_ranked
    assert call(s, two.ctypes.data_as(C.c_void_p), prev.ctypes.data_as(C.c_void_p), 2, None, None) == -2
    assert b"duplicate" in L.rio_cuda_last_error(h)
    far = np.array([32], np.uint32)
    assert call(s, far.ctypes.data_as(C.c_void_p), prev.ctypes.data_as(C.c_void_p), 1, None, None) == -2
    assert b"range" in L.rio_cuda_last_error(h)
    assert call(s, None, None, 1, None, None) == -2 and b"null" in L.rio_cuda_last_error(h)
    assert call(s, None, None, 0, None, None) == 0
    with pytest.raises(gp.Unknown):
        c.s.rebalance_changes_ranked([1, 2], [1])
    fresh = c.p.new_set(10)
    fresh.load_keys(c.keys[:10])
    with pytest.raises(gp.Unknown, match="no ranked lists"):
        fresh.read_ranked()
    with pytest.raises(gp.Unknown, match="no ranked lists"):
        fresh.rebalance_changes_ranked([1], [0])
    c.check_state(c.cur)


RANKED_DOUBLES = [os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "hostsim", f)
                  for f in ("ranked_launchers.cpp", "change_launchers.cpp")]
SET_DOUBLES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp", "hostsim", "ranked_change_launchers.cpp")


def test_the_ranked_set_doubles_cover_every_ranked_set_launcher():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    decl = set(re.findall(r"\b(launch_[a-z0-9_]+)\s*\(", open(os.path.join(root, "rio_rs_b200", "csrc", "k_ranked_changes.cuh")).read()))
    have = set(re.findall(r"^void\s+([a-z0-9_]+)\s*\(", open(SET_DOUBLES).read(), flags=re.M))
    assert len(decl) == 4 and decl <= have, decl - have


def _hostsim_library(HS, name, doubles):
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, name)
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + doubles + ["-o", so, "-ldl", "-lpthread"])
    return so


def test_ranked_set_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + the ranked, change-set and
    ranked-set doubles)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_set_ranked.so", RANKED_DOUBLES + [SET_DOUBLES])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=3000, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 92 and "failed" not in r.stdout, tail


def test_ranked_sets_report_an_error_where_the_kernels_are_not_linked():
    """The engine's host code built with the ranked and change-set launchers but WITHOUT the ranked-set ones loads, refuses
    set_assign_ranked and the ranked change set with RIO_ERR_UPSTREAM and a message, and still serves the unranked change set."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_noranked_sets.so", RANKED_DOUBLES)
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
        "    s = p.new_set(len(keys)); s.load_keys(keys)\n"
        "    for call in (lambda: s.assign_ranked(2), lambda: s.rebalance_changes_ranked([5], [int(w[5])])):\n"
        "        try:\n"
        "            call()\n"
        "        except R.Upstream as e:\n"
        "            assert 'ranked-set kernels' in str(e), e\n"
        "            continue\n"
        "        raise AssertionError('not refused')\n"
        "    s.assign()\n"
        "    p.node_set_active(5, False)\n"
        "    w2 = w.copy(); w2[5] = 0\n"
        "    s.rebalance_changes([5], [int(w[5])])\n"
        "    want = O.assign_hrw2(keys, seeds, w2) if policy == 'hrw2' else O.assign_hrw(keys, seeds, w2)\n"
        "    assert (s.read() == want).all()\n"
        "print('refused ok')\n"
    )
    r = subprocess.run([sys.executable, "-c", code, so], capture_output=True, text=True, timeout=300, cwd=HS.ROOT)
    assert r.returncode == 0 and "refused ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

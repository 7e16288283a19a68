"""Failure-domain resident sets (DESIGN.md 3.13): a set keeps each object's first R nodes in R distinct domains, and one change-set call
brings every list up to date over the current live set and the CURRENT labels, relabels since the last call included.  Every state is
compared with the spread CPU oracle (tests/spread_oracle.c) over the final live weights and labels under both policies: the lists, the
set's primary index (column 0), its counters, out_moved (rows whose rank 1 changed) and out_changed (rows that changed at any rank).

The CPU tests at the end run this module's GPU bodies, unchanged, against the engine's host logic compiled with g++ (the host-sim
library of tests/test_engine_host_sim.py) with plain restatements of the spread-set launchers, and check that a build without the
spread-set launchers refuses the spread-set calls while plain ranked sets keep working."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import ranked_oracle as RO
import spread_oracle as SO

NONE = 0xFFFFFFFF
POLICIES = ["hrw", "hrw2"]
THREADS = os.cpu_count() or 8
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rio_rs_b200", "csrc")
HOSTSIM = bool(os.environ.get("RIO_HOSTSIM_LIBRARY"))

# the staging thresholds the spread-set launchers branch on: (source file, the text that defines it, its value); a CPU test checks
# the text is there.  The flat change-set pass stages up to 6144 interned nodes; its S1 rows are recomputed by the flat spread kernel,
# staged while the records and domain ids fit 96 KB; the HRW2 compare mode is k_assign_trie_spread with its 200 KB staging budget.
CHANGES_STAGED = ("k_directory.cu", "return tab.n_total <= 6144 ? (size_t)tab.n_total * 17 + (size_t)cs.n_cand * 4 : 0;", 6144)
FLAT_STAGED = ("k_spread.cu", "const size_t smem = (size_t)tab.n_live * 16 + ((size_t)tab.n_live * 4 + 15) / 16 * 16;\n    if (smem <= 96u * 1024u) {",
               96 * 1024)
TRIE_STAGED = ("k_spread.cu", "const size_t smem = (size_t)t.blob_bytes + sp.o_ndom;\n    if (smem <= kSpreadSmemBudget) {", 200 * 1024)
FLAT_MAX_STAGED = max(m for m in range(FLAT_STAGED[2] // 16 + 1) if m * 16 + (m * 4 + 15) // 16 * 16 <= FLAT_STAGED[2])


@pytest.fixture(scope="module")
def gp():
    from rio_rs_b200 import build

    build.build()
    import rio_rs_b200 as R

    return R


def labels(name, M, rng):
    """The label layouts: equal racks, uneven racks, no labels, one single domain, and three domains (fewer than most R here)."""
    j = np.arange(M, dtype=np.uint32)
    if name == "racks":
        return j // 16
    if name == "uneven":
        return np.sort(rng.integers(0, max(2, M // 12), size=M)).astype(np.uint32) * 3 + 5
    if name == "none":
        return np.full(M, NONE, dtype=np.uint32)
    if name == "single":
        return np.full(M, 77, dtype=np.uint32)
    if name == "few":
        return (j * 7) % 3
    raise AssertionError(name)


class SpreadCluster:
    """A provider, its node table mirrored as live weights (0 = not live), seeds and labels, and a resident set holding spread lists."""

    def __init__(self, gp, oracle, policy, M, n, R, dom, live_frac=0.9, key_seed=3, weight_seed=7, twins=(), weights=None):
        self.gp, self.oracle, self.policy, self.R = gp, oracle, policy, R
        self.p = gp.GpuObjectPlacement()
        self.p.set_solver(policy, 0)
        self.addrs, self.seeds, self.w = oracle.synth_nodes(M, weight_seed=weight_seed)
        if weights is not None:
            self.w = np.asarray(weights, dtype=np.uint32)
        rng = np.random.default_rng(M + n + R)
        self.live = self.w.copy()
        self.live[rng.random(M) > live_frac] = 0
        self.p.set_nodes(self.addrs, self.live)
        for a, b in twins:                       # b gets a's seed: equal pair hashes, ties inside the lists
            self.seeds[b] = self.seeds[a]
            self.p.dev_set_node_seed(b, int(self.seeds[a]))
        self.dom = np.asarray(dom, dtype=np.uint32).copy()
        self.p.set_node_domains(np.arange(M, dtype=np.uint32), self.dom)
        self.keys = oracle.synth_keys(n, key_seed)
        self.s = self.p.new_set(n)
        self.s.load_keys(self.keys)
        self.s.assign_ranked_spread(R)
        self.cur = self.fresh()
        self.check_state(self.cur)

    def fresh(self):
        return SO.assign_spread(self.policy, self.keys, self.seeds, self.live, self.dom, self.R, threads=THREADS)

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

    def relabel(self, relabels):
        """relabels: {node: new label}"""
        idx = np.array(sorted(relabels), dtype=np.uint32)
        self.dom[idx] = [relabels[int(j)] for j in idx]
        self.p.set_node_domains(idx, self.dom[idx])

    def rebalance_and_check(self, idx, prev, tag=""):
        moved, changed = self.s.rebalance_changes_ranked(idx, prev)
        want = self.fresh()
        self.check_state(want, tag)
        want_moved = int((self.cur[:, 0] != want[:, 0]).sum())
        want_changed = int((self.cur != want).any(axis=1).sum())
        assert (moved, changed) == (want_moved, want_changed), (tag, moved, changed, want_moved, want_changed)
        old, self.cur = self.cur, want
        return old, want


EMPTY = (np.empty(0, np.uint32), np.empty(0, np.uint32))


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
def test_assign_equals_the_batch_call_and_the_oracle(gp, oracle, policy, R):
    M = 300
    c = SpreadCluster(gp, oracle, policy, M, 20_001, R, labels("racks", M, None))
    assert (c.s.read_ranked() == c.p.assign_ranked_spread(c.keys, R)).all()
    assert (c.s.read() == c.p.assign_batch(c.keys)).all()
    assert (c.s.read_ranked(1000, 77) == c.cur[1000:1077]).all()
    assert c.s.read_ranked(5, 0).shape == (0, R)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
@pytest.mark.parametrize("M", [128, 1024])
@pytest.mark.parametrize("k", [1, 4, 32, "all"])
@pytest.mark.parametrize("layout", ["racks", "uneven", "none", "single", "few"])
def test_random_change_sets_equal_fresh_lists(gp, oracle, policy, M, k, layout):
    rng = np.random.default_rng(1000 * M + (0 if k == "all" else k) + len(layout))
    R = 4 if layout != "racks" else (2 if M == 128 else 8)
    c = SpreadCluster(gp, oracle, policy, M, 8_000 if M == 128 else 4_000, R, labels(layout, M, rng))
    for rnd in range(3):
        idx, prev = c.apply(random_changes(rng, c.live, M if k == "all" else k))
        c.rebalance_and_check(idx, prev, (rnd, len(idx)))
    if layout == "single":
        assert (c.cur[:, 1:] == NONE).all()
    if layout == "few":
        assert (c.cur[:, 3:] == NONE).all()


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_no_labels_is_a_plain_ranked_set(gp, oracle, policy):
    """Without labels a spread set and a plain ranked set driven by the same change sets hold the same lists, assignment, counters and
    counts at every step."""
    M, R = 256, 3
    c = SpreadCluster(gp, oracle, policy, M, 20_000, R, np.full(M, NONE, np.uint32))
    plain = c.p.new_set(len(c.keys))
    plain.load_keys(c.keys)
    plain.assign_ranked(R)
    rng = np.random.default_rng(5)
    for k in (1, 8, 64, 0):
        idx, prev = c.apply(random_changes(rng, c.live, k)) if k else EMPTY
        got = c.s.rebalance_changes_ranked(idx, prev)
        assert got == plain.rebalance_changes_ranked(idx, prev), k
        assert (c.s.read_ranked() == plain.read_ranked()).all() and (c.s.read() == plain.read()).all()
        assert (c.s.counters() == plain.counters()).all()
    c.check_state(c.fresh())


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_rank_one_is_the_unranked_change_set(gp, oracle, policy):
    M = 256
    c = SpreadCluster(gp, oracle, policy, M, 50_000, 1, labels("racks", M, None))
    twin = c.p.new_set(len(c.keys))
    twin.load_keys(c.keys)
    twin.assign()
    rng = np.random.default_rng(11)
    for k in (1, 8, 64):
        idx, prev = c.apply(random_changes(rng, c.live, k))
        moved_twin = twin.rebalance_changes(idx, prev)
        moved, changed = c.s.rebalance_changes_ranked(idx, prev)
        assert moved == changed == moved_twin
        assert (c.s.read() == twin.read()).all() and (c.s.counters() == twin.counters()).all()


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_a_whole_rack_leaving_promotes_rank_two(gp, oracle, policy):
    """A rack of 32 leaves as one change set: every object whose rank 1 was in it has its old rank 2 as rank 1."""
    M, R = 1024, 4
    c = SpreadCluster(gp, oracle, policy, M, 40_000, R, np.arange(M, dtype=np.uint32) // 32, live_frac=2.0)
    for d in (3, 20):
        rack = np.flatnonzero(c.dom == d)
        hit = np.isin(c.cur[:, 0], rack)
        assert hit.sum() > 0
        idx, prev = c.apply({int(j): 0 for j in rack})
        old, new = c.rebalance_and_check(idx, prev, d)
        assert (new[hit, 0] == old[hit, 1]).all() and (new[hit, : R - 1] == old[hit, 1:]).all(), d
        assert not np.isin(new, rack).any()


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_a_node_displaces_the_listed_member_of_its_own_domain(gp, oracle, policy):
    """A node joins, and another gains weight, inside racks already listed.  Under the flat policy, where it now beats its rack's listed
    member it takes that member's place, the other ranks unchanged (the replace-in-place path of the domain-aware insert)."""
    M, R = 256, 4
    c = SpreadCluster(gp, oracle, policy, M, 40_000, R, np.arange(M, dtype=np.uint32) // 8, live_frac=2.0)
    z = 42
    idx, prev = c.apply({z: 0})
    c.rebalance_and_check(idx, prev, "leave")
    for changes in ({z: 60}, {z + 1: int(c.live[z + 1]) * 8}):
        y = next(iter(changes))
        idx, prev = c.apply(changes)
        old, new = c.rebalance_and_check(idx, prev, changes)
        if policy == "hrw2":   # the exclusion-adjusted walk has no fixed order to replace in: the oracle check above is the test
            continue
        rack = np.flatnonzero(c.dom == c.dom[y])
        # rows where y entered: the rack's member it replaced sat at the same rank, every other rank is as it was
        rows, cols = np.nonzero(new == y)
        same_rack = np.isin(old[rows, cols], rack) & (old[rows, cols] != y)
        assert same_rack.sum() > 100, changes
        r2, c2 = rows[same_rack], cols[same_rack]
        keep = np.ones((len(r2), R), dtype=bool)
        keep[np.arange(len(r2)), c2] = False
        assert (old[r2][keep] == new[r2][keep]).all(), changes


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_relabels(gp, oracle, policy):
    """Relabels with k = 0 and inside change sets: a listed node moved to another rack, an unlisted node moved into a domain of its
    own, a node that is not live relabelled (no effect), and a new node labelled before it joins."""
    M, R = 200, 3
    c = SpreadCluster(gp, oracle, policy, M, 30_000, R, np.arange(M, dtype=np.uint32) // 10, live_frac=2.0)
    x = int(np.bincount(c.cur[:, 1].astype(np.int64), minlength=M).argmax())
    assert (c.cur[:, 1:] == x).sum() > 100
    c.relabel({x: int(c.dom[(x + 50) % M])})                       # a listed node moves to another rack
    c.rebalance_and_check(*EMPTY, "listed")
    counts = np.bincount(c.cur.ravel().astype(np.int64), minlength=M)
    u = int(np.argmin(np.where(c.live > 0, counts, 1 << 30)))       # the live node listed least
    c.relabel({u: 5000})                                            # ... moves into a domain of its own
    c.rebalance_and_check(*EMPTY, "unlisted")
    assert c.s.rebalance_changes_ranked(*EMPTY) == (0, 0)           # nothing changed since: a no-op
    idx, prev = c.apply({7: 0})
    c.relabel({7: 4000})                                            # relabelled while not live: no effect on the lists
    assert c.s.rebalance_changes_ranked(idx, prev)[1] > 0
    c.cur = c.fresh()
    c.check_state(c.cur)
    assert c.s.rebalance_changes_ranked(*EMPTY) == (0, 0)
    c.check_state(c.cur)
    idx, prev = c.apply({7: int(c.w[7])})                           # ... and rejoins under its new label
    c.rebalance_and_check(idx, prev, "rejoin")
    # a relabel and a weight change in one change set
    c.relabel({11: 4000, 12: NONE})
    idx, prev = c.apply({13: 0, 60: int(c.live[60]) + 9})
    c.rebalance_and_check(idx, prev, "mixed")
    # a node interned after the labels were recorded, labelled before it joins
    a_new = "10.99.0.1:7000"
    j = c.p.node_intern(a_new)
    assert j == M
    c.p.set_node_domains(np.array([j], np.uint32), np.array([3], np.uint32))
    assert c.s.rebalance_changes_ranked(*EMPTY) == (0, 0)           # interned and labelled, not live: no effect
    assert c.p.node_upsert(a_new, 40) == j
    c.addrs = list(c.addrs) + [a_new]
    c.seeds = np.append(c.seeds, np.uint64(oracle.node_seed(a_new)))
    c.w = np.append(c.w, np.uint32(40))
    c.live = np.append(c.live, np.uint32(40))
    c.dom = np.append(c.dom, np.uint32(3))
    c.rebalance_and_check(np.array([j], np.uint32), np.array([0], np.uint32), "new node")
    assert (c.cur == j).sum() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_relabels_leave_a_plain_ranked_set_alone(gp, oracle, policy):
    """A plain ranked set ignores labels: relabels between its change sets change nothing in what it computes."""
    M, R = 128, 3
    c = SpreadCluster(gp, oracle, policy, M, 20_000, R, np.arange(M, dtype=np.uint32) // 8, live_frac=2.0)
    c.s.assign_ranked(R)
    want = RO.assign_ranked(policy, c.keys, c.seeds, c.live, R, threads=THREADS)
    rng = np.random.default_rng(3)
    for rnd in range(3):
        c.relabel({int(j): int(rng.integers(0, 4)) for j in rng.choice(M, 20, replace=False)})
        assert c.s.rebalance_changes_ranked(*EMPTY) == (0, 0)
        idx, prev = c.apply(random_changes(rng, c.live, 6))
        moved, changed = c.s.rebalance_changes_ranked(idx, prev)
        now = RO.assign_ranked(policy, c.keys, c.seeds, c.live, R, threads=THREADS)
        assert (c.s.read_ranked() == now).all() and (moved, changed) == (int((now[:, 0] != want[:, 0]).sum()), int((now != want).any(axis=1).sum()))
        want = now


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_ties_between_twin_seeds(gp, oracle, policy):
    """Nodes with equal seeds and weights tie on the score and the pair hash: the node index decides, in the kernels as in the oracle,
    whether the twins share a rack or not."""
    M = 200
    twins = [(3, 44), (10, 11), (100, 149), (5, 6), (7, 6)]
    c = SpreadCluster(gp, oracle, policy, M, 40_000, 4, np.arange(M, dtype=np.uint32) // 5, live_frac=2.0, weight_seed=1, twins=twins)
    for j in (3, 44, 10, 11, 5, 6, 7, 100, 149):
        c.apply({j: 9})
    c.s.assign_ranked_spread(4)
    c.cur = c.fresh()
    c.check_state(c.cur)
    for changes in ({6: 0, 50: 0}, {6: 9, 11: 0}, {11: 9, 44: 12, 3: 12}, {5: 9, 7: 0, 149: 0, 60: 30}):
        idx, prev = c.apply(changes)
        c.rebalance_and_check(idx, prev, changes)
    c.relabel({44: 0, 149: 20})
    c.rebalance_and_check(*EMPTY, "relabel twins")


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_extreme_weights(gp, oracle, policy):
    """Weights near 2^32 - 1 in one rack, weight 1 beside them, and change sets moving weight between them."""
    M = 96
    w = oracle.synth_nodes(M)[2].astype(np.uint32)
    w[:12] = 0xFFFFFFFF - np.arange(12, dtype=np.uint32)
    w[40:44] = 0xFFFFFFF0
    w[60:64] = 1
    dom = np.where(np.arange(M) < 12, 0, 1 + np.arange(M) // 8).astype(np.uint32)
    c = SpreadCluster(gp, oracle, policy, M, 20_000, 3, dom, live_frac=2.0, weights=w)
    for changes in ({0: 0, 1: 1}, {60: 0xFFFFFFFE, 41: 2}, {0: 0xFFFFFFFF, 1: 0xFFFFFFFF, 61: 0}):
        idx, prev = c.apply(changes)
        c.rebalance_and_check(idx, prev, changes)
    c.relabel({40: 0, 2: 50})
    c.rebalance_and_check(*EMPTY, "relabel heavy")


@pytest.mark.gpu
@pytest.mark.parametrize("policy,which", [("hrw", "changes"), ("hrw", "flat"), ("hrw2", "trie")])
@pytest.mark.parametrize("side", [0, 1])
def test_both_sides_of_the_staging_thresholds(gp, oracle, policy, which, side):
    """changes: the flat change-set pass at 6144 / 6145 interned nodes.  flat: the S1 rows recomputed by the flat spread kernel, on the
    last staged live count or one past it (relabels and weight gains keep the live count).  trie: the HRW2 compare mode on the
    largest staged node set or one past it (relabels keep the table)."""
    import test_gpu_boundaries as TB

    if which == "changes":
        M = CHANGES_STAGED[2] + side
    elif which == "flat":
        M = FLAT_MAX_STAGED + side
    else:
        M = TB.largest_staged_ranked_trie(oracle, 12, 8000) + side
    c = SpreadCluster(gp, oracle, policy, M, 3_000, 3, np.arange(M, dtype=np.uint32) // 32, live_frac=0.95 if which == "changes" else 2.0)
    rng = np.random.default_rng(M)
    for rnd in range(2):
        c.relabel({int(j): int(rng.integers(0, M // 32)) for j in rng.choice(M, 24, replace=False)})
        if which == "changes":
            idx, prev = c.apply(random_changes(rng, c.live, 48))
        elif which == "flat":
            idx, prev = c.apply({int(j): int(c.live[j]) + 5 for j in rng.choice(M, 8, replace=False)})
        else:
            idx, prev = EMPTY
        c.rebalance_and_check(idx, prev, rnd)
    if which != "changes":
        assert int((c.live > 0).sum()) == M


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_kind_switches_drops_and_policy(gp, oracle, policy):
    M, R = 40, 2
    c = SpreadCluster(gp, oracle, policy, M, 2_000, R, np.arange(M, dtype=np.uint32) // 4, live_frac=2.0)
    j = 5
    # spread -> plain: the lists are the ranked ones and labels stop counting; plain -> spread: the labels count again
    c.s.assign_ranked(R)
    assert (c.s.read_ranked() == RO.assign_ranked(policy, c.keys, c.seeds, c.live, R, threads=THREADS)).all()
    c.relabel({1: 9})
    assert c.s.rebalance_changes_ranked(*EMPTY) == (0, 0)
    c.s.assign_ranked_spread(R)
    c.cur = c.fresh()
    c.check_state(c.cur)
    c.relabel({c.cur[0, 0]: 99})
    c.rebalance_and_check(*EMPTY, "after the switch back")

    def leave_and_rejoin(s):
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
        c.s.assign_ranked_spread(R)
        call(c.s)
        with pytest.raises(gp.Unknown, match="no ranked lists"):
            c.s.read_ranked()
        with pytest.raises(gp.Unknown, match="no ranked lists"):
            c.s.rebalance_changes_ranked(*EMPTY)
        assert c.s.read().shape == (len(c.keys),), name
    # the lists record their policy: another solver, or another trie depth, is refused and leaves them (and the snapshot) as they were
    c.s.load_keys(c.keys)
    c.s.assign_ranked_spread(R)
    c.cur = c.fresh()
    other = "hrw2" if policy == "hrw" else "hrw"
    for solver, bits in ((other, 0), (policy, 7)):
        c.p.set_solver(solver, bits)
        c.relabel({3: 123})
        with pytest.raises(gp.Unknown, match="another solver"):
            c.s.rebalance_changes_ranked(*EMPTY)
        c.p.set_solver(policy, 12)
        c.check_state(c.cur, solver)
    c.rebalance_and_check(*EMPTY, "relabels kept for the next call")


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_bad_arguments(gp, oracle, policy):
    M = 32
    c = SpreadCluster(gp, oracle, policy, M, 1000, 3, np.arange(M, dtype=np.uint32) // 4)
    L, h, s = c.p.L, c.p.h, c.s.s
    for r in (0, 9):
        assert L.rio_cuda_set_assign_ranked_spread(s, r) == -2 and b"ranks" in L.rio_cuda_last_error(h)
    assert L.rio_cuda_set_assign_ranked_spread(None, 2) == -2
    two, prev = np.array([3, 3], np.uint32), np.array([1, 1], np.uint32)
    call = L.rio_cuda_set_rebalance_changes_ranked
    assert call(s, two.ctypes.data_as(C.c_void_p), prev.ctypes.data_as(C.c_void_p), 2, None, None) == -2
    assert b"duplicate" in L.rio_cuda_last_error(h)
    far = np.array([M], np.uint32)
    assert call(s, far.ctypes.data_as(C.c_void_p), prev.ctypes.data_as(C.c_void_p), 1, None, None) == -2
    assert call(s, None, None, 1, None, None) == -2 and b"null" in L.rio_cuda_last_error(h)
    c.relabel({0: 1})
    assert call(s, None, None, 0, None, None) == 0                  # k = 0 with a relabel: applied, NULL outputs allowed
    c.cur = c.fresh()
    c.check_state(c.cur)
    c.check_state(c.cur)


@pytest.mark.gpu
@pytest.mark.parametrize("policy", POLICIES)
def test_one_million_objects_in_racks(gp, oracle, policy):
    """1 M objects x 1024 nodes in 32 racks of 32 at R = 4: a rack leaving, a join, a relabel, each against the oracle."""
    if HOSTSIM:
        pytest.skip("sized for the GPU: the host restatements take minutes at this size")
    M = 1024
    c = SpreadCluster(gp, oracle, policy, M, 1_000_000, 4, np.arange(M, dtype=np.uint32) // 32)
    idx, prev = c.apply({int(j): 0 for j in range(64, 96)})
    c.rebalance_and_check(idx, prev, "rack")
    c.relabel({100: 7, 101: 900})
    idx, prev = c.apply({int(j): 12 for j in np.flatnonzero(c.live == 0)[:5]})
    c.rebalance_and_check(idx, prev, "join + relabel")


# ---- CPU ---------------------------------------------------------------------------------------------------------------------------
SET_DOUBLES = os.path.join(ROOT, "tests", "cpp", "hostsim", "spread_change_launchers.cpp")
OTHER_DOUBLES = [os.path.join(ROOT, "tests", "cpp", "hostsim", f) for f in ("ranked_launchers.cpp", "change_launchers.cpp",
                                                                              "ranked_change_launchers.cpp", "spread_launchers.cpp")]


def test_staging_thresholds_are_where_the_launchers_define_them():
    for f, text, _ in (CHANGES_STAGED, FLAT_STAGED, TRIE_STAGED):
        assert text in open(os.path.join(CSRC, f)).read(), f
    assert FLAT_MAX_STAGED == 4915


def test_the_spread_set_doubles_cover_every_spread_set_launcher():
    decl = set(re.findall(r"\b(launch_[a-z0-9_]+)\s*\(", open(os.path.join(CSRC, "k_spread_changes.cuh")).read()))
    have = set(re.findall(r"^void\s+([a-z0-9_]+)\s*\(", open(SET_DOUBLES).read(), flags=re.M))
    assert len(decl) == 2 and decl <= have, decl - have


def _hostsim_library(HS, name, doubles):
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, name)
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + doubles + ["-o", so, "-ldl", "-lpthread"])
    return so


def test_spread_set_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + the ranked, change-set,
    ranked-set, spread and spread-set doubles)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_set_spread.so", OTHER_DOUBLES + [SET_DOUBLES])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=3000, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 100 and "failed" not in r.stdout, tail


def test_spread_sets_report_an_error_where_the_kernels_are_not_linked():
    """The engine's host code built with the ranked, ranked-set and spread launchers but WITHOUT the spread-set ones loads, refuses
    set_assign_ranked_spread with RIO_ERR_UPSTREAM and a message, and still serves plain ranked sets and the unranked change set."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_nospread_sets.so", OTHER_DOUBLES)
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
        "    p.set_node_domains(np.arange(16), np.arange(16) // 4)\n"
        "    s = p.new_set(len(keys)); s.load_keys(keys)\n"
        "    try:\n"
        "        s.assign_ranked_spread(2)\n"
        "        raise AssertionError('not refused')\n"
        "    except R.Upstream as e:\n"
        "        assert 'spread-set kernels' in str(e), e\n"
        "    s.assign_ranked(2)\n"
        "    p.node_set_active(5, False)\n"
        "    w2 = w.copy(); w2[5] = 0\n"
        "    s.rebalance_changes_ranked([5], [int(w[5])])\n"
        "    assert (s.read_ranked() == p.assign_ranked(keys, 2)).all()\n"
        "    s.assign()\n"
        "    p.node_set_active(6, False)\n"
        "    w2[6] = 0\n"
        "    s.rebalance_changes([6], [int(w[6])])\n"
        "    want = O.assign_hrw2(keys, seeds, w2) if policy == 'hrw2' else O.assign_hrw(keys, seeds, w2)\n"
        "    assert (s.read() == want).all()\n"
        "print('refused ok')\n"
    )
    r = subprocess.run([sys.executable, "-c", code, so], capture_output=True, text=True, timeout=300, cwd=HS.ROOT)
    assert r.returncode == 0 and "refused ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

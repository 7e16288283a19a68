"""Weighted bounded sets kept within load capacity (DESIGN.md 3.21): ObjectSet.rebalance_changes_bounded_weighted and
ObjectSet.write_weights_by_key against tests/set_bounded_weighted_changes_oracle.py.

* Event sequences, bit for bit after every call (idx, counters, loads, moved, passes): a single leave, a rack leaving and rejoining, a
  join of a new node, weight halving and increase, an active node set to weight 0, everyone leaving and rejoining, weight drift written
  by key with k = 0 and churn between calls; flat HRW, HRW2 at 12 and 5 bits, affinity on the CUDA cores (K = 8, 24, and 16 with
  ffma) and on the tensor cores (integer features against c32, U(-1, 1) features against a twin handle); uniform, lognormal, 1 % hot
  and partly zero weights; caps 5/4, 101/100, 1/1 and max_rounds 1..16; live counts either side of 64, 256 and 2304.  After every call
  set_commit_changes' manifest equals the diff of the set against what was committed before, and the movement contract holds.
* The identity anchors, the record's lifetime, every refusal, the by-key writes, and two ranks against one.

The CPU tests at the end run this module's GPU bodies, unchanged, against the engine's host logic (the host-sim library of
tests/test_engine_host_sim.py) with a plain restatement of the new launchers, run the host-sim multirank script, and check that a
build without the new launchers refuses both calls while every other call keeps working.  There the tensor path is never taken."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import bounded_weighted_oracle as BW
import set_bounded_weighted_changes_oracle as W
import spec_py as S
from test_gpu_set_bounded_weighted import addresses, host_sim, int_feats, variant, weight_mix

NONE = 0xFFFFFFFF
U32 = 0xFFFFFFFF
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MIXES = ["uniform", "lognormal", "hot", "zeros"]
SCHEDULE = [((5, 4), 4), ((101, 100), 16), ((1, 1), 2), ((5, 4), 1), ((1, 1), 16), ((5, 4), 8)]


@pytest.fixture(scope="module")
def gp():
    from rio_rs_b200 import build

    build.build()
    import rio_rs_b200 as R

    return R


class Sim:
    """A handle with M nodes and a weighted set assigned by assign_bounded_weighted, mirrored here (node weights, liveness, features,
    keys, object features and weights, the committed directory) for the oracle.  policy: 'hrw', 'hrw2' or 'affinity'."""

    def __init__(self, gp, policy, M, n, K=0, seed=0, bits=12, mix="uniform", var="ffma", fo=None, fn=None, engine=False, dead=(),
                 zero_weight=(), cap=(5, 4), rounds=8):
        rng = np.random.default_rng(4000 + seed)
        self.gp, self.policy, self.bits, self.var, self.engine, self.rng = gp, policy, bits, var, engine, rng
        self.aff = policy == "affinity"
        self.K = K
        self.w = rng.integers(1, 17, M).astype(np.uint32)
        self.w[list(zero_weight)] = 0
        self.active = np.ones(M, bool)
        self.active[list(dead)] = False
        self.fn = (rng.uniform(-1, 1, (M, K)).astype(np.float32) if fn is None else np.asarray(fn, np.float32)) if K else None
        self.fo = (rng.uniform(-1, 1, (n, K)).astype(np.float32) if fo is None else np.asarray(fo, np.float32)) if K else None
        self.keys = rng.integers(0, 2**63, n, dtype=np.uint64)
        self.ow = weight_mix(mix, n, rng)
        self.p = self.handle(self.active)
        self.s = self.p.new_set(2 * n + 256)
        self.s.load_keys(self.keys)
        if K:
            self.s.load_feats(self.fo)
        self.s.write_weights(self.ow)
        with variant(var):
            self.s.assign_bounded_weighted(self.aff, 0, cap[0], cap[1], rounds)
        self.dir = {}
        self.refeatured = []
        self.commit()

    @property
    def M(self):
        return len(self.w)

    @property
    def live(self):
        return self.active & (self.w > 0)

    def seeds(self):
        return [S.node_seed(a) for a in addresses(self.M)]

    def handle(self, mask):
        p = self.gp.GpuObjectPlacement()
        p.set_solver("hrw2" if self.policy == "hrw2" else "hrw", self.bits)
        p.set_nodes(addresses(self.M), self.w, self.fn)
        for j in np.flatnonzero(~np.asarray(mask, bool)):
            p.node_set_active(int(j), False)
        return p

    def argmin(self):
        if not self.aff:
            return BW.hash_argmin(self.keys, self.seeds(), self.w, self.policy, self.bits)
        if self.engine:
            fo = self.fo
            return lambda rows, mask: self.handle(mask).assign_batch(obj_feats=fo[rows])
        return BW.c32_argmin(self.fo, self.fn)

    # ---- node events: each returns the change set (idx, prev_weight) --------------------------------------------------------
    def _changes(self, js, before_live, before_w):
        js = sorted(set(int(j) for j in js))
        return js, [int(before_w[j]) if j < len(before_live) and before_live[j] else 0 for j in js]

    def set_active(self, js, on):
        bl, bw = self.live.copy(), self.w.copy()
        for j in js:
            self.p.node_set_active(int(j), on)
            self.active[j] = on
        return self._changes(js, bl, bw)

    def set_weight(self, js, ws):
        bl, bw = self.live.copy(), self.w.copy()
        for j, nw in zip(js, ws):
            self.p.node_upsert(addresses(self.M)[j], int(nw))
            self.w[j] = nw
        return self._changes(js, bl, bw)

    def join_new(self, wt):
        bl, bw = self.live.copy(), self.w.copy()
        j = self.M
        f = self.rng.uniform(-1, 1, self.K).astype(np.float32) if self.K else None
        if self.K and self.fo is not None and self.fo.dtype == np.float32 and np.all(self.fo == np.round(self.fo)):
            f = np.round(f * 4)
        assert self.p.node_upsert(addresses(j + 1)[j], int(wt), f) == j
        self.w = np.append(self.w, np.uint32(wt))
        self.active = np.append(self.active, True)
        if self.K:
            self.fn = np.vstack([self.fn, f[None, :]])
        return self._changes([j], bl, bw)

    def refeature(self, j):
        """node j keeps its weight and gets new features: no change-set entry, the set's feature snapshot finds it"""
        f = self.rng.uniform(-1, 1, self.K).astype(np.float32)
        if np.all(self.fn == np.round(self.fn)):
            f = np.round(f * 4)
        self.p.node_upsert(addresses(self.M)[j], int(self.w[j]), f)
        self.fn = self.fn.copy()
        self.fn[j] = f
        self.refeatured.append(int(j))
        return [], []

    # ---- object events ---------------------------------------------------------------------------------------------------------
    def drift(self, frac=0.02):
        rows = self.rng.choice(len(self.keys), max(int(len(self.keys) * frac), 1), replace=False)
        nw = weight_mix("uniform", len(rows), self.rng)
        assert self.s.write_weights_by_key(self.keys[rows], nw) == len(rows)
        self.ow[rows] = nw
        return [], []

    def churn(self, m=40):
        new = self.rng.integers(0, 2**63, m, dtype=np.uint64)
        nf = None
        if self.K:
            nf = self.rng.uniform(-1, 1, (m, self.K)).astype(np.float32)
            if np.all(self.fo == np.round(self.fo)):
                nf = np.round(nf * 4)
        first = self.s.insert(new, nf)
        with variant(self.var):
            want = self.p.assign_batch(obj_feats=nf) if self.aff else self.p.assign_batch(new)
        assert self.s.read(first).tobytes() == want.tobytes()
        self.keys = np.concatenate([self.keys, new])
        if self.K:
            self.fo = np.vstack([self.fo, nf])
        nw = weight_mix("uniform", m, self.rng)
        assert self.s.write_weights_by_key(new, nw) == m
        self.ow = np.concatenate([self.ow, nw])
        gone = self.keys[self.rng.choice(len(self.keys), m // 2, replace=False)]
        rows = BW.erase_pairing(self.keys, gone)
        assert self.s.erase(gone) == m // 2
        self.keys, self.ow = self.keys[rows], self.ow[rows]
        if self.K:
            self.fo = self.fo[rows]
        assert self.s.read(want_keys=True)[0].tobytes() == self.keys.tobytes()
        assert self.s.read_weights().tobytes() == self.ow.tobytes()
        return [], []

    # ---- the call ---------------------------------------------------------------------------------------------------------------
    def call(self, changes, cap=(5, 4), rounds=8, load_total=0, tag=""):
        idx, prev = changes
        before = self.s.read()
        want = W.rebalance(self.policy, self.keys, before, self.ow, self.w, self.live, self.active, idx, prev, self.argmin(), load_total, cap[0], cap[1],
                           rounds, self.seeds(), self.bits, self.fo, self.fn, self.refeatured)
        self.refeatured = []
        with variant(self.var):
            moved, passes = self.s.rebalance_changes_bounded_weighted(idx, prev, load_total, cap[0], cap[1], rounds)
        got, cnt, ld = self.s.read(), self.s.counters(), self.s.loads()
        assert got.tobytes() == want["idx"].tobytes(), (tag, int((got != want["idx"]).sum()))
        assert (cnt == want["counters"]).all() and (ld == want["loads"]).all(), tag
        assert moved == want["moved"] and passes == want["passes"], (tag, moved, want["moved"], passes, want["passes"])
        # the movement contract: S1, taken by a candidate in pass 0, or spilled (weight > 0) from a node over its load capacity
        mv = got != before
        p0 = want["pass0"]
        spilled = (got != p0) & (p0 != NONE) & (self.ow > 0)
        spilled[spilled] = want["closed"][p0[spilled]]
        assert (want["s1"] | want["beaten"] | spilled)[mv].all(), tag
        self.commit(tag)
        return want

    def commit(self, tag=""):
        """set_commit_changes' manifest is the diff of the set against the last commit: {row, key, from = committed, to = idx}."""
        keys, idx = self.s.read(want_keys=True)
        frm = np.array([self.dir.get(int(k), NONE) for k in keys], np.uint32)
        rows = np.flatnonzero(frm != idx)
        r, k, f, t = self.s.commit_changes()
        assert r.tolist() == rows.tolist() and k.tobytes() == keys[rows].tobytes(), tag
        assert f.tobytes() == frm[rows].tobytes() and t.tobytes() == idx[rows].tobytes(), tag
        for kk, ii in zip(keys.tolist(), idx.tolist()):
            self.dir[kk] = ii


def events(sim, rng):
    """The event sequence of 3.21's tests, as (name, thunk returning a change set)."""
    live = lambda: [int(j) for j in np.flatnonzero(sim.live)]   # noqa: E731
    one = int(rng.choice(live()))
    rack = [int(j) for j in rng.choice([j for j in live() if j != one], 4, replace=False)]
    heavy = [int(j) for j in rng.choice(live(), 3, replace=False)]
    zero = int(rng.choice([j for j in live() if j not in rack and j != one]))
    refeat = [("refeature", lambda: sim.refeature(heavy[2]))] if sim.aff else []
    return [
        ("leave", lambda: sim.set_active([one], False)),
        ("drift", lambda: sim.drift()),
        ("rack leaves", lambda: sim.set_active(rack, False)),
        ("churn", lambda: sim.churn()),
        ("rack rejoins", lambda: sim.set_active(rack + [one], True)),
        ("join", lambda: sim.join_new(9)),
        ("halve", lambda: sim.set_weight(heavy, [max(int(sim.w[j]) // 2, 1) for j in heavy])),
        ("increase", lambda: sim.set_weight(heavy[:2], [int(sim.w[j]) * 3 for j in heavy[:2]])),
    ] + refeat + [
        ("weight 0", lambda: sim.set_weight([zero], [0])),
        ("all leave", lambda: sim.set_active(range(sim.M), False)),
        ("k = 0 with no live node", lambda: ([], [])),
        ("all rejoin", lambda: sim.set_active(range(sim.M), True)),
        ("drift again", lambda: sim.drift(0.05)),
    ]


def run_sequence(sim, rng, skip=()):
    fired = 0
    for t, (name, ev) in enumerate(events(sim, rng)):
        if name in skip:
            continue
        cap, rounds = SCHEDULE[t % len(SCHEDULE)]
        want = sim.call(ev(), cap, rounds, tag=name)
        fired += want["passes"] > 1
    return fired


# ---- against the oracle ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("policy,bits", [("hrw", 12), ("hrw2", 12), ("hrw2", 5)])
@pytest.mark.parametrize("mix", MIXES)
def test_hash_event_sequence_equals_the_oracle(gp, policy, bits, mix):
    sim = Sim(gp, policy, 40, 1500, seed=bits + MIXES.index(mix), bits=bits, mix=mix, dead=(2,), zero_weight=(9,), cap=(1, 1), rounds=4)
    assert run_sequence(sim, np.random.default_rng(bits)) >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("K", [8, 24, 16])
@pytest.mark.parametrize("mix", MIXES)
def test_cuda_cores_event_sequence_equals_the_oracle(gp, K, mix):
    sim = Sim(gp, "affinity", 48, 4000, K, seed=K + MIXES.index(mix), mix=mix, var="ffma", dead=(5,), zero_weight=(30,), cap=(1, 1), rounds=4)
    assert run_sequence(sim, np.random.default_rng(K)) >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("M", [48, 64, 65, 256, 257])
@pytest.mark.parametrize("mix", ["lognormal", "zeros"])
def test_tensor_cores_event_sequence_equals_the_oracle_on_integer_features(gp, M, mix):
    rng = np.random.default_rng(M)
    n = 4000
    sim = Sim(gp, "affinity", M, n, 16, seed=M, mix=mix, var="umma", fo=int_feats(rng, (n, 16)), fn=int_feats(rng, (M, 16)))
    run_sequence(sim, rng)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [2304, 2305])
def test_live_count_at_the_tensor_core_limit(gp, M):
    rng = np.random.default_rng(M)
    n = 5000
    sim = Sim(gp, "affinity", M, n, 16, seed=M, mix="hot", var="umma", fo=int_feats(rng, (n, 16)), fn=int_feats(rng, (M, 16)))
    run_sequence(sim, rng, skip=("all leave", "k = 0 with no live node", "all rejoin"))


@pytest.mark.gpu
def test_tensor_cores_with_uniform_features_equal_the_engine_restatement(gp):
    sim = Sim(gp, "affinity", 200, 12000, 16, seed=11, mix="uniform", var="umma", engine=True, dead=(3,))
    run_sequence(sim, np.random.default_rng(11), skip=("all leave", "k = 0 with no live node", "all rejoin"))


@pytest.mark.gpu
@pytest.mark.parametrize("policy", ["hrw", "hrw2", "affinity"])
def test_explicit_load_total_and_zero_weight_objects(gp, policy):
    K = 8 if policy == "affinity" else 0
    sim = Sim(gp, policy, 24, 1200, K, seed=3, mix="zeros", cap=(1, 1), rounds=16)
    big = int(sim.ow.astype(np.int64).sum()) * 2
    sim.call(sim.set_active([4], False), (5, 4), 8, load_total=int(sim.ow.astype(np.int64).sum()), tag="explicit = G")
    sim.call(sim.set_active([4], True), (1, 1), 16, load_total=big, tag="explicit > G")
    sim.call(sim.drift(0.1), (1, 1), 16, tag="drift")
    z = sim.s.read()[sim.ow == 0]
    sim.call(sim.set_active([5, 6], False), (1, 1), 16, tag="zero-weight objects only move off leaving nodes")
    after = sim.s.read()[sim.ow == 0]
    assert ((after == z) | np.isin(z, [5, 6])).all()


# ---- identity anchors ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("K,var", [(8, "ffma"), (16, "ffma"), (16, "umma")])
def test_all_ones_equal_the_bounded_affinity_change_call(gp, K, var):
    """Every weight 1 and load_total = n equals set_rebalance_changes_bounded_affinity on a twin set: idx, counters, moved, passes."""
    sim = Sim(gp, "affinity", 48, 6000, K, seed=K, mix="ones", var=var, dead=(5,), cap=(1, 1), rounds=4)
    n = len(sim.keys)
    twin = sim.p.new_set(n)
    twin.load_keys(sim.keys)
    twin.load_feats(sim.fo)
    with variant(var):
        twin.assign_bounded_affinity(n, 1, 1, 4)
        sim.s.assign_bounded_weighted(True, n, 1, 1, 4)
    assert twin.read().tobytes() == sim.s.read().tobytes()
    rng = np.random.default_rng(K)
    fired = 0
    for t, (name, ev) in enumerate(events(sim, rng)):
        if name in ("drift", "churn", "drift again"):
            continue
        cap, rounds = SCHEDULE[t % len(SCHEDULE)]
        idx, prev = ev()
        with variant(var):
            a = twin.rebalance_changes_bounded_affinity(idx, prev, n, cap[0], cap[1], rounds)
            b = sim.s.rebalance_changes_bounded_weighted(idx, prev, n, cap[0], cap[1], rounds)
        assert a == b and twin.read().tobytes() == sim.s.read().tobytes() and (twin.counters() == sim.s.counters()).all(), name
        fired += a[1] > 1
    assert fired >= 2


@pytest.mark.gpu
def test_flat_hrw_with_an_unreachable_capacity_equals_the_plain_change_call(gp):
    sim = Sim(gp, "hrw", 40, 3000, seed=21, mix="lognormal", cap=(1000, 1), rounds=4)
    twin = sim.p.new_set(len(sim.keys))
    twin.load_keys(sim.keys)
    twin.assign()
    assert twin.read().tobytes() == sim.s.read().tobytes()
    for name, ev in events(sim, np.random.default_rng(21)):
        if name in ("drift", "churn", "drift again"):
            continue
        idx, prev = ev()
        a = twin.rebalance_changes(idx, prev)
        moved, passes = sim.s.rebalance_changes_bounded_weighted(idx, prev, 0, 1000, 1, 4)
        assert (moved, passes) == (a, 1) and twin.read().tobytes() == sim.s.read().tobytes() and (twin.counters() == sim.s.counters()).all(), name


@pytest.mark.gpu
@pytest.mark.parametrize("policy", ["hrw", "hrw2", "affinity"])
def test_k_zero_after_a_balanced_assign_moves_nothing(gp, policy):
    K = 8 if policy == "affinity" else 0
    sim = Sim(gp, policy, 32, 3000, K, seed=31, mix="uniform")
    L = int(sim.ow.astype(np.int64).sum())
    W_ = int(sim.w[sim.live].astype(np.int64).sum())
    for num, den in [(5, 4), (3, 2), (2, 1), (4, 1)]:   # the first factor whose rounds end with no node over capacity
        sim.s.assign_bounded_weighted(sim.aff, 0, num, den, 16)
        cap = np.array([S.capacity(L, int(sim.w[j]), W_, num, den) if sim.live[j] else 0 for j in range(sim.M)])
        if (sim.s.loads() <= cap).all():
            break
    else:
        pytest.fail("no factor ended balanced")
    before = sim.s.read()
    assert sim.s.rebalance_changes_bounded_weighted([], [], 0, num, den, 16) == (0, 1)
    assert sim.s.read().tobytes() == before.tobytes()


# ---- the record ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("policy", ["hrw", "affinity"])
def test_record_dropped_and_kept(gp, policy):
    K = 8 if policy == "affinity" else 0
    aff = policy == "affinity"
    sim = Sim(gp, policy, 16, 500, K, seed=41)
    s, R = sim.s, gp

    def fresh():
        s.load_keys(sim.keys)
        if K:
            s.load_feats(sim.fo)
        s.write_weights(sim.ow)
        s.assign_bounded_weighted(aff)

    keeping = [
        ("insert", lambda: s.insert(sim.keys[:3] + np.uint64(1), sim.fo[:3] if K else None)),
        ("erase", lambda: s.erase(sim.keys[:2])),
        ("write_weights", lambda: s.write_weights(np.full(4, 3, np.uint32))),
        ("write_weights_by_key", lambda: s.write_weights_by_key(sim.keys[5:9], np.full(4, 2, np.uint32))),
        ("commit", lambda: s.commit()),
        ("commit_changes", lambda: s.commit_changes()),
    ] + ([] if aff else [("load_feats on a hash record", lambda: s.load_feats(np.zeros((s.size(), 4), np.float32)))])
    dropping = [
        ("assign", lambda: s.assign(aff)),
        ("assign_bounded", lambda: s.assign_bounded(0, 5, 4, 4)),
        ("rebalance", lambda: (sim.p.node_set_active(1, False), s.rebalance(1, 1), sim.p.node_set_active(1, True))),
        ("rebalance_changes", lambda: s.rebalance_changes([], [])),
        ("assign_ranked", lambda: s.assign_ranked(2)),
        ("load_keys", lambda: s.load_keys(sim.keys)),
        ("synth_keys", lambda: s.synth_keys(0, 500, 3)),
    ]
    if aff:
        dropping += [("assign_bounded_affinity", lambda: s.assign_bounded_affinity(0, 5, 4, 4)),
                     ("load_feats", lambda: s.load_feats(sim.fo[:s.size()]))]
    for name, call in keeping:
        fresh()
        call()
        s.rebalance_changes_bounded_weighted([], [])
    for name, call in dropping:
        fresh()
        call()
        with pytest.raises(R.Unknown):
            s.rebalance_changes_bounded_weighted([], [])


# ---- refusals --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_errors_change_nothing(gp):
    R = gp
    sim = Sim(gp, "affinity", 16, 400, 16, seed=8)
    s, p, L = sim.s, sim.p, sim.p.L

    def state():
        k, idx = s.read(want_keys=True)
        return s.size(), k.tobytes(), idx.tobytes(), s.counters().tobytes(), s.read_weights().tobytes()

    def refused(call, tag, exc=R.Unknown):
        before = state()
        with pytest.raises(exc):
            call()
        assert state() == before, tag
        s.rebalance_changes_bounded_weighted([], [])   # the record survived

    assert L.rio_cuda_set_rebalance_changes_bounded_weighted(None, None, None, 0, 0, 5, 4, 4, None, None) != 0
    assert L.rio_cuda_set_write_weights_by_key(None, None, None, 0, None) != 0
    refused(lambda: s.rebalance_changes_bounded_weighted([], [], 0, 5, 0, 4), "cap_den 0")
    refused(lambda: s.rebalance_changes_bounded_weighted([], [], 0, 5, 4, 0), "max_rounds 0")
    refused(lambda: s.rebalance_changes_bounded_weighted([99], [1]), "change-set index out of range")
    refused(lambda: s.rebalance_changes_bounded_weighted([2, 2], [1, 1]), "duplicate change-set index")
    refused(lambda: s._ck(L.rio_cuda_set_rebalance_changes_bounded_weighted(s.s, None, None, 2, 0, 5, 4, 4, None, None)), "null change set")
    refused(lambda: s.rebalance_changes_bounded_weighted([], [], int(sim.ow.sum()) - 1), "load_total below G")
    refused(lambda: s.rebalance_changes_bounded_weighted([], [], 1 << 32), "load_total past u32")
    refused(lambda: s._ck(L.rio_cuda_set_write_weights_by_key(s.s, None, None, 3, None)), "null keys")
    s.load_feats(sim.fo[:, :8])
    with pytest.raises(R.Unknown):
        s.rebalance_changes_bounded_weighted([], [])   # load_feats dropped the affinity record
    s.load_feats(sim.fo)
    s.assign_bounded_weighted(True)
    # a handle K other than the recorded one
    q = sim.handle(sim.active)
    t = q.new_set(100)
    t.load_keys(sim.keys[:100])
    t.load_feats(sim.fo[:100])
    t.assign_bounded_weighted(True)
    q.set_nodes(addresses(sim.M), sim.w, sim.fn[:, :8])
    with pytest.raises(R.Unknown):
        t.rebalance_changes_bounded_weighted([], [])
    # another solver than the recorded one; then a bounded call in flight: every _begin drops the record, so the rebalance refuses for
    # want of one, and the by-key write refuses for the call in flight
    h = Sim(gp, "hrw", 16, 400, seed=9)
    s2 = h.s
    h.p.set_solver("hrw2", 12)
    with pytest.raises(R.Unknown):
        s2.rebalance_changes_bounded_weighted([], [])   # another solver than the recorded one
    h.p.set_solver("hrw", 12)
    u = h.p.new_set(100)
    u.load_keys(h.keys[:100])
    u.assign_bounded_weighted(False)
    u.assign_bounded_begin(0, 5, 4, 4)
    with pytest.raises(R.Unknown):
        u.rebalance_changes_bounded_weighted([], [])
    with pytest.raises(R.Unknown):
        u.write_weights_by_key(h.keys[:3], np.ones(3, np.uint32))
    u.assign_bounded_end()
    # the u32 rule: G of exactly 2^32 - 1 runs, one more is refused with the set unchanged
    big = np.zeros(len(h.keys), np.uint32)
    big[0], big[1] = U32 - 5, 5
    s2.write_weights(big)
    s2.rebalance_changes_bounded_weighted([], [])
    big[2] = 1
    s2.write_weights(big)
    before = (s2.read().tobytes(), s2.counters().tobytes(), s2.read_weights().tobytes())
    with pytest.raises(R.Unknown):
        s2.rebalance_changes_bounded_weighted([], [])
    assert (s2.read().tobytes(), s2.counters().tobytes(), s2.read_weights().tobytes()) == before


# ---- writes by key ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_write_weights_by_key(gp):
    p = gp.GpuObjectPlacement()
    p.set_nodes(addresses(8))
    rng = np.random.default_rng(5)
    keys = rng.integers(0, 2**63, 3000, dtype=np.uint64)
    keys[10] = keys[20] = keys[30]                       # a key in three rows
    keys[40] = np.uint64(U32 * (2**32 + 1))              # ~0
    keys[41] = keys[40] - np.uint64(1)
    s = p.new_set(4000)
    s.load_keys(keys)
    assert s.write_weights_by_key(keys[:0], np.zeros(0, np.uint32)) == 0    # m = 0 writes nothing
    assert (s.read_weights() == 1).all()
    # first write: the column, 1 elsewhere; duplicates in the list: the last occurrence wins; absent keys ignored; weight 0
    wk = np.array([keys[5], keys[30], 12345, keys[5], keys[40], keys[7]], np.uint64)
    wv = np.array([7, 9, 11, 8, 13, 0], np.uint32)
    assert s.write_weights_by_key(wk, wv) == 6
    want = np.ones(len(keys), np.uint32)
    want[5], want[[10, 20, 30]], want[40], want[7] = 8, 9, 13, 0
    assert s.read_weights().tobytes() == want.tobytes()
    # against write_weights on the same rows after an erase has moved them
    gone = keys[rng.choice(3000, 300, replace=False)]
    rows = BW.erase_pairing(keys, gone)
    erased = s.erase(gone)
    keys, want = keys[rows], want[rows]
    assert s.size() == 3000 - erased and s.read_weights().tobytes() == want.tobytes()
    _, first, count = np.unique(keys, return_index=True, return_counts=True)
    pick = rng.choice(first[count == 1], 500, replace=False)            # rows whose key no other row holds
    nw = rng.integers(0, 1000, 500).astype(np.uint32)
    twin = p.new_set(4000)
    twin.load_keys(keys)
    twin.write_weights(want)
    for r, v in zip(pick, nw):
        twin.write_weights(np.array([v], np.uint32), first=int(r))
    assert s.write_weights_by_key(keys[pick], nw) == 500
    assert s.read_weights().tobytes() == twin.read_weights().tobytes()
    # many keys, most absent
    many = rng.integers(0, 2**63, 50_000, dtype=np.uint64)
    assert s.write_weights_by_key(many, np.full(len(many), 3, np.uint32)) == int(np.isin(keys, many).sum())


# ---- two ranks -------------------------------------------------------------------------------------------------------------------
def _worker(rank, world, port, n, M, q, comm):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["RIO_COMM"] = comm
    import torch.distributed as dist

    import rio_rs_b200 as R
    from rio_rs_b200 import parallel

    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)  # bootstrap only
    p = R.GpuObjectPlacement(device=rank)
    parallel.init_comm(p, dist)
    lo, hi = parallel.shard_range(n, rank, world)
    q.put((rank, lo, hi, _ranks_sequence(R, p, n, M, lo, hi)))
    dist.barrier()
    dist.destroy_process_group()


def _ranks_sequence(R, p, n, M, lo, hi):
    rng = np.random.default_rng(78)
    fo = rng.uniform(-1, 1, (n, 16)).astype(np.float32)
    fn = rng.uniform(-1, 1, (M, 16)).astype(np.float32)
    w = rng.integers(1, 17, M).astype(np.uint32)
    ow = weight_mix("lognormal", n, rng)
    keys = rng.integers(0, 2**63, n, dtype=np.uint64)
    out = {}
    for aff in (False, True):
        p.set_nodes(addresses(M), w, fn)
        s = p.new_set(hi - lo)
        s.load_keys(keys[lo:hi])
        s.load_feats(fo[lo:hi])
        s.write_weights(ow[lo:hi])
        s.assign_bounded_weighted(aff, 0, 5, 4, 8)
        p.node_set_active(3, False)
        out[aff, 0] = s.rebalance_changes_bounded_weighted([3], [int(w[3])], 0, 1, 1, 8), s.read().tolist(), s.counters().tolist(), s.loads().tolist()
        s.write_weights_by_key(keys[::7], np.full(len(keys[::7]), 50, np.uint32))
        out[aff, 1] = s.rebalance_changes_bounded_weighted([], [], 0, 1, 1, 8), s.read().tolist(), s.counters().tolist(), s.loads().tolist()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("comm", ["p2p", "nccl"])
def test_two_ranks_equal_one_rank_on_the_global_set(gp, comm):
    """Two ranks with one shard each: passes, idx, counters and loads equal the one-rank call on the global set, and the moved counts
    add up.  Skipped with fewer than two GPUs."""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    n, M, world = 200_000, 96, 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 500 + (11 if comm == "nccl" else 0)
    procs = [ctx.Process(target=_worker, args=(r, world, port, n, M, q, comm)) for r in range(world)]
    try:
        for pr in procs:
            pr.start()
        res = sorted(q.get(timeout=600) for _ in range(world))
        for pr in procs:
            pr.join(timeout=120)
    finally:   # a worker that failed or got stuck must not outlive the test
        for pr in procs:
            if pr.is_alive():
                pr.kill()
                pr.join(timeout=30)
    want = _ranks_sequence(gp, gp.GpuObjectPlacement(), n, M, 0, n)
    for key, ((moved, passes), idx, cnt, ld) in want.items():
        assert sum(out[key][0][0] for _, _, _, out in res) == moved, key
        for _, lo, hi, out in res:
            (_, gpasses), gi, gc, gl = out[key]
            assert gpasses == passes and gi == idx[lo:hi] and gc == cnt and gl == ld, key


# ---- host-sim --------------------------------------------------------------------------------------------------------------------
DOUBLES = os.path.join(ROOT, "tests", "cpp", "hostsim", "set_weighted_changes_launchers.cpp")
OTHER_DOUBLES = [os.path.join(ROOT, "tests", "cpp", "hostsim", f) for f in ("ranked_launchers.cpp", "change_launchers.cpp", "ranked_change_launchers.cpp",
                                                                              "spread_launchers.cpp", "spread_change_launchers.cpp",
                                                                              "affinity_ranked_launchers.cpp", "affinity_spread_launchers.cpp",
                                                                              "affinity_set_launchers.cpp", "affinity_bounded_launchers.cpp",
                                                                              "set_bounded_affinity_launchers.cpp", "set_churn_launchers.cpp",
                                                                              "set_commit_launchers.cpp", "bounded_weighted_launchers.cpp")]


def test_the_doubles_cover_the_new_launchers():
    decl = set(re.findall(r"\b(launch_[a-z0-9_]+)\s*\(", open(os.path.join(ROOT, "rio_rs_b200", "csrc", "k_set_weighted_changes.cuh")).read()))
    have = set(re.findall(r"^void\s+([a-z0-9_]+)\s*\(", open(DOUBLES).read(), flags=re.M))
    assert len(decl) == 3 and decl <= have, decl - have


def _hostsim_library(HS, name, doubles):
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, name)
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + doubles + ["-o", so, "-ldl", "-lpthread"])
    return so


def test_weighted_change_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + every double, the new one
    included)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_weighted_changes.so", OTHER_DOUBLES + [DOUBLES])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider",
           "-k", "not two_ranks"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=3000, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 40 and "failed" not in r.stdout, tail


@pytest.mark.parametrize("world", [2, 4])
def test_ranks_equal_one_rank_on_the_host_logic(world):
    """tests/hostsim_multirank_weighted_changes.py: `world` ranks as threads of one process over the host-sim library."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_weighted_changes_mr.so", OTHER_DOUBLES + [DOUBLES])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostsim_multirank_weighted_changes.py"), str(world)], capture_output=True, text=True,
                       timeout=900, env=env, cwd=ROOT)
    assert r.returncode == 0 and "multirank weighted changes ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


def test_both_calls_report_an_error_where_their_kernels_are_not_linked():
    """The engine's host code built WITHOUT the new launchers refuses both calls with RIO_ERR_UPSTREAM and changes nothing; the weighted
    assign, the other weight calls, churn, the commits and the count-based change calls keep working."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_no_weighted_changes.so", OTHER_DOUBLES)
    code = (
        "import sys, numpy as np\n"
        "from rio_rs_b200 import _native as N\n"
        "N.library_path = lambda: sys.argv[1]\n"
        "import rio_rs_b200 as R\n"
        "p = R.GpuObjectPlacement()\n"
        "p.set_nodes(['10.0.0.%d:5000' % j for j in range(8)])\n"
        "keys = np.arange(100, dtype=np.uint64)\n"
        "s = p.new_set(200); s.load_keys(keys); s.write_weights(np.arange(100, dtype=np.uint32))\n"
        "assert s.assign_bounded_weighted(False, 0, 5, 4, 4) >= 1\n"
        "before = (s.read().tobytes(), s.read_weights().tobytes(), s.counters().tobytes())\n"
        "p.node_set_active(2, False)\n"
        "for call in (lambda: s.write_weights_by_key(keys[:3], np.ones(3, np.uint32)), lambda: s.rebalance_changes_bounded_weighted([2], [1])):\n"
        "    try:\n"
        "        call()\n"
        "        raise SystemExit('ran without kernels')\n"
        "    except R.Upstream as e:\n"
        "        assert 'weighted change-set kernels' in str(e), e\n"
        "assert (s.read().tobytes(), s.read_weights().tobytes(), s.counters().tobytes()) == before\n"
        "s.write_weights(np.ones(100, dtype=np.uint32)); assert s.loads().sum() == 100\n"
        "assert s.erase(keys[90:]) == 10 and s.insert(keys[90:]) == 90\n"
        "s.commit_changes(); s.rebalance_changes([2], [1]); assert s.counters().sum() == 100\n"
        "print('refused ok')\n"
    )
    r = subprocess.run([sys.executable, "-c", code, so], capture_output=True, text=True, timeout=300, cwd=HS.ROOT)
    assert r.returncode == 0 and "refused ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

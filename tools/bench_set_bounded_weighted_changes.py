"""Weighted bounded sets kept within load capacity (DESIGN.md 3.21): set_rebalance_changes_bounded_weighted after one event against a
fresh set_assign_bounded_weighted of the same state on a twin set, and set_write_weights_by_key.

Workload: a resident set of 10 M objects over M = 1024 nodes of weights 1..16, cap 5/4, max_rounds 8 and 16; object weights lognormal
(sigma = 1.5, scaled so the total stays near 2^31, clipped to [1, 2^20]) and 1 % hot at 100x.  Policies: HRW2, flat HRW, and affinity
on the tensor cores (K = 16, features U(-1, 1)).  Events, in this order from a weighted assign: a node of weight 1 leaves, a node of
weight 16 leaves, a rack of 32 nodes leaves, a new node of weight 8 joins, 8 nodes halve their weight, and 1 % of the objects get new
weights written by key (k = 0).  Per event: ms of the change-set call and of the fresh call (median of `--trials` repetitions of the
whole sequence after one warm-up repetition; host clock around the call and a device synchronise), passes, objects moved by each
(the fresh call's moves counted against the state before the event), the lower bound (objects on nodes that left or, under the hash
policies, lost weight), and the largest load / capacity over live nodes after each call.  Then a 32-event run (random leaves, joins,
weight changes and drift) under HRW2 that reports how the fullest node and the moves drift, and the by-key write at m = 10 k, 100 k
and 1 M.  The card's name, power limit and max SM clock are read in the same run.  Writes nothing into the source tree; `--out FILE`
also writes the JSON there.
usage: python tools/bench_set_bounded_weighted_changes.py [--n 10000000] [--trials 3] [--out FILE]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_bounded_affinity import card_info  # noqa: E402
from bench_set_bounded_weighted import addr, timed, weights_of  # noqa: E402

M, K = 1024, 16
CAP = (5, 4)
POLICIES = ["hrw2", "hrw", "affinity_tensor"]
MIXES = ["lognormal", "hot"]
ROUNDS = [8, 16]


def capacity(L, w, W, num, den):
    return -(-(num * L * w) // (den * W)) if w and W else 0


def fullest(s, live_w, L):
    """max over live nodes of load / capacity"""
    ld = s.loads()[:len(live_w)].astype(np.float64)
    W = int(live_w.sum())
    caps = np.array([capacity(L, int(w), W, *CAP) for w in live_w], np.float64)
    on = caps > 0
    return float((ld[on] / caps[on]).max()) if on.any() else 0.0


class Bench:
    def __init__(self, R, policy, n, mix, rounds, seed=1):
        self.R, self.policy, self.n, self.rounds = R, policy, n, rounds
        rng = np.random.default_rng(seed)
        self.w0 = rng.integers(1, 17, M).astype(np.uint32)
        self.w0[0], self.w0[1] = 1, 16   # the two single leaves
        self.fn = rng.uniform(-1, 1, (M + 1, K)).astype(np.float32)
        self.aff = policy.startswith("affinity")
        self.p = R.GpuObjectPlacement()
        self.p.set_solver("hrw2" if policy == "hrw2" else "hrw", 12)
        self.s, self.t = self.p.new_set(n), self.p.new_set(n)
        for x in (self.s, self.t):
            x.synth_keys(0, n, 77)
        self.keys = self.s.read(want_keys=True)[0]
        self.ow = weights_of(mix, n, rng)
        if self.aff:
            fo = rng.uniform(-1, 1, (n, K)).astype(np.float32)
            for x in (self.s, self.t):
                x.load_feats(fo)
            del fo
        self.rack = rng.choice(np.arange(2, M), 32, replace=False)
        self.halve = rng.choice(np.setdiff1d(np.arange(2, M), self.rack), 8, replace=False)
        self.drift_rows = rng.choice(n, n // 100, replace=False)
        self.drift_w = self.ow[rng.choice(n, len(self.drift_rows))]   # new weights from the same distribution as the set's

    def reset(self):
        os.environ["RIO_AFFINITY_VARIANT"] = "umma"
        self.w = self.w0.copy()
        self.p.set_nodes([addr(j) for j in range(M)], self.w, self.fn[:M])
        if self.p.node_count()[0] > M:   # the node the last repetition joined leaves again
            self.p.node_set_active(M, False)
        self.live = np.ones(M, bool)
        self.ow_now = self.ow.copy()
        for x in (self.s, self.t):
            x.write_weights(self.ow)
        self.s.assign_bounded_weighted(self.aff, 0, CAP[0], CAP[1], self.rounds)

    def events(self):
        def leave(js):
            for j in js:
                self.p.node_set_active(int(j), False)
                self.live[j] = False
            return [int(j) for j in js], [int(self.w[j]) for j in js], list(js)

        def join():
            j = self.p.node_upsert(addr(M), 8, self.fn[M])
            self.w = np.append(self.w, np.uint32(8))
            self.live = np.append(self.live, True)
            return [j], [0], []

        def halve():
            prev = [int(self.w[j]) for j in self.halve]
            for j in self.halve:
                self.w[j] = max(int(self.w[j]) // 2, 1)
                self.p.node_upsert(addr(int(j)), int(self.w[j]))
            return [int(j) for j in self.halve], prev, ([] if self.aff else list(self.halve))

        def drift():
            self.s.write_weights_by_key(self.keys[self.drift_rows], self.drift_w)
            self.t.write_weights_by_key(self.keys[self.drift_rows], self.drift_w)
            self.ow_now[self.drift_rows] = self.drift_w
            return [], [], []

        return [("leave w=1", lambda: leave([0])), ("leave w=16", lambda: leave([1])), ("rack of 32 leaves", lambda: leave(self.rack)),
                ("join w=8", join), ("8 nodes halve", halve), ("1 % drift by key", drift)]

    def run_once(self):
        self.reset()
        rows = []
        for name, ev in self.events():
            before = self.s.read()
            idx, prev, replaced = ev()
            lower = int(np.isin(before, np.asarray(replaced, np.uint32)).sum()) if replaced else 0
            L = int(self.ow_now.astype(np.int64).sum())
            live_w = np.where(self.live, self.w, 0)
            ms_new, (moved, passes) = timed(self.p, lambda: self.s.rebalance_changes_bounded_weighted(idx, prev, 0, CAP[0], CAP[1], self.rounds))
            over_new = fullest(self.s, live_w, L)
            ms_fresh, fpasses = timed(self.p, lambda: self.t.assign_bounded_weighted(self.aff, 0, CAP[0], CAP[1], self.rounds))
            fresh_moved = int((self.t.read() != before).sum())
            over_fresh = fullest(self.t, live_w, L)
            rows.append(dict(event=name, ms_new=ms_new, ms_fresh=ms_fresh, passes=passes, passes_fresh=fpasses, moved=moved, moved_fresh=fresh_moved,
                             lower_bound=lower, max_load_over_cap=over_new, max_load_over_cap_fresh=over_fresh))
        return rows


def drift_run(R, n, events=32, seed=5):
    b = Bench(R, "hrw2", n, "lognormal", 8, seed)
    b.reset()
    rng = np.random.default_rng(seed)
    out = []
    for e in range(events):
        before = b.s.read()
        kind = e % 4
        if kind == 0:    # a live node leaves
            j = int(rng.choice(np.flatnonzero(b.live)))
            b.p.node_set_active(j, False)
            b.live[j] = False
            idx, prev, lower = [j], [int(b.w[j])], int((before == j).sum())
        elif kind == 1:  # a dead node rejoins
            dead = np.flatnonzero(~b.live)
            j = int(rng.choice(dead)) if len(dead) else 0
            b.p.node_set_active(j, True)
            b.live[j] = True
            idx, prev, lower = [j], [0], 0
        elif kind == 2:  # a live node changes weight
            j = int(rng.choice(np.flatnonzero(b.live)))
            pw, nw = int(b.w[j]), int(rng.integers(1, 17))
            b.p.node_upsert(addr(j), nw)
            b.w[j] = nw
            idx, prev, lower = [j], [pw], int((before == j).sum()) if nw < pw else 0
        else:            # 1 % of the objects drift
            rows = rng.choice(n, n // 100, replace=False)
            nw = b.ow[rng.choice(n, len(rows))]
            b.s.write_weights_by_key(b.keys[rows], nw)
            b.ow_now[rows] = nw
            idx, prev, lower = [], [], 0
        ms, (moved, passes) = timed(b.p, lambda: b.s.rebalance_changes_bounded_weighted(idx, prev, 0, CAP[0], CAP[1], 8))
        out.append(dict(event=e, kind=["leave", "rejoin", "reweight", "drift"][kind], ms=ms, passes=passes, moved=moved, lower_bound=lower,
                        max_load_over_cap=fullest(b.s, np.where(b.live, b.w, 0), int(b.ow_now.astype(np.int64).sum()))))
    return out


def by_key(R, n, trials):
    p = R.GpuObjectPlacement()
    p.set_nodes([addr(j) for j in range(M)])
    s = p.new_set(n)
    s.synth_keys(0, n, 77)
    keys = s.read(want_keys=True)[0]
    rng = np.random.default_rng(9)
    out = []
    for m in [m for m in (10_000, 100_000, 1_000_000) if m <= n]:
        k = keys[rng.choice(n, m, replace=False)]
        w = rng.integers(1, 100, m).astype(np.uint32)
        s.write_weights_by_key(k, w)   # warm-up (and the column)
        ts = sorted(timed(p, lambda: s.write_weights_by_key(k, w))[0] for _ in range(max(trials, 5)))
        out.append(dict(m=m, ms_median=ts[len(ts) // 2], ms_min=ts[0], ms_max=ts[-1]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--trials", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    import rio_rs_b200 as R
    from rio_rs_b200 import build

    build.build()
    res = dict(card=card_info(), n=a.n, M=M, cap=CAP, cases=[])
    for policy in POLICIES:
        for mix in MIXES:
            for rounds in ROUNDS:
                b = Bench(R, policy, a.n, mix, rounds)
                b.run_once()   # warm-up repetition
                reps = [b.run_once() for _ in range(a.trials)]
                rows = []
                for i, r in enumerate(reps[0]):
                    for col in ("ms_new", "ms_fresh"):
                        r[col] = float(np.median([rep[i][col] for rep in reps]))
                    rows.append(r)
                res["cases"].append(dict(policy=policy, mix=mix, rounds=rounds, events=rows))
                print(json.dumps(res["cases"][-1]), flush=True)
                del b
    res["drift"] = drift_run(R, a.n)
    print(json.dumps(dict(drift=res["drift"])), flush=True)
    res["by_key"] = by_key(R, a.n, a.trials)
    print(json.dumps(dict(by_key=res["by_key"], card=res["card"])), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

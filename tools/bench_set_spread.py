"""Timing of the failure-domain change set (DESIGN.md 3.13) against recomputing every list, and against a plain ranked set's change
set for the same workload, both policies.

Workload: a resident set of `--n` synthetic keys (default 100 M) over M0 = 1024 nodes with weights 1..16 in 32 racks of 32, plus four
spare nodes, holding its spread lists for R = 2, 4 and 8; a plain ranked set of the same keys holds its ranked lists beside it.  Four
membership changes, each applied as one change set:
  c5       C5's eight join/leave events (the spares join their racks);
  rack     one rack of 32 leaves;
  halve    one node halves its weight;
  relabel  one node moves to another rack, k = 0.
Each is timed as the spread change set (set.rebalance_changes_ranked on the spread set), as a full set.assign_ranked_spread(R) after
the same update, and as the plain ranked set's change set (for relabel: its k = 0 call, which ignores labels).  A point's time is a
host clock around the node-table update and the call, which ends in a device synchronise; after every timed point the state is put
back by one untimed change set, so every window starts from the same lists.  Every point is warmed up once, then `--trials` windows
are taken round-robin; the median and min..max are reported.  The card's name, power limit and max SM clock are read in the same run.
After the timing, every workload is applied once more and the lists of a `--check`-object sample are compared with the spread CPU
oracle.  Writes nothing into the source tree; `--out FILE` also writes the JSON there.
usage: python tools/bench_set_spread.py [--n N] [--trials T] [--check C] [--ranks 2,4,8] [--out FILE]"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_set_ranked import C5, M0, card_info  # noqa: E402

RACK = list(range(192, 224))   # rack 6
HALVE = [150]
RELABEL = 300                  # rack 9 -> rack 20
WORKLOADS = ("c5", "rack", "halve", "relabel")


class Bench:
    def __init__(self, R, O, n, policy, ranks):
        self.p = R.GpuObjectPlacement(device=0)
        self.p.set_solver(policy, 12)
        self.ranks = ranks
        self.addrs, self.seeds, self.w = O.synth_nodes(M0 + 4)
        self.live = self.w.copy()
        self.live[M0:] = 0
        self.p.set_nodes(self.addrs[:M0], self.w[:M0])
        for j in range(M0, M0 + 4):
            assert self.p.node_intern(self.addrs[j]) == j
        self.dom = (np.arange(M0 + 4) // 32).astype(np.uint32)
        self.dom[M0:] = [17, 3, 100 // 32, 64 // 32]   # each spare joins the rack of the node C5 swaps it for
        self.p.set_node_domains(np.arange(M0 + 4, dtype=np.uint32), self.dom)
        self.s = self.p.new_set(n)
        self.s.synth_keys(0, n, 11)
        self.s.assign_ranked_spread(ranks)
        self.plain = self.p.new_set(n)
        self.plain.synth_keys(0, n, 11)
        self.plain.assign_ranked(ranks)
        self.p.sync()

    def set_weights(self, target):
        """Apply {node: new live weight} to the node table; returns the change set (idx, prev_weight)."""
        idx = np.array(sorted(target), dtype=np.uint32)
        prev = np.array([self.live[j] for j in idx], dtype=np.uint32)
        for j, nw in target.items():
            if nw:
                self.p.node_upsert(self.addrs[j], int(nw))
            else:
                self.p.node_set_active(int(j), False)
            self.live[j] = nw
        return idx, prev

    def relabel(self, label):
        self.dom[RELABEL] = label
        self.p.set_node_domains(np.array([RELABEL], np.uint32), np.array([label], np.uint32))

    def changes(self, wl):
        if wl == "c5":
            return {j: (0 if ev == "leave" else int(self.w[j])) for ev, j in C5}
        if wl == "rack":
            return {j: 0 for j in RACK}
        if wl == "halve":
            return {j: max(1, int(self.w[j]) // 2) for j in HALVE}
        return {}

    def apply(self, wl, forward):
        if wl == "relabel":
            self.relabel(20 if forward else RELABEL // 32)
            return np.empty(0, np.uint32), np.empty(0, np.uint32)
        target = self.changes(wl) if forward else {j: (int(self.w[j]) if j < M0 else 0) for j in self.changes(wl)}
        return self.set_weights(target)

    def forward(self, wl, how):
        """One timed application of workload wl; `how` = spread | assign | ranked.  Untimed, the other set then takes the same change
        set, so both sets always describe the current node table."""
        t0 = time.perf_counter()
        idx, prev = self.apply(wl, True)
        if how == "spread":
            self.s.rebalance_changes_ranked(idx, prev)
        elif how == "assign":
            self.s.assign_ranked_spread(self.ranks)
        else:
            self.plain.rebalance_changes_ranked(idx, prev)
        self.p.sync()
        ms = (time.perf_counter() - t0) * 1e3
        (self.s if how == "ranked" else self.plain).rebalance_changes_ranked(idx, prev)
        return ms

    def restore(self, wl):
        idx, prev = self.apply(wl, False)
        self.s.rebalance_changes_ranked(idx, prev)
        self.plain.rebalance_changes_ranked(idx, prev)
        self.p.sync()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--check", type=int, default=20_000)
    ap.add_argument("--ranks", default="2,4,8")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import rio_rs_b200 as R
    from rio_rs_b200 import build
    from oracle import pyoracle as O
    import spread_oracle as SO

    build.build()
    O.build()
    results, checks = {}, {}
    for policy in ("hrw", "hrw2"):
        for ranks in [int(r) for r in a.ranks.split(",")]:
            b = Bench(R, O, a.n, policy, ranks)
            points = [(wl, how) for wl in WORKLOADS for how in ("spread", "assign", "ranked")]
            times = {pt: [] for pt in points}
            for trial in range(a.trials + 1):   # trial 0 is the warm-up
                for pt in points:
                    ms = b.forward(*pt)
                    b.restore(pt[0])
                    if trial:
                        times[pt].append(ms)
            res = {}
            for (wl, how), v in times.items():
                v = np.array(v)
                res["%s/%s" % (wl, how)] = {"ms_median": round(float(np.median(v)), 3), "ms_min": round(float(v.min()), 3),
                                            "ms_max": round(float(v.max()), 3)}
            key = "%s/R%d" % (policy, ranks)
            results[key] = res
            # correctness after the timing: each workload once more, the first --check lists against the oracle
            keys, _ = b.s.read(0, a.check, want_keys=True)
            ok = {}
            for wl in WORKLOADS:
                idx, prev = b.apply(wl, True)
                b.s.rebalance_changes_ranked(idx, prev)
                want = SO.assign_spread(policy, keys, b.seeds, b.live, b.dom, ranks, threads=os.cpu_count() or 8)
                got = b.s.read_ranked(0, a.check)
                ok[wl] = bool((got == want).all() and (b.s.read(0, a.check) == want[:, 0]).all())
                b.plain.rebalance_changes_ranked(idx, prev)
                b.restore(wl)
            checks[key] = ok
            del b
    out = {"n": a.n, "nodes": M0, "racks": "32 x 32", "weights": "1..16", "trials": a.trials, "card": card_info(), "results_ms": results,
           "checks_vs_oracle": {"objects": a.check, **checks}}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")
    sys.exit(0 if all(all(v.values()) for v in checks.values()) else 1)


if __name__ == "__main__":
    main()

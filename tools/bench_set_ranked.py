"""Timing of the ranked change set (DESIGN.md 3.11) against recomputing every list, both policies.

Workload: a resident set of `--n` synthetic keys (default 100 M) over M0 = 1024 nodes with weights 1..16 plus four spare nodes,
holding its R-lists for R = 1, 2, 4 and 8.  Three membership changes, each applied as one change set:
  c5     C5's eight join/leave events;
  rack   32 nodes leave together;
  halve  8 nodes halve their weight.
Each is timed as the ranked change set (set.rebalance_changes_ranked) and as a full set.assign_ranked(R) after the same node-table
update; at R = 1 also as set.rebalance_changes on an unranked set of the same keys.  A point's time is a host clock around the
node-table updates and the call, which ends in a device synchronise; after every timed point the state is put back by one untimed
change set, so every window starts from the same lists.  Every point is warmed up once, then `--trials` windows are taken
round-robin; the median and min..max are reported.  The card's name, power limit and max SM clock are read in the same run.  After
the timing, every workload is applied once more and the lists of a `--check`-object sample are compared with the ranked CPU oracle.
Writes nothing into the source tree; `--out FILE` also writes the JSON there.
usage: python tools/bench_set_ranked.py [--n N] [--trials T] [--check C] [--ranks 1,2,4,8] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

M0 = 1024
C5 = [("leave", 17), ("join", M0), ("leave", 3), ("join", M0 + 1), ("leave", 100), ("join", M0 + 2), ("leave", 64), ("join", M0 + 3)]
RACK = list(range(200, 232))
HALVE = [5, 50, 150, 250, 350, 450, 550, 650]


def card_info():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clk}
    except Exception as e:  # noqa: BLE001
        return {"error": repr(e)}


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
        self.s = self.p.new_set(n)
        self.s.synth_keys(0, n, 11)
        self.s.assign_ranked(ranks)
        self.plain = None
        if ranks == 1:   # the unranked change set on the same keys
            self.plain = self.p.new_set(n)
            self.plain.synth_keys(0, n, 11)
            self.plain.assign()
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

    def changes(self, wl):
        if wl == "c5":
            return {j: (0 if ev == "leave" else int(self.w[j])) for ev, j in C5}
        if wl == "rack":
            return {j: 0 for j in RACK}
        return {j: max(1, int(self.w[j]) // 2) for j in HALVE}

    def forward(self, wl, how):
        """One timed application of workload wl; `how` = ranked | assign | plain."""
        t0 = time.perf_counter()
        idx, prev = self.set_weights(self.changes(wl))
        if how == "ranked":
            self.s.rebalance_changes_ranked(idx, prev)
        elif how == "assign":
            self.s.assign_ranked(self.ranks)
        else:
            self.plain.rebalance_changes(idx, prev)
        self.p.sync()
        return (time.perf_counter() - t0) * 1e3

    def restore(self, wl, how):
        base = {j: (int(self.w[j]) if j < M0 else 0) for j in self.changes(wl)}
        idx, prev = self.set_weights(base)
        if how == "plain":
            self.plain.rebalance_changes(idx, prev)
        else:
            self.s.rebalance_changes_ranked(idx, prev)
        self.p.sync()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100_000_000)
    ap.add_argument("--trials", type=int, default=7)
    ap.add_argument("--check", type=int, default=20_000)
    ap.add_argument("--ranks", default="1,2,4,8")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import rio_rs_b200 as R
    from rio_rs_b200 import build
    from oracle import pyoracle as O
    import ranked_oracle as RO

    build.build()
    O.build()
    results, checks = {}, {}
    for policy in ("hrw", "hrw2"):
        for ranks in [int(r) for r in a.ranks.split(",")]:
            b = Bench(R, O, a.n, policy, ranks)
            points = [(wl, how) for wl in ("c5", "rack", "halve") for how in (("ranked", "assign", "plain") if ranks == 1 else ("ranked", "assign"))]
            times = {pt: [] for pt in points}
            for trial in range(a.trials + 1):   # trial 0 is the warm-up
                for pt in points:
                    ms = b.forward(*pt)
                    b.restore(*pt)
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
            for wl in ("c5", "rack", "halve"):
                idx, prev = b.set_weights(b.changes(wl))
                b.s.rebalance_changes_ranked(idx, prev)
                want = RO.assign_ranked(policy, keys, b.seeds, b.live, ranks, threads=os.cpu_count() or 8)
                got = b.s.read_ranked(0, a.check)
                ok[wl] = bool((got == want).all() and (b.s.read(0, a.check) == want[:, 0]).all())
                b.restore(wl, "ranked")
            checks[key] = ok
            del b
    out = {"n": a.n, "nodes": M0, "weights": "1..16", "trials": a.trials, "card": card_info(), "results_ms": results,
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

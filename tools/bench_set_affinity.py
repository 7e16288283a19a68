"""Timing of the affinity change set (DESIGN.md 3.15) against recomputing every list, both kinds and both kernel paths.

Workload: a resident set of `--n` objects (default 10 M, the size of the DESIGN.md 7 affinity tables) with K = 16 features over
M0 = 1024 nodes in 32 racks of 32, plus four spare nodes interned with features and not live, holding its affinity lists (ranked or
failure-domain) for R = 1, 2, 4 and 8, assigned on the tensor cores (the default) or the CUDA cores (RIO_AFFINITY_VARIANT=ffma).
Workloads, each applied as one change set:
  leave      one node leaves;
  join       one spare joins;
  rack       a rack of 32 nodes leaves;
  refeature  one node gets a new feature row;
  halve      8 nodes halve their weight (a no-op for affinity lists);
  relabel    (failure-domain lists) one node moves to a rack of its own, k = 0.
Each is timed as the change set (set.rebalance_changes_ranked) and as a full set.assign_ranked_affinity(_spread)(R) after the same
node-table update.  A point's time is a host clock around the update and the call, which ends in a device synchronise; after every
timed point the update is undone and applied by one untimed change set, so every window starts from the same lists.  Every point is
warmed up once, then `--trials` windows are taken round-robin; the median and min..max are reported.  The card's name, power limit and
max SM clock are read in the same run.  After the timing every workload is applied once more and the first `--check` lists are
checked with the fp64 oracles.  Writes nothing into the source tree; `--out FILE` also writes the JSON there.
usage: python tools/bench_set_affinity.py [--n N] [--trials T] [--check C] [--ranks 1,2,4,8] [--out FILE]"""
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

M0, K = 1024, 16
RACK = list(range(64, 96))   # rack 2
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
    def __init__(self, R, O, fo, kind, path, ranks):
        self.kind, self.ranks = kind, ranks
        self.p = R.GpuObjectPlacement(device=0)
        self.addrs = O.synth_nodes(M0 + 4)[0]
        rng = np.random.default_rng(5)
        self.fn = rng.uniform(-1, 1, (M0 + 4, K)).astype(np.float32)
        self.fn_alt = rng.uniform(-1, 1, K).astype(np.float32)
        self.w = np.ones(M0 + 4, np.uint32) * 8
        self.live = np.ones(M0 + 4, bool)
        self.dom = (np.arange(M0 + 4) // 32).astype(np.uint32)
        self.p.set_nodes(self.addrs, self.w, self.fn)
        self.p.set_node_domains(np.arange(M0 + 4, dtype=np.uint32), self.dom)
        for j in range(M0, M0 + 4):
            self.p.node_set_active(j, False)
            self.live[j] = False
        self.s = self.p.new_set(len(fo))
        self.s.synth_keys(0, len(fo), 11)
        self.s.load_feats(fo)
        self.full()
        self.p.sync()

    def full(self):
        if self.kind == "spread":
            self.s.assign_ranked_affinity_spread(self.ranks)
        else:
            self.s.assign_ranked_affinity(self.ranks)

    def update(self, wl, undo=False):
        """Apply workload wl (or undo it) to the node table; returns the change set (idx, prev_weight)."""
        if wl in ("leave", "join", "rack"):
            js = {"leave": [17], "join": [M0], "rack": RACK}[wl]
            go_live = (wl == "join") != undo
            prev = [int(self.w[j]) if self.live[j] else 0 for j in js]
            for j in js:
                if go_live:
                    self.p.node_upsert(self.addrs[j], int(self.w[j]))
                else:
                    self.p.node_set_active(j, False)
                self.live[j] = go_live
            return js, prev
        if wl == "refeature":
            self.p.node_upsert(self.addrs[300], int(self.w[300]), self.fn[300] if undo else self.fn_alt)
            return [], []
        if wl == "halve":
            prev = [int(self.w[j]) for j in HALVE]
            for j in HALVE:
                self.w[j] = self.w[j] * 2 if undo else self.w[j] // 2
                self.p.node_upsert(self.addrs[j], int(self.w[j]))
            return HALVE, prev
        self.p.set_node_domains(np.array([400], np.uint32), np.array([self.dom[400] if undo else 9999], np.uint32))
        return [], []

    def forward(self, wl, how):
        t0 = time.perf_counter()
        idx, prev = self.update(wl)
        if how == "changes":
            self.s.rebalance_changes_ranked(idx, prev)
        else:
            self.full()
        self.p.sync()
        return (time.perf_counter() - t0) * 1e3

    def restore(self, wl):
        idx, prev = self.update(wl, undo=True)
        self.s.rebalance_changes_ranked(idx, prev)
        self.p.sync()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--check", type=int, default=20_000)
    ap.add_argument("--ranks", default="1,2,4,8")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import rio_rs_b200 as R
    from rio_rs_b200 import build
    from oracle import pyoracle as O
    import affinity_ranked_oracle as AO
    import affinity_spread_oracle as SO

    build.build()
    O.build()
    fo = np.random.default_rng(3).uniform(-1, 1, (a.n, K)).astype(np.float32)
    results, checks = {}, {}
    for path in ("tensor", "cuda"):
        if path == "cuda":
            os.environ["RIO_AFFINITY_VARIANT"] = "ffma"
        else:
            os.environ.pop("RIO_AFFINITY_VARIANT", None)
        for kind in ("ranked", "spread"):
            for ranks in [int(r) for r in a.ranks.split(",")]:
                b = Bench(R, O, fo, kind, path, ranks)
                wls = ["leave", "join", "rack", "refeature", "halve"] + (["relabel"] if kind == "spread" else [])
                points = [(wl, how) for wl in wls for how in ("changes", "full")]
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
                key = "%s/%s/R%d" % (path, kind, ranks)
                results[key] = res
                ok = {}
                for wl in wls:
                    idx, prev = b.update(wl)
                    b.s.rebalance_changes_ranked(idx, prev)
                    got = b.s.read_ranked(0, a.check)
                    fn = b.fn.copy()
                    if wl == "refeature":
                        fn[300] = b.fn_alt
                    dom = b.dom.copy()
                    if wl == "relabel":
                        dom[400] = 9999
                    try:
                        if kind == "spread":
                            SO.check(got, fo[:a.check], fn, b.live, dom)
                        else:
                            AO.check(got, fo[:a.check], fn, b.live)
                        ok[wl] = bool((b.s.read(0, a.check) == got[:, 0]).all())
                    except AssertionError as e:
                        ok[wl] = False
                        print("oracle check failed", key, wl, e, file=sys.stderr)
                    b.restore(wl)
                checks[key] = ok
                print(key, json.dumps(res), file=sys.stderr, flush=True)
                del b
    out = {"n": a.n, "nodes": M0, "K": K, "racks": 32, "trials": a.trials, "card": card_info(), "results_ms": results,
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

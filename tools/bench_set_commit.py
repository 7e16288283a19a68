"""Delta commit of a resident set (DESIGN.md 3.20): what rio_cuda_set_commit_changes and its dry run cost next to the full
rio_cuda_set_commit, after one membership or object event.

Workload: a resident set of `--n` objects (default 10 M, synthetic keys) over M = 1024 nodes of weights 1..16, under HRW2 (12 trie
bits) and flat HRW.  Two handles hold the same set and the same history: A commits with commit_changes, B with set_commit.  Each trial
starts from a committed set, applies one event to both sets and times, on A, the dry run and then the real call (both with manifest
buffers of n entries, so one C call each), and on B the full set_commit.  The event is then undone and committed, untimed.  Events: none;
the leave of a weight-1 node; the leave of a weight-16 node; a rack of 32 nodes leaving; a join of a new node of weight 8; 1 % churn
(erase 1 % random keys, insert as many new ones); a weighted bounded call (0.1 % of the objects at weight 100, cap 5/4, max_rounds 16,
from the plain assignment).  Times: host clock around the call and a device synchronise, median of `--trials` windows after one
warm-up trial, min..max beside it.  The pass-1 floor is the diff pass's algorithmic bytes (8 B key + 4 B idx + one 32-byte sector per
probe + 1 B flag per row) at 3.35 TB/s.  After every event A's and B's directories are compared on 200 k sampled keys.  The card's
name, power limit and max SM clock are read in the same run.  Writes nothing into the source tree; `--out FILE` also writes the JSON.
usage: python tools/bench_set_commit.py [--n N] [--trials T] [--policies hrw2,hrw] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_bounded_affinity import card_info  # noqa: E402

M = 1024
HBM_BPS = 3.35e12
PASS1_BYTES_PER_ROW = 8 + 4 + 32 + 1
EVENTS = ["none", "leave_w1", "leave_w16", "rack32", "join", "churn_1pct", "weighted_bounded"]


def addr(j):
    return "10.4.%d.%d:7000" % (j >> 8, j & 255)


def stats(ms):
    return {"median": round(float(np.median(ms)), 4), "min": round(float(np.min(ms)), 4), "max": round(float(np.max(ms)), 4)}


class Manifest:
    """preallocated manifest buffers of n entries and the raw C call"""

    def __init__(self, s, n):
        self.s, self.L = s, s.L
        self.bufs = [np.empty(n, np.uint64), np.empty(n, np.uint64), np.empty(n, np.uint32), np.empty(n, np.uint32)]
        self.ptrs = [b.ctypes.data_as(C.c_void_p) for b in self.bufs]
        self.n = n

    def __call__(self, dry_run):
        m = C.c_uint64(0)
        self.s._ck(self.L.rio_cuda_set_commit_changes(self.s.s, dry_run, self.n, *self.ptrs, C.byref(m)))
        return m.value


def timed(p, f):
    p.sync()
    t0 = time.perf_counter()
    out = f()
    p.sync()
    return (time.perf_counter() - t0) * 1e3, out


def run_policy(R_, policy, n, trials, w):
    sides = []
    for _ in range(2):
        p = R_.GpuObjectPlacement()
        p.set_solver(policy, 12)
        p.set_nodes([addr(j) for j in range(M)], w)
        s = p.new_set(n)
        s.synth_keys(0, n, 2026)
        s.assign(False)
        s.commit()
        sides.append((p, s))
    (pa, sa), (pb, sb) = sides
    man = Manifest(sa, n)
    assert man(1) == 0
    rng = np.random.default_rng(7)
    j1, j16 = int(np.flatnonzero(w == 1)[0]), int(np.flatnonzero(w == 16)[0])
    rack = list(range(64, 96))
    out = []

    def leave(js):
        for p, s in sides:
            for j in js:
                p.node_set_active(j, False)
            s.rebalance_changes(js, [int(w[j]) for j in js])

    def rejoin(js):
        for p, s in sides:
            for j in js:
                p.node_set_active(j, True)
            s.rebalance_changes(js, [0] * len(js))

    def churn():
        keys = sa.read(want_keys=True)[0]
        gone = rng.choice(keys, n // 100, replace=False)
        new = rng.integers(0, 2**63, n // 100, dtype=np.uint64) * np.uint64(2) + 1
        for _, s in sides:
            s.erase(gone)
            s.insert(new)

    def weighted():
        wt = np.ones(n, np.uint32)
        wt[rng.choice(n, n // 1000, replace=False)] = 100
        for _, s in sides:
            s.write_weights(wt)
            s.assign_bounded_weighted(False, 0, 5, 4, 16)

    def unweighted():
        for _, s in sides:
            s.write_weights(np.ones(n, np.uint32))
            s.assign(False)

    events = {
        "none": (lambda: None, lambda: None),
        "leave_w1": (lambda: leave([j1]), lambda: rejoin([j1])),
        "leave_w16": (lambda: leave([j16]), lambda: rejoin([j16])),
        "rack32": (lambda: leave(rack), lambda: rejoin(rack)),
        "join": (lambda: [s.rebalance_changes([p.node_upsert("10.9.0.1:7000", 8)], [0]) for p, s in sides],
                 lambda: [(p.node_set_active(p.node_index("10.9.0.1:7000"), False), s.rebalance_changes([p.node_index("10.9.0.1:7000")], [8])) for p, s in sides]),
        "churn_1pct": (churn, lambda: None),
        "weighted_bounded": (weighted, unweighted),
    }
    for ev in EVENTS:
        apply, undo = events[ev]
        t_full, t_delta, t_dry, sizes = [], [], [], []
        for t in range(trials + 1):
            apply()
            ms_dry, m_dry = timed(pa, lambda: man(1))
            ms_delta, m = timed(pa, lambda: man(0))
            ms_full, _ = timed(pb, sb.commit)
            assert m == m_dry
            if t:
                t_dry.append(ms_dry)
                t_delta.append(ms_delta)
                t_full.append(ms_full)
                sizes.append(m)
            sample = rng.choice(sa.read(want_keys=True)[0], 200_000)
            assert (pa.lookup_many(sample) == pb.lookup_many(sample)).all(), ev
            assert man(1) == 0, ev
            undo()
            man(0)
            sb.commit()
        n_now = sa.size()
        pt = {"policy": policy, "event": ev, "n": n_now, "manifest": int(np.median(sizes)), "moved_fraction": round(float(np.median(sizes)) / n_now, 6),
              "set_commit_ms": stats(t_full), "commit_changes_ms": stats(t_delta), "dry_run_ms": stats(t_dry),
              "pass1_floor_ms": round(n_now * PASS1_BYTES_PER_ROW / HBM_BPS * 1e3, 4),
              "speedup": round(float(np.median(t_full)) / float(np.median(t_delta)), 2)}
        print(json.dumps(pt), flush=True)
        out.append(pt)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--policies", default="hrw2,hrw")
    ap.add_argument("--out")
    a = ap.parse_args()
    import rio_rs_b200 as R_
    from rio_rs_b200 import build

    build.build()
    res = {"card": card_info(), "n": a.n, "M": M, "points": []}
    print(json.dumps({"card": res["card"]}), flush=True)
    w = np.random.default_rng(2026).integers(1, 17, M).astype(np.uint32)
    for policy in a.policies.split(","):
        res["points"] += run_policy(R_, policy, a.n, a.trials, w)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

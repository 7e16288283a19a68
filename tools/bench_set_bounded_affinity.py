"""Bounded-load affinity sets kept through membership changes (DESIGN.md 3.17): what one change-set call costs and moves next to a
fresh set.assign_bounded_affinity on the post-change table.

Workload: the 3.16 one, a resident set of `--n` objects (default 10 M) with K = 16 features over M = 1024 nodes of weights 1..16,
features U(-1, 1) or clustered (8 centres, spread 0.15), on the tensor cores and on the CUDA cores (RIO_AFFINITY_VARIANT=ffma), caps
5/4 and 11/10, max_rounds 16.  Events, each applied to the state a fresh bounded call left: one leave of a weight-16 node, one of a
weight-1 node, one join of a node new to the set, a rack of 32 leaving, 8 nodes halving their weight, one refeature.  For each:
ms (median of `--trials` windows, min..max; host clock around the call and a device synchronise), passes, objects moved from the
pre-event state, the lower bound (objects that were on REPLACE nodes), the largest c_j / cap_j at the end and the mean fp32 cost of the
final assignment, for the new call and for the fresh call.  Then `--drift` random events in a row (leave / rejoin / reweight /
refeature) on one set kept by the new call next to a twin set assigned afresh after every event, cap 5/4.  The card's name, power limit
and max SM clock are read in the same run.  Writes nothing into the source tree; `--out FILE` also writes the JSON there.
usage: python tools/bench_set_bounded_affinity.py [--n N] [--trials T] [--drift D] [--out FILE]"""
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

from bench_bounded_affinity import card_info, features  # noqa: E402

M, K = 1024, 16
CAPS = [(5, 4), (11, 10)]
ROUNDS = 16
NONE = 0xFFFFFFFF


def addr(j):
    return "10.3.%d.%d:7000" % (j >> 8, j & 255)


class Table:
    """The handle's node table, mirrored: weights, active flags, feature rows."""

    def __init__(self, p, w, fn):
        self.p, self.w, self.fn = p, w.copy(), fn.copy()
        self.active = np.ones(len(w), bool)
        p.set_nodes([addr(j) for j in range(len(w))], w, fn)

    def live(self):
        return self.active & (self.w > 0)

    def prev(self, js):
        return [int(self.w[j]) if self.live()[j] else 0 for j in js]

    def leave(self, js):
        prev = self.prev(js)
        for j in js:
            self.p.node_set_active(int(j), False)
            self.active[j] = False
        return list(js), prev, list(js)

    def join(self, js):
        prev = self.prev(js)
        for j in js:
            self.p.node_upsert(addr(j), int(self.w[j]))
            self.active[j] = True
        return list(js), prev, []

    def join_new(self, rng):
        j = len(self.w)
        f = rng.uniform(-1, 1, K).astype(np.float32)
        self.w = np.append(self.w, np.uint32(8))
        self.fn = np.vstack([self.fn, f[None]])
        self.active = np.append(self.active, True)
        assert self.p.node_upsert(addr(j), 8, f) == j
        return [j], [0], [j]   # a node new to the set is also refeatured: REPLACE | CANDIDATE (it holds no object)

    def reweight(self, js, w):
        prev = self.prev(js)
        for j, x in zip(js, w):
            self.w[j] = x
            self.p.node_upsert(addr(j), int(x))
            self.active[j] = True
        return list(js), prev, []

    def refeature(self, j, f):
        self.fn[j] = f
        self.p.node_upsert(addr(j), int(self.w[j]), f)
        return [], [], [j]


def timed(p, f):
    t0 = time.perf_counter()
    out = f()
    p.sync()
    return (time.perf_counter() - t0) * 1e3, out


class Metrics:
    """max c_j / cap_j and the mean fp32 cost of an assignment, on the GPU (torch)"""

    def __init__(self, fo):
        import torch

        self.torch = torch
        self.fo = torch.from_numpy(fo).cuda()

    def __call__(self, tab, idx, counters, cap):
        from spec_py import capacity

        torch = self.torch
        live = tab.live()
        W = int(tab.w[live].sum())
        n = len(idx)
        caps = np.array([capacity(n, int(tab.w[j]), W, cap[0], cap[1]) if live[j] else 0 for j in range(len(tab.w))], dtype=np.float64)
        c = counters[: len(caps)].astype(np.float64)
        load = float((c[live] / caps[live]).max()) if live.any() else 0.0
        i = torch.from_numpy(idx.astype(np.int64)).cuda()
        ok = i != NONE
        fn = torch.from_numpy(tab.fn).cuda()
        cost = -(self.fo[ok] * fn[i[ok]]).sum(dim=1)
        return load, float(cost.double().mean())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--trials", type=int, default=3)
    ap.add_argument("--drift", type=int, default=32)
    ap.add_argument("--out")
    a = ap.parse_args()

    import rio_rs_b200 as R

    res = {"card": card_info(), "n": a.n, "M": M, "K": K, "max_rounds": ROUNDS, "events": [], "drift": []}
    print(json.dumps({"card": res["card"]}), flush=True)
    for layout in ("uniform", "clustered"):
        fo = features(layout, a.n, np.random.default_rng(4))
        metrics = Metrics(fo)
        for path in ("umma", "ffma"):
            os.environ["RIO_AFFINITY_VARIANT"] = path
            rng = np.random.default_rng(3)
            w0 = rng.integers(1, 17, M).astype(np.uint32)
            fn0 = rng.uniform(-1, 1, (M, K)).astype(np.float32)
            p = R.GpuObjectPlacement(device=0)
            tab = Table(p, w0, fn0)
            s, s2 = p.new_set(a.n), p.new_set(a.n)   # s: kept by the new call; s2: assigned afresh
            for x in (s, s2):
                x.synth_keys(0, a.n, 21)
                x.load_feats(fo)
            heavy, light = int(np.flatnonzero(w0 == 16)[0]), int(np.flatnonzero(w0 == 1)[0])
            for cap in CAPS:
                events = {
                    "leave w=16": lambda: tab.leave([heavy]),
                    "leave w=1": lambda: tab.leave([light]),
                    "join (new node)": lambda: tab.join_new(rng),
                    "rack of 32 leaves": lambda: tab.leave(list(range(64, 96))),
                    "8 nodes halve": lambda: tab.reweight(list(range(200, 208)), [max(1, int(w0[j]) // 2) for j in range(200, 208)]),
                    "refeature": lambda: tab.refeature(300, rng.uniform(-1, 1, K).astype(np.float32)),
                }
                for name, ev in events.items():
                    pt = {"layout": layout, "path": path, "cap": "%d/%d" % cap, "event": name, "ms": [], "fresh_ms": []}
                    for t in range(a.trials + 1):   # window 0 warms up and gives the point's counts
                        # the pre-event state: the original table, a fresh bounded call
                        tab.w[:M], tab.fn[:M] = w0, fn0
                        tab.active[:] = False
                        tab.active[:M] = True
                        p.set_nodes([addr(j) for j in range(M)], w0, fn0)
                        s.assign_bounded_affinity(0, cap[0], cap[1], ROUNDS)
                        pre = s.read()
                        idx, prev, refeat = ev()
                        live = tab.live()
                        ms, (moved, passes) = timed(p, lambda: s.rebalance_changes_bounded_affinity(idx, prev, 0, cap[0], cap[1], ROUNDS))
                        fms, fpasses = timed(p, lambda: s2.assign_bounded_affinity(0, cap[0], cap[1], ROUNDS))
                        if t == 0:
                            got, fresh = s.read(), s2.read()
                            on = pre[pre != NONE].astype(np.int64)
                            bound = int((~live[on]).sum() + np.isin(on, refeat).sum())
                            load, cost = metrics(tab, got, s.counters(), cap)
                            fload, fcost = metrics(tab, fresh, s2.counters(), cap)
                            assert moved == int((got != pre).sum())
                            pt.update(passes=passes, moved=moved, lower_bound=bound, max_load=round(load, 4), mean_cost=round(cost, 5),
                                      fresh_passes=fpasses, fresh_moved=int((fresh != pre).sum()), fresh_max_load=round(fload, 4),
                                      fresh_mean_cost=round(fcost, 5))
                        else:
                            pt["ms"].append(ms)
                            pt["fresh_ms"].append(fms)
                    for key in ("ms", "fresh_ms"):
                        v = sorted(pt.pop(key))
                        pt[key] = {"median": round(v[len(v) // 2], 3), "min": round(v[0], 3), "max": round(v[-1], 3)}
                    res["events"].append(pt)
                    print(json.dumps(pt), flush=True)
            # drift: random events in a row, cap 5/4; s kept by the new call, s2 assigned afresh after each event
            cap = CAPS[0]
            tab.w[:M], tab.fn[:M] = w0, fn0
            tab.active[:] = False
            tab.active[:M] = True
            p.set_nodes([addr(j) for j in range(M)], w0, fn0)
            s.assign_bounded_affinity(0, cap[0], cap[1], ROUNDS)
            s2.assign_bounded_affinity(0, cap[0], cap[1], ROUNDS)
            drng = np.random.default_rng(11)
            prev_s, prev_s2 = s.read(), s2.read()
            for e in range(a.drift):
                kind = drng.integers(0, 4)
                off = [int(j) for j in np.flatnonzero(~tab.active[:M])]
                if kind == 0 or (kind == 1 and not off):
                    ch = tab.leave([int(drng.choice(np.flatnonzero(tab.active[:M])))])
                elif kind == 1:
                    ch = tab.join([int(drng.choice(off))])
                elif kind == 2:
                    j = int(drng.choice(np.flatnonzero(tab.active[:M])))
                    ch = tab.reweight([j], [int(drng.integers(1, 17))])
                else:
                    ch = tab.refeature(int(drng.integers(0, M)), drng.uniform(-1, 1, K).astype(np.float32))
                ms, (moved, passes) = timed(p, lambda: s.rebalance_changes_bounded_affinity(ch[0], ch[1], 0, cap[0], cap[1], ROUNDS))
                fms, fpasses = timed(p, lambda: s2.assign_bounded_affinity(0, cap[0], cap[1], ROUNDS))
                got, fresh = s.read(), s2.read()
                load, cost = metrics(tab, got, s.counters(), cap)
                fload, fcost = metrics(tab, fresh, s2.counters(), cap)
                d = {"layout": layout, "path": path, "event": e, "kind": ["leave", "join", "reweight", "refeature"][kind], "ms": round(ms, 3),
                     "passes": passes, "moved": moved, "max_load": round(load, 4), "mean_cost": round(cost, 5), "fresh_ms": round(fms, 3),
                     "fresh_passes": fpasses, "fresh_moved": int((fresh != prev_s2).sum()), "fresh_max_load": round(fload, 4),
                     "fresh_mean_cost": round(fcost, 5)}
                prev_s, prev_s2 = got, fresh
                res["drift"].append(d)
                print(json.dumps(d), flush=True)
            del s, s2, p
            os.environ.pop("RIO_AFFINITY_VARIANT", None)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

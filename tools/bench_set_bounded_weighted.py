"""Weighted objects in bounded-load placement (DESIGN.md 3.19): how far over its capacity the fullest node's LOAD sits after a plain
set_assign, after the count-based bounded call, and after set_assign_bounded_weighted, with the weighted call's passes, moved objects
and time.

Workload: a resident set of 1 M and 10 M objects over M = 1024 nodes of weights 1..16, cap 5/4, max_rounds 8.  Object weights: all 1,
uniform 1..64, lognormal (sigma = 1.5, scaled so that the total stays near 2^31 and clipped to [1, 2^20]) and 1 % hot at 100x.
Policies: HRW2, flat HRW, and affinity on the tensor cores (K = 16, features U(-1, 1)).  For each case: max over live nodes of
load / cap (cap = ceil(5 L w / (4 W)), L = the weight total) after each of the three calls, the weighted call's passes and the objects
it moved away from the plain assignment, and its ms per call (median of `--trials` windows, min..max; host clock around the call and a
device synchronise).  The card's name, power limit and max SM clock are read in the same run.  Writes nothing into the source tree;
`--out FILE` also writes the JSON there.
usage: python tools/bench_set_bounded_weighted.py [--sizes 1000000,10000000] [--trials T] [--out FILE]"""
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

M, K = 1024, 16
CAP = (5, 4)
ROUNDS = 8
MIXES = ["ones", "uniform", "lognormal", "hot"]
POLICIES = ["hrw2", "hrw", "affinity_tensor"]


def addr(j):
    return "10.5.%d.%d:7000" % (j >> 8, j & 255)


def weights_of(mix, n, rng):
    if mix == "ones":
        return np.ones(n, np.uint32)
    if mix == "uniform":
        return rng.integers(1, 65, n).astype(np.uint32)
    if mix == "lognormal":
        scale = max(1.0, float(2**31) / (n * np.exp(1.5**2 / 2)))
        return np.clip(np.round(np.exp(rng.normal(0.0, 1.5, n)) * scale), 1, 2**20).astype(np.uint32)
    w = np.ones(n, np.uint32)
    w[rng.choice(n, n // 100, replace=False)] = 100
    return w


def timed(p, f):
    p.sync()
    t0 = time.perf_counter()
    out = f()
    p.sync()
    return (time.perf_counter() - t0) * 1e3, out


def max_over(s, cap, live):
    ld = s.loads().astype(np.float64)
    return round(float((ld[live] / cap[live]).max()), 4)


def run(n, trials, rng):
    import rio_rs_b200 as R

    nw = rng.integers(1, 17, M).astype(np.uint32)
    fn = rng.uniform(-1, 1, (M, K)).astype(np.float32)
    fo = rng.uniform(-1, 1, (n, K)).astype(np.float32)
    keys = rng.integers(0, 2**63, n, dtype=np.uint64)
    live = nw > 0
    out = []
    for pol in POLICIES:
        p = R.GpuObjectPlacement()
        p.set_solver("hrw" if pol == "hrw" else "hrw2", 12)
        p.set_nodes([addr(j) for j in range(M)], nw, fn)
        aff = pol.startswith("affinity")
        s = p.new_set(n)
        s.load_keys(keys)
        if aff:
            s.load_feats(fo)
        for mix in MIXES:
            w = weights_of(mix, n, rng)
            s.write_weights(w)
            L = int(w.astype(np.int64).sum())
            cap = np.ceil(CAP[0] * L * nw.astype(np.float64) / (CAP[1] * float(nw.sum())))
            s.assign(aff)
            plain = s.read()
            r_plain = max_over(s, cap, live)
            if aff:
                s.assign_bounded_affinity(0, CAP[0], CAP[1], ROUNDS)
            else:
                s.assign_bounded(0, CAP[0], CAP[1], ROUNDS)
            r_count = max_over(s, cap, live)
            ms, passes = [], 0
            for _ in range(trials + 1):   # the first call warms up the shapes
                t, passes = timed(p, lambda: s.assign_bounded_weighted(aff, 0, CAP[0], CAP[1], ROUNDS))
                ms.append(t)
            ms = ms[1:]
            moved = int((s.read() != plain).sum())
            pt = {"n": n, "policy": pol, "mix": mix, "load_total": L, "max_load_over_cap": {"plain": r_plain, "count_bounded": r_count,
                  "weighted": max_over(s, cap, live)}, "passes": int(passes), "moved": moved,
                  "ms": {"median": round(float(np.median(ms)), 3), "min": round(float(np.min(ms)), 3), "max": round(float(np.max(ms)), 3)}}
            print(json.dumps(pt), flush=True)
            out.append(pt)
        del s, p
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1000000,10000000")
    ap.add_argument("--trials", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this benchmark measures the GPU and has no CPU path")
    res = {"card": card_info()}
    print(json.dumps({"card": res["card"]}), flush=True)
    rng = np.random.default_rng(3119)
    res["cases"] = []
    for n in [int(x) for x in a.sizes.split(",")]:
        res["cases"] += run(n, a.trials, rng)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

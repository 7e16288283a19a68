"""Bounded-load rounds under the affinity cost (DESIGN.md 3.16): how imbalanced plain affinity placement is, and what the spill rounds
cost next to it.

Workload: a resident set of `--n` objects (default 10 M) with K = 16 features over M = 1024 nodes of weights 1..16, features U(-1, 1)
or clustered (objects drawn around 8 centres with spread 0.15, the nodes U(-1, 1)), on the tensor cores (the default) and on the
CUDA cores (RIO_AFFINITY_VARIANT=ffma), at caps 5/4 and 11/10 and max_rounds 4 and 16.  For every point: ms per
set.assign_bounded_affinity next to ms per plain set.assign(use_affinity = 1), each a host clock around the call and a device
synchronise, warmed up once and timed over `--trials` windows taken round-robin (median, min..max); the passes run; the objects moved
from their pass-0 node; the largest c_j / cap_j after pass 0 and at the end.  The card's name, power limit and max SM clock are read in
the same run.  Writes nothing into the source tree; `--out FILE` also writes the JSON there.
usage: python tools/bench_bounded_affinity.py [--n N] [--trials T] [--out FILE]"""
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

M, K = 1024, 16
CAPS = [(5, 4), (11, 10)]
ROUNDS = [4, 16]


def card_info():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clk}
    except Exception as e:  # noqa: BLE001
        return {"error": repr(e)}


def features(layout, n, rng):
    if layout == "uniform":
        return rng.uniform(-1, 1, (n, K)).astype(np.float32)
    centres = rng.uniform(-1, 1, (8, K)).astype(np.float32)
    return (centres[rng.integers(0, 8, n)] + rng.normal(0, 0.15, (n, K))).astype(np.float32)


def timed(p, f):
    t0 = time.perf_counter()
    out = f()
    p.sync()
    return (time.perf_counter() - t0) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()

    import rio_rs_b200 as R
    from spec_py import capacity

    res = {"card": card_info(), "n": a.n, "M": M, "K": K, "points": []}
    rng = np.random.default_rng(3)
    fn = rng.uniform(-1, 1, (M, K)).astype(np.float32)
    w = rng.integers(1, 17, M).astype(np.uint32)
    W = int(w.sum())
    p = R.GpuObjectPlacement(device=0)
    p.set_nodes(["10.2.%d.%d:7000" % (j >> 8, j & 255) for j in range(M)], w, fn)
    s = p.new_set(a.n)
    s.synth_keys(0, a.n, 21)
    for layout in ("uniform", "clustered"):
        s.load_feats(features(layout, a.n, np.random.default_rng(4)))
        for path in ("umma", "ffma"):
            os.environ["RIO_AFFINITY_VARIANT"] = path
            s.assign(True)
            pass0, c0 = s.read(), s.counters().astype(np.int64)
            points = []
            for cap in CAPS:
                caps = np.array([capacity(a.n, int(x), W, cap[0], cap[1]) for x in w], dtype=np.int64)
                for rounds in ROUNDS:
                    passes = s.assign_bounded_affinity(0, cap[0], cap[1], rounds)   # warm-up, and the point's results
                    idx, c = s.read(), s.counters().astype(np.int64)
                    points.append({"layout": layout, "path": path, "cap": "%d/%d" % cap, "max_rounds": rounds, "passes": passes,
                                   "moved": int((idx != pass0).sum()), "max_load_pass0": float((c0 / caps).max()),
                                   "max_load_end": float((c / caps).max()), "ms": [], "plain_ms": []})
            timed(p, lambda: s.assign(True))
            for _ in range(a.trials):
                for pt in points:
                    cap = [int(x) for x in pt["cap"].split("/")]
                    pt["ms"].append(timed(p, lambda: s.assign_bounded_affinity(0, cap[0], cap[1], pt["max_rounds"]))[0])
                    pt["plain_ms"].append(timed(p, lambda: s.assign(True))[0])
            for pt in points:
                for key in ("ms", "plain_ms"):
                    v = sorted(pt.pop(key))
                    pt[key] = {"median": round(v[len(v) // 2], 3), "min": round(v[0], 3), "max": round(v[-1], 3)}
                res["points"].append(pt)
                print(json.dumps(pt), flush=True)
            os.environ.pop("RIO_AFFINITY_VARIANT", None)
    print(json.dumps({"card": res["card"]}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

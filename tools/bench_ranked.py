"""Kernel-call timing of the ranked placement lists (DESIGN.md 3.9) against the single assignment, both policies.

Workload: 10 M device-resident keys x 1024 weighted nodes (the C4 shape).  Timed with CUDA events on the engine stream:
rio_cuda_assign_batch_dev and rio_cuda_assign_ranked_batch_dev at R = 1, 2, 4 on the same keys, `--launches` calls per window after
a warm-up, `--trials` windows per point taken round-robin over the points; the median and the spread (min..max) of the per-call
time of those windows are reported with the ratio to the single assignment.  The card's name, power limit and max SM clock are
read in the same run.  Before timing, 200 k objects of every ranked output are checked against the CPU oracle
(tests/ranked_oracle.c).  Writes nothing into the source tree; `--out FILE` also writes the JSON there.
usage: python tools/bench_ranked.py [--n N] [--nodes M] [--launches K] [--trials T] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card_info():
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [s.strip() for s in q.split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clk}
    except Exception as e:  # noqa: BLE001
        return {"error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--nodes", type=int, default=1024)
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--trials", type=int, default=7)
    ap.add_argument("--check", type=int, default=200_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import rio_rs_b200 as R
    from rio_rs_b200 import build
    from oracle import pyoracle as O
    import ranked_oracle as RO

    build.build()
    O.build()
    p = R.GpuObjectPlacement(device=0)
    L, h = p.L, p.h
    addrs, seeds, w = O.synth_nodes(a.nodes)
    p.set_nodes(addrs, w)
    n, ranks_list = a.n, (1, 2, 4)
    keys = O.synth_keys(n, 1)
    dk, di = C.c_void_p(), C.c_void_p()
    p._ck(L.rio_cuda_dev_alloc(h, n * 8, C.byref(dk)))
    p._ck(L.rio_cuda_dev_alloc(h, n * max(ranks_list) * 4, C.byref(di)))
    p._ck(L.rio_cuda_memcpy_h2d(h, dk, keys.ctypes.data_as(C.c_void_p), n * 8))
    p.sync()
    m = min(a.check, n)

    def call(r):
        if r == 0:
            p._ck(L.rio_cuda_assign_batch_dev(h, dk, None, n, di))
        else:
            p._ck(L.rio_cuda_assign_ranked_batch_dev(h, dk, n, r, di))

    results = {}
    for policy in ("hrw2", "hrw"):
        p.set_solver(policy, 12)
        launches = a.launches if policy == "hrw2" else max(2, a.launches // 10)
        # correctness: the first m objects of every ranked output against the oracle, and rank 1 against assign_batch
        call(0)
        one = np.empty(m, dtype=np.uint32)
        p._ck(L.rio_cuda_memcpy_d2h(h, one.ctypes.data_as(C.c_void_p), di, m * 4))
        p.sync()
        checks = {}
        for r in ranks_list:
            call(r)
            got = np.empty((m, r), dtype=np.uint32)
            p._ck(L.rio_cuda_memcpy_d2h(h, got.ctypes.data_as(C.c_void_p), di, m * r * 4))
            p.sync()
            want = RO.assign_ranked(policy, keys[:m], seeds, w, r, threads=os.cpu_count() or 8)
            checks["R%d" % r] = bool((got == want).all() and (got[:, 0] == one).all())
        # timing: every point warmed up, then `trials` windows per point, round-robin
        points = [0] + list(ranks_list)
        for r in points:
            for _ in range(3):
                call(r)
        p.sync()
        per_call = {r: [] for r in points}
        for _ in range(a.trials):
            for r in points:
                p.event_record(0)
                for _ in range(launches):
                    call(r)
                p.event_record(1)
                p.sync()
                per_call[r].append(p.event_elapsed_ms(0, 1) * 1e3 / launches)
        base = float(np.median(per_call[0]))
        res = {"checks_200k_vs_oracle": checks, "launches_per_window": launches}
        for r in points:
            v = np.array(per_call[r])
            name = "assign_batch_dev" if r == 0 else "assign_ranked_batch_dev_R%d" % r
            res[name] = {"us_median": round(float(np.median(v)), 1), "us_min": round(float(v.min()), 1), "us_max": round(float(v.max()), 1),
                         "ratio_to_assign": round(float(np.median(v)) / base, 2)}
        results[policy] = res
    p._ck(L.rio_cuda_dev_free(h, dk))
    p._ck(L.rio_cuda_dev_free(h, di))
    out = {"n": n, "nodes": a.nodes, "weights": "1..16", "trials": a.trials, "card": card_info(), "device": p.device_info(), "results": results}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")
    ok = all(all(r["checks_200k_vs_oracle"].values()) for r in results.values())
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()

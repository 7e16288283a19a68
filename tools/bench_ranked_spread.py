"""Kernel-call timing of the failure-domain ranked lists (DESIGN.md 3.12) beside the ranked lists (3.9), both policies.

Workload: 10 M device-resident keys x 1024 nodes with weights 1..16 (the C4 shape) under three label layouts: none, 32 racks of 32
and 4 zones of 256 contiguous node indices, one handle per layout.  Timed with CUDA events on each handle's stream:
rio_cuda_assign_ranked_spread_batch_dev at R = 1, 2, 4, 8 under every layout, beside rio_cuda_assign_ranked_batch_dev at the same R,
`--launches` calls per window after a warm-up, `--trials` windows per point taken round-robin over the points; the median and the
spread (min..max) of the per-call time of those windows are reported with the ratio to the ranked call.  The card's name, power limit
and max SM clock are read in the same run.  Before timing, the first 200 k lists of every output are checked against the CPU oracle
(tests/spread_oracle.c).  Writes nothing into the source tree; `--out FILE` also writes the JSON there.
usage: python tools/bench_ranked_spread.py [--n N] [--nodes M] [--launches K] [--trials T] [--out FILE]"""
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

RANKS = (1, 2, 4, 8)


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
    import spread_oracle as SO

    build.build()
    O.build()
    M, n, m = a.nodes, a.n, min(a.check, a.n)
    addrs, seeds, w = O.synth_nodes(M)
    keys = O.synth_keys(n, 1)
    j = np.arange(M, dtype=np.uint32)
    layouts = {"none": np.full(M, 0xFFFFFFFF, dtype=np.uint32), "racks_32x32": j // 32, "zones_4x256": j // 256}
    hs = {}
    for name, dom in layouts.items():   # one handle per layout: a label change never falls inside a timed window
        p = R.GpuObjectPlacement(device=0)
        p.set_nodes(addrs, w)
        if name != "none":
            p.set_node_domains(j, dom)
        dk, di = C.c_void_p(), C.c_void_p()
        p._ck(p.L.rio_cuda_dev_alloc(p.h, n * 8, C.byref(dk)))
        p._ck(p.L.rio_cuda_dev_alloc(p.h, n * max(RANKS) * 4, C.byref(di)))
        p._ck(p.L.rio_cuda_memcpy_h2d(p.h, dk, keys.ctypes.data_as(C.c_void_p), n * 8))
        p.sync()
        hs[name] = (p, dk, di)

    def call(point):
        name, r = point
        p, dk, di = hs["none" if name == "ranked" else name]
        fn = p.L.rio_cuda_assign_ranked_batch_dev if name == "ranked" else p.L.rio_cuda_assign_ranked_spread_batch_dev
        p._ck(fn(p.h, dk, n, r, di))
        return p

    results = {}
    for policy in ("hrw2", "hrw"):
        for p, _, _ in hs.values():
            p.set_solver(policy, 12)
        launches = a.launches if policy == "hrw2" else max(2, a.launches // 10)
        checks = {}
        for name, dom in layouts.items():
            want = SO.assign_spread(policy, keys[:m], seeds, w, dom, max(RANKS), threads=os.cpu_count() or 8)
            for r in RANKS:
                p, _, di = hs[name]
                call((name, r))
                got = np.empty((m, r), dtype=np.uint32)
                p._ck(p.L.rio_cuda_memcpy_d2h(p.h, got.ctypes.data_as(C.c_void_p), di, m * r * 4))
                p.sync()
                checks["%s_R%d" % (name, r)] = bool((got == want[:, :r]).all())
        points = [(name, r) for r in RANKS for name in ["ranked"] + list(layouts)]
        for pt in points:
            for _ in range(3):
                call(pt)
        for p, _, _ in hs.values():
            p.sync()
        per_call = {pt: [] for pt in points}
        for _ in range(a.trials):
            for pt in points:
                p = hs["none" if pt[0] == "ranked" else pt[0]][0]
                p.event_record(0)
                for _ in range(launches):
                    call(pt)
                p.event_record(1)
                p.sync()
                per_call[pt].append(p.event_elapsed_ms(0, 1) * 1e3 / launches)
        res = {"checks_200k_vs_oracle": checks, "launches_per_window": launches}
        for pt in points:
            v = np.array(per_call[pt])
            base = float(np.median(per_call[("ranked", pt[1])]))
            key = ("assign_ranked_batch_dev" if pt[0] == "ranked" else "spread_" + pt[0]) + "_R%d" % pt[1]
            res[key] = {"us_median": round(float(np.median(v)), 1), "us_min": round(float(v.min()), 1), "us_max": round(float(v.max()), 1),
                        "ratio_to_ranked": round(float(np.median(v)) / base, 2)}
        results[policy] = res
    for p, dk, di in hs.values():
        p._ck(p.L.rio_cuda_dev_free(p.h, dk))
        p._ck(p.L.rio_cuda_dev_free(p.h, di))
    out = {"n": n, "nodes": M, "weights": "1..16", "trials": a.trials, "card": card_info(), "device": hs["none"][0].device_info(),
           "results": results}
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

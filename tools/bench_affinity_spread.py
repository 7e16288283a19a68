"""Kernel-call timing of the failure-domain affinity lists (DESIGN.md 3.14) against the ranked affinity lists (3.9), on both paths.

Workload: 10 M device-resident objects x 1024 nodes x K = 16, features U(-1, 1) from seeds 11 (objects) and 13 (nodes), as in
tools/bench_affinity_ranked.py.  Three label layouts: "none" (no labels: every node a domain of its own), "racks" (32 racks of 32
consecutive nodes) and "zones" (4 zones of 256, nodes dealt round robin).  Timed with CUDA events on the engine stream:
rio_cuda_assign_ranked_affinity_spread_batch_dev under every layout and rio_cuda_assign_ranked_affinity_batch_dev (which ignores
labels), at R = 1, 2, 4, 8, on the tensor-core path and on the CUDA-core path (RIO_AFFINITY_VARIANT=ffma), `--launches` calls per
window after a warm-up, `--trials` windows per point taken round-robin over the points.  The median and the spread (min..max) of the
per-call time are reported with the ratio to the ranked call at the same R and path.  The card's name, power limit and max SM clock
are read in the same run.  Before timing, the first `--check` lists of every output are checked with the conditioned fp64 rule of
tests/affinity_spread_oracle.py, and rank 1 against assign_batch.  Writes nothing into the source tree; `--out FILE` also writes the
JSON there.
usage: python tools/bench_affinity_spread.py [--n N] [--nodes M] [--launches K] [--trials T] [--check C] [--out FILE]"""
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


def layouts(M):
    j = np.arange(M, dtype=np.uint32)
    return {"none": np.full(M, 0xFFFFFFFF, np.uint32), "racks": j // max(1, M // 32), "zones": j % 4}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--nodes", type=int, default=1024)
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--check", type=int, default=200_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import rio_rs_b200 as R
    from rio_rs_b200 import build
    from oracle import pyoracle as O
    import affinity_spread_oracle as SO

    build.build()
    O.build()
    n, M, K, ranks_list = a.n, a.nodes, 16, (1, 2, 4, 8)
    fo = np.random.default_rng(11).uniform(-1, 1, (n, K)).astype(np.float32)
    fn = np.random.default_rng(13).uniform(-1, 1, (M, K)).astype(np.float32)
    p = R.GpuObjectPlacement(device=0)
    L, h = p.L, p.h
    addrs, _, _ = O.synth_nodes(M)
    p.set_nodes(addrs, None, fn)
    all_idx = np.arange(M, dtype=np.uint32)
    df, di = C.c_void_p(), C.c_void_p()
    p._ck(L.rio_cuda_dev_alloc(h, n * K * 4, C.byref(df)))
    p._ck(L.rio_cuda_dev_alloc(h, n * max(ranks_list) * 4, C.byref(di)))
    p._ck(L.rio_cuda_memcpy_h2d(h, df, fo.ctypes.data_as(C.c_void_p), n * K * 4))
    p.sync()
    m = min(a.check, n)
    lays = layouts(M)

    def call(kind, r):
        if kind == "assign":
            p._ck(L.rio_cuda_assign_batch_dev(h, None, df, n, di))
        elif kind == "ranked":
            p._ck(L.rio_cuda_assign_ranked_affinity_batch_dev(h, df, n, r, di))
        else:
            p._ck(L.rio_cuda_assign_ranked_affinity_spread_batch_dev(h, df, n, r, di))

    results = {}
    for path, var in (("tensor", "umma"), ("cuda_core", "ffma")):
        os.environ["RIO_AFFINITY_VARIANT"] = var
        launches = a.launches if path == "tensor" else max(2, a.launches // 5)
        call("assign", 0)
        one = np.empty(m, dtype=np.uint32)
        p._ck(L.rio_cuda_memcpy_d2h(h, one.ctypes.data_as(C.c_void_p), di, m * 4))
        p.sync()
        checks = {}
        for lay in lays:
            p.set_node_domains(all_idx, lays[lay])
            for r in ranks_list:
                call("spread", r)
                got = np.empty((m, r), dtype=np.uint32)
                p._ck(L.rio_cuda_memcpy_d2h(h, got.ctypes.data_as(C.c_void_p), di, m * r * 4))
                p.sync()
                try:
                    near_ties = SO.check(got, fo[:m], fn, np.ones(M, bool), lays[lay])
                    checks["%s_R%d" % (lay, r)] = {"ok": bool((got[:, 0] == one).all()), "index_differs_at_near_ties": near_ties}
                except AssertionError as e:
                    checks["%s_R%d" % (lay, r)] = {"ok": False, "error": str(e)[:300]}
        # timing: one layout at a time (the first call after a relabel uploads the domain ids), every point warmed up, then
        # `trials` windows per point, round-robin over the ranked call and the spread call at each R
        per_call = {}
        for lay in lays:
            p.set_node_domains(all_idx, lays[lay])
            points = [(k, r) for r in ranks_list for k in ("ranked", lay)]
            for k, r in points:
                for _ in range(2):
                    call(k, r)
            p.sync()
            for pt in points:
                per_call.setdefault(pt, [])
            for _ in range(a.trials):
                for k, r in points:
                    p.event_record(0)
                    for _ in range(launches):
                        call(k, r)
                    p.event_record(1)
                    p.sync()
                    per_call[(k, r)].append(p.event_elapsed_ms(0, 1) / launches)
        res = {"checks_vs_fp64_oracle": checks, "objects_checked": m, "launches_per_window": launches}
        for (k, r), v in per_call.items():
            v = np.array(v)
            base = float(np.median(per_call[("ranked", r)]))
            res["%s_R%d" % (k, r)] = {"ms_median": round(float(np.median(v)), 3), "ms_min": round(float(v.min()), 3), "ms_max": round(float(v.max()), 3),
                                      "ratio_to_ranked": round(float(np.median(v)) / base, 2)}
        results[path] = res
    os.environ.pop("RIO_AFFINITY_VARIANT", None)
    p._ck(L.rio_cuda_dev_free(h, df))
    p._ck(L.rio_cuda_dev_free(h, di))
    out = {"n": n, "nodes": M, "K": K, "trials": a.trials, "card": card_info(), "device": p.device_info(), "results": results}
    s = json.dumps(out, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s + "\n")
    ok = all(c["ok"] for r in results.values() for c in r["checks_vs_fp64_oracle"].values())
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()

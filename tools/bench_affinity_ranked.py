"""Kernel-call timing of the ranked affinity lists (DESIGN.md 3.9) against the single affinity assignment, on both paths.

Workload: 10 M device-resident objects x 1024 nodes x K = 16, features U(-1, 1) from seeds 11 (objects) and 13 (nodes) as in
SURVEY 8d.  Timed with CUDA events on the engine stream: rio_cuda_assign_batch_dev(obj_feats) and
rio_cuda_assign_ranked_affinity_batch_dev at R = 1, 2, 4, 8, on the tensor-core path and on the CUDA-core path
(RIO_AFFINITY_VARIANT=ffma), `--launches` calls per window after a warm-up, `--trials` windows per point taken round-robin over the
points.  The median and the spread (min..max) of the per-call time are reported with the ratio to the single assignment of the same
path.  On the tensor path the two passes (k_affinity_wgmma_ranked, k_affinity_resolve_ranked) are also timed apart with
torch.profiler in a separate run.  The card's name, power limit and max SM clock are read in the same run.  Before timing, the first
`--check` lists of every output are checked against the fp64 oracle (tests/affinity_ranked_oracle.py).  Writes nothing into the
source tree; `--out FILE` also writes the JSON there.
usage: python tools/bench_affinity_ranked.py [--n N] [--nodes M] [--launches K] [--trials T] [--check C] [--out FILE]"""
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
    ap.add_argument("--launches", type=int, default=10)
    ap.add_argument("--trials", type=int, default=7)
    ap.add_argument("--check", type=int, default=200_000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import rio_rs_b200 as R
    from rio_rs_b200 import build
    from oracle import pyoracle as O
    import affinity_ranked_oracle as AO

    build.build()
    O.build()
    n, M, K, ranks_list = a.n, a.nodes, 16, (1, 2, 4, 8)
    fo = np.random.default_rng(11).uniform(-1, 1, (n, K)).astype(np.float32)
    fn = np.random.default_rng(13).uniform(-1, 1, (M, K)).astype(np.float32)
    p = R.GpuObjectPlacement(device=0)
    L, h = p.L, p.h
    addrs, _, _ = O.synth_nodes(M)
    p.set_nodes(addrs, None, fn)
    df, di = C.c_void_p(), C.c_void_p()
    p._ck(L.rio_cuda_dev_alloc(h, n * K * 4, C.byref(df)))
    p._ck(L.rio_cuda_dev_alloc(h, n * max(ranks_list) * 4, C.byref(di)))
    p._ck(L.rio_cuda_memcpy_h2d(h, df, fo.ctypes.data_as(C.c_void_p), n * K * 4))
    p.sync()
    m = min(a.check, n)
    want = AO.ranked(fo[:m], fn, np.ones(M, bool), max(ranks_list) + 1)

    def call(r):
        if r == 0:
            p._ck(L.rio_cuda_assign_batch_dev(h, None, df, n, di))
        else:
            p._ck(L.rio_cuda_assign_ranked_affinity_batch_dev(h, df, n, r, di))

    results = {}
    for path, var in (("tensor", "umma"), ("cuda_core", "ffma")):
        os.environ["RIO_AFFINITY_VARIANT"] = var
        launches = a.launches if path == "tensor" else max(2, a.launches // 5)
        # correctness: the first m lists of every output against the fp64 oracle, and rank 1 against assign_batch
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
            try:
                near_ties = AO.check(got, fo[:m], fn, np.ones(M, bool), want)
                checks["R%d" % r] = {"ok": bool((got[:, 0] == one).all()), "index_differs_at_near_ties": near_ties}
            except AssertionError as e:
                checks["R%d" % r] = {"ok": False, "error": str(e)[:300]}
        # timing: every point warmed up, then `trials` windows per point, round-robin
        points = [0] + list(ranks_list)
        for r in points:
            for _ in range(2):
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
                per_call[r].append(p.event_elapsed_ms(0, 1) / launches)
        base = float(np.median(per_call[0]))
        res = {"checks_vs_fp64_oracle": checks, "objects_checked": m, "launches_per_window": launches}
        for r in points:
            v = np.array(per_call[r])
            name = "assign_batch_dev" if r == 0 else "ranked_R%d" % r
            res[name] = {"ms_median": round(float(np.median(v)), 3), "ms_min": round(float(v.min()), 3), "ms_max": round(float(v.max()), 3),
                         "ratio_to_assign": round(float(np.median(v)) / base, 2)}
        results[path] = res
    # the two passes of the tensor path apart: kernel times from torch.profiler, in a run of their own after the timed windows
    os.environ["RIO_AFFINITY_VARIANT"] = "umma"
    passes = {}
    try:
        import torch
        from torch.profiler import ProfilerActivity, profile

        torch.cuda.init()
        for r in (0,) + ranks_list:
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    call(r)
                p.sync()
            ks = {}
            for e in prof.events():
                if e.device_type.name == "CUDA" and "k_affinity" in e.name:
                    key = "wgmma" if "wgmma" in e.name else "resolve"
                    ks.setdefault(key, []).append(e.device_time_total / 1e3)
            passes["assign_batch_dev" if r == 0 else "ranked_R%d" % r] = {k: round(float(np.median(v)), 3) for k, v in ks.items()}
    except Exception as e:  # noqa: BLE001
        passes = {"error": repr(e)[:300]}
    os.environ.pop("RIO_AFFINITY_VARIANT", None)
    p._ck(L.rio_cuda_dev_free(h, df))
    p._ck(L.rio_cuda_dev_free(h, di))
    out = {"n": n, "nodes": M, "K": K, "trials": a.trials, "card": card_info(), "device": p.device_info(), "results": results,
           "tensor_path_passes_ms": passes}
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

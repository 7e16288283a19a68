"""Object churn in resident sets (DESIGN.md 3.18): what set_erase and set_insert cost next to what a caller does without them, a
set_load_keys (+ set_load_feats) of the new population and the kind's full assign.

Workload: a resident set of `--n` objects (default 10 M) over M = 1024 nodes of weights 1..16; the affinity kinds carry K = 16
features U(-1, 1).  Kinds: plain HRW2, ranked hash R = 4 under HRW2 and under flat HRW, ranked affinity R = 4 on the tensor cores
and on the CUDA cores (RIO_AFFINITY_VARIANT=ffma at the assign), and bounded affinity (cap 5/4, max_rounds 16; each of its churn
steps is followed by the k = 0 change-set call that brings it back within capacity).  Churn: erase 1 % and 0.1 % of the set's keys,
either random keys or every object of whole nodes (nodes taken in index order until the fraction is reached), then insert as many
new keys; the set is back at n rows after each step.  For each: ms per call (median of `--trials` windows, min..max; host clock
around the call and a device synchronise), and for erase the algorithmic bytes (8 B of key per row, 4 B of idx per erased row, and
each moved row read and written: key, idx, list row, feature row) with the time they take at 3.35 TB/s.  The baseline is timed the
same way on a second set.  The card's name, power limit and max SM clock are read in the same run.  Writes nothing into the source
tree; `--out FILE` also writes the JSON there.
usage: python tools/bench_set_churn.py [--n N] [--trials T] [--out FILE]"""
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

M, K, R = 1024, 16, 4
HBM_BPS = 3.35e12
KINDS = ["plain_hrw2", "ranked_hrw2", "ranked_hrw", "ranked_affinity_tensor", "ranked_affinity_cuda", "bounded_affinity"]


def addr(j):
    return "10.4.%d.%d:7000" % (j >> 8, j & 255)


class variant:
    def __init__(self, v):
        self.v = v

    def __enter__(self):
        os.environ["RIO_AFFINITY_VARIANT"] = self.v

    def __exit__(self, *a):
        os.environ.pop("RIO_AFFINITY_VARIANT", None)


def timed(p, f):
    p.sync()
    t0 = time.perf_counter()
    out = f()
    p.sync()
    return (time.perf_counter() - t0) * 1e3, out


def stats(ms):
    return {"median": round(float(np.median(ms)), 4), "min": round(float(np.min(ms)), 4), "max": round(float(np.max(ms)), 4)}


def assign(s, kind):
    """the kind's full assign of the set as loaded"""
    with variant("ffma" if kind == "ranked_affinity_cuda" else "umma"):
        if kind == "plain_hrw2":
            s.assign(False)
        elif kind.startswith("ranked_affinity"):
            s.assign_ranked_affinity(R)
        elif kind.startswith("ranked"):
            s.assign_ranked(R)
        else:
            s.assign_bounded_affinity(0, 5, 4, 16)


def run_kind(R_, kind, n, trials, rng, w, fn):
    p = R_.GpuObjectPlacement()
    p.set_solver("hrw2" if kind in ("plain_hrw2", "ranked_hrw2") else "hrw", 12)
    affinity = "affinity" in kind
    p.set_nodes([addr(j) for j in range(M)], w, fn if affinity else None)
    s = p.new_set(n)
    keys = rng.integers(0, 2**63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)
    fo = rng.uniform(-1, 1, (n, K)).astype(np.float32) if affinity else None
    s.load_keys(keys)
    if affinity:
        s.load_feats(fo)
    assign(s, kind)
    ranks = R if kind.startswith("ranked") else 0
    row_bytes = 8 + 4 + 4 * ranks + (4 * K if affinity else 0)
    out = []
    for frac in (0.01, 0.001):
        for pattern in ("random", "nodes"):
            m_target = int(n * frac)
            t_erase, t_insert, t_k0, bytes_erase, erased_n, moved_n = [], [], [], [], [], []
            for _ in range(trials):
                cur_keys, idx = s.read(want_keys=True)
                if pattern == "random":
                    gone = rng.choice(cur_keys, size=m_target, replace=False)
                else:
                    order = np.argsort(idx, kind="stable")
                    cnt = np.bincount(idx[idx < M].astype(np.int64), minlength=M)
                    upto = int(np.searchsorted(np.cumsum(cnt), m_target)) + 1
                    gone = cur_keys[order[: int(cnt[:upto].sum())]]
                n_before = len(cur_keys)
                n_new = n_before - len(gone)
                flag = np.isin(cur_keys, gone)
                moved = int((~flag[n_new:]).sum())
                new_keys = rng.integers(0, 2**63, len(gone), dtype=np.uint64) * np.uint64(2) + 1
                new_feats = rng.uniform(-1, 1, (len(gone), K)).astype(np.float32) if affinity else None
                ms, erased = timed(p, lambda: s.erase(gone))
                assert erased == len(gone)
                t_erase.append(ms)
                bytes_erase.append(8 * n_before + 4 * erased + 2 * row_bytes * moved)
                erased_n.append(erased)
                moved_n.append(moved)
                ms, _ = timed(p, lambda: s.insert(new_keys, new_feats))
                t_insert.append(ms)
                if kind == "bounded_affinity":
                    ms, _ = timed(p, lambda: s.rebalance_changes_bounded_affinity([], [], 0, 5, 4, 16))
                    t_k0.append(ms)
            b = float(np.median(bytes_erase))
            pt = {"kind": kind, "fraction": frac, "pattern": pattern, "erased": int(np.median(erased_n)), "moved_rows": int(np.median(moved_n)),
                  "erase_ms": stats(t_erase), "insert_ms": stats(t_insert), "erase_bytes": int(b), "erase_floor_ms": round(b / HBM_BPS * 1e3, 4)}
            if t_k0:
                pt["k0_ms"] = stats(t_k0)
            print(json.dumps(pt), flush=True)
            out.append(pt)
    # the baseline: the new population loaded and assigned from scratch, on a second set
    cur_keys, _ = s.read(want_keys=True)
    t = p.new_set(n)
    base = []
    for _ in range(trials):
        def reload():
            t.load_keys(cur_keys)
            if affinity:
                t.load_feats(fo)
            assign(t, kind)
        base.append(timed(p, reload)[0])
    b = {"kind": kind, "baseline_reload_assign_ms": stats(base)}
    print(json.dumps(b), flush=True)
    out.append(b)
    del s, t
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--trials", type=int, default=5)
    ap.add_argument("--kinds", default=",".join(KINDS))
    ap.add_argument("--out")
    a = ap.parse_args()
    import rio_rs_b200 as R_
    from rio_rs_b200 import build

    build.build()
    res = {"card": card_info(), "n": a.n, "M": M, "K": K, "R": R, "points": []}
    print(json.dumps({"card": res["card"]}), flush=True)
    rng = np.random.default_rng(2026)
    w = rng.integers(1, 17, M).astype(np.uint32)
    fn = rng.uniform(-1, 1, (M, K)).astype(np.float32)
    for kind in a.kinds.split(","):
        res["points"] += run_kind(R_, kind, a.n, a.trials, rng, w, fn)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()

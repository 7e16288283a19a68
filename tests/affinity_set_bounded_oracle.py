"""A bounded-load affinity set kept through a change set (DESIGN.md 3.17), restated from the document (test infrastructure): pass 0
re-places the S1 objects over the live set and moves every other object to the first node of {its node} u CANDIDATES in (c32, j)
order; then the round loop of 3.5 / 3.16 runs from the counters that leaves, closed set empty, rounds numbered from 1.

`argmin(rows, mask)` places the objects `rows` over the nodes `mask` allows, as in tests/affinity_bounded_oracle.py: the exact c32
minimum, or an argmin built from the engine itself.  The S2 merge always uses c32 (tests/affinity_c32_ref.py): on both kernel paths
the pass costs a row against its node and the candidates with the shared fmaf order.

`replace` is the REPLACE flag of every interned node (not live, or live and refeatured since the last call); `cand` the CANDIDATES
(joined or refeatured live nodes).  `live` and `active` as in affinity_bounded_oracle.py.  The counts are of the global key set."""
import numpy as np

import affinity_c32_ref as C32
from affinity_bounded_oracle import NONE, counts, spill_hash
from spec_py import capacity


def rebalance(keys, idx, fo, fn, argmin, replace, cand, weights, live, active=None, n_total=0, num=5, den=4, max_rounds=4):
    """-> dict: idx, counters, passes, moved (objects whose node differs from `idx`), s1 (objects re-placed by pass 0), beaten (S2
    objects a candidate took), spilled (objects spilled in some round), over (nodes over capacity in some round), stop ('rounds',
    'balanced' or 'closed')."""
    keys = np.asarray(keys, dtype=np.uint64)
    prev = np.asarray(idx, dtype=np.uint32)
    weights = np.asarray(weights, dtype=np.uint64)
    live = np.asarray(live, bool)
    active = live if active is None else np.asarray(active, bool)
    replace = np.asarray(replace, bool)
    cand = [int(j) for j in cand]
    n, M = len(keys), len(weights)
    # pass 0
    out = prev.copy()
    interned = prev < M
    s1 = ~interned
    s1[interned] = replace[prev[interned]]
    beaten = np.zeros(n, bool)
    rows = np.flatnonzero(~s1)
    if cand and len(rows):
        c = C32.c32(fo[rows], fn)
        y = prev[rows].astype(np.int64)
        bc, bj = c[np.arange(len(rows)), y], y.copy()
        for j in cand:
            cj = c[:, j]
            take = (cj < bc) | ((cj == bc) & (j < bj))
            bc, bj = np.where(take, cj, bc), np.where(take, j, bj)
        out[rows] = bj.astype(np.uint32)
        beaten[rows] = bj != y
    sel = np.flatnonzero(s1)
    if len(sel):
        out[sel] = argmin(sel, live)
    # the rounds of 3.5 from here
    N = n_total or n
    W = int(weights[live].sum())
    cap = np.array([capacity(N, int(weights[j]), W, num, den) if live[j] else 0 for j in range(M)], dtype=np.int64)
    closed = np.zeros(M, bool)
    spilled = np.zeros(n, bool)
    passes, stop = 1, "rounds"
    for r in range(1, max_rounds):
        cnt = counts(out, M).astype(np.int64)
        over = active & (cnt > cap)
        closed |= over
        if not over.any():
            stop = "balanced"
            break
        if not (active & ~closed).any():
            stop = "closed"
            break
        thr = np.zeros(M, dtype=np.uint64)
        thr[over] = [((int(cnt[j]) - int(cap[j])) << 32) // int(cnt[j]) for j in np.flatnonzero(over)]
        placed = out != NONE
        on_over = np.zeros(n, bool)
        on_over[placed] = over[out[placed]]
        spill = on_over & (spill_hash(keys, r) < thr[np.where(placed, out, 0)])
        rows = np.flatnonzero(spill)
        if len(rows):
            out[rows] = argmin(rows, live & ~closed)
        spilled |= spill
        passes += 1
    return dict(idx=out, counters=counts(out, M), passes=passes, moved=int((out != prev).sum()), s1=s1, beaten=beaten, spilled=spilled,
                over=closed, stop=stop, cap=cap)

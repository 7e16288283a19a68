"""Bounded-load placement over object weights (DESIGN.md 3.19), restated from the document (test infrastructure): the round loop of 3.5
with each node's load -- the sum of its objects' weights -- in place of its object count, and weight-0 objects never spilling.

`argmin(rows, mask)` places the objects `rows` over the nodes `mask` allows: hash_argmin restates the hash policy from
tests/spec_py.py (flat HRW, or the HRW2 walk with the closed nodes left out); affinity_bounded_oracle.c32_argmin is the exact fp32
affinity argmin.  `live` is the solver's liveness (active, weight > 0), `active` what the capacity check counts as open.  The loads
are of the global object set, so the result is what every rank of a sharded run sees."""
import numpy as np

import spec_py as S
from affinity_bounded_oracle import NONE, c32_argmin, counts, spill_hash  # noqa: F401  (c32_argmin is re-exported for the tests)


def loads(idx, obj_w, M):
    placed = idx != NONE
    return np.bincount(idx[placed].astype(np.int64), weights=np.asarray(obj_w, np.float64)[placed], minlength=M).astype(np.int64)


def hash_argmin(keys, seeds, weights, solver="hrw", bits=12):
    sd, wl = [int(x) for x in seeds], [int(x) for x in weights]

    def argmin(rows, mask):
        closed = set(np.flatnonzero(~np.asarray(mask, bool)).tolist())
        if solver == "hrw":
            return np.array([S.hrw(int(keys[i]), sd, wl, closed) for i in rows], dtype=np.uint32)
        return np.array([S.hrw2(int(keys[i]), sd, wl, closed, bits) for i in rows], dtype=np.uint32)
    return argmin


def assign_bounded_weighted(keys, obj_w, argmin, weights, live, active=None, load_total=0, num=5, den=4, max_rounds=4):
    """-> dict(idx, counters, loads, passes, pass0, closed, stop); stop is 'rounds', 'balanced' or 'closed'."""
    keys = np.asarray(keys, dtype=np.uint64)
    obj_w = np.asarray(obj_w, dtype=np.int64)
    weights = np.asarray(weights, dtype=np.uint64)
    live = np.asarray(live, bool)
    active = live if active is None else np.asarray(active, bool)
    n, M = len(keys), len(weights)
    L = load_total or int(obj_w.sum())
    W = int(weights[live].sum())
    cap = np.array([S.capacity(L, int(weights[j]), W, num, den) if live[j] else 0 for j in range(M)], dtype=np.int64)
    idx = np.asarray(argmin(np.arange(n), live), dtype=np.uint32)
    pass0 = idx.copy()
    closed = np.zeros(M, bool)
    passes, stop = 1, "rounds"
    for r in range(1, max_rounds):
        ld = loads(idx, obj_w, M)
        over = active & (ld > cap)
        closed |= over
        if not over.any():
            stop = "balanced"
            break
        if not (active & ~closed).any():
            stop = "closed"
            break
        thr = np.zeros(M, dtype=np.uint64)
        thr[over] = [((int(ld[j]) - int(cap[j])) << 32) // int(ld[j]) for j in np.flatnonzero(over)]
        placed = idx != NONE
        on_over = np.zeros(n, bool)
        on_over[placed] = over[idx[placed]]
        spill = on_over & (obj_w > 0) & (spill_hash(keys, r) < thr[np.where(placed, idx, 0)])
        rows = np.flatnonzero(spill)
        if len(rows):
            idx[rows] = argmin(rows, live & ~closed)
        passes += 1
    return dict(idx=idx, counters=counts(idx, M), loads=loads(idx, obj_w, M), passes=passes, pass0=pass0, closed=closed, stop=stop)


def erase_pairing(keys, erase):
    """The rows of set_erase (DESIGN.md 3.18) as an index array: row i of the set after the call is row out[i] before it."""
    keys = np.asarray(keys, dtype=np.uint64)
    gone = np.isin(keys, np.asarray(erase, dtype=np.uint64))
    n_new = len(keys) - int(gone.sum())
    rows = np.arange(n_new)
    holes = np.flatnonzero(gone[:n_new])
    movers = n_new + np.flatnonzero(~gone[n_new:])
    rows[holes] = movers
    return rows

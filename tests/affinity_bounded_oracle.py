"""Bounded-load placement under the affinity cost (DESIGN.md 3.16), restated from the document (test infrastructure): the round loop
of 3.5 (tests/spec_py.py::assign_bounded) with the rendezvous hash replaced by an affinity argmin over the live nodes not closed.

`argmin(rows, mask)` places the objects `rows` over the nodes `mask` allows.  c32_argmin gives the exact fp32 minimum of
tests/affinity_c32_ref.py, the answer on the CUDA cores and, for features whose products and sums are exact, on the tensor cores too;
the GPU tests also pass an argmin built from the engine itself (a twin handle whose closed nodes are inactive).

`live` is the solver's liveness (active, weight > 0); `active` is what the capacity check of 3.5 counts as open (an active node of
weight 0 keeps the rounds going, though nothing can be placed on it).  The counts are of the global key set, so the result is what
every rank of a sharded run sees."""
import numpy as np

import affinity_c32_ref as C32
from spec_py import capacity

NONE = 0xFFFFFFFF
M64 = (1 << 64) - 1
SALT_SPILL = 0x2545F4914F6CDD1D
GOLDEN = 0x9E3779B97F4A7C15


def mix64(x):
    x = x.astype(np.uint64)
    x ^= x >> np.uint64(30)
    x *= np.uint64(0xBF58476D1CE4E5B9)
    x ^= x >> np.uint64(27)
    x *= np.uint64(0x94D049BB133111EB)
    x ^= x >> np.uint64(31)
    return x


def spill_hash(keys, rnd):
    """hi32(mix64(key ^ (SALT_SPILL + round * GOLDEN))) for every key (tests/spec_py.py::spill_hash, vectorised)."""
    return mix64(np.asarray(keys, dtype=np.uint64) ^ np.uint64((SALT_SPILL + rnd * GOLDEN) & M64)) >> np.uint64(32)


def c32_argmin(fo, fn):
    def argmin(rows, mask):
        return C32.ranked(fo[rows], fn, mask, 1)[:, 0]
    return argmin


def counts(idx, M):
    return np.bincount(idx[idx != NONE].astype(np.int64), minlength=M).astype(np.uint32)


def assign_bounded(keys, argmin, weights, live, active=None, n_total=0, num=5, den=4, max_rounds=4):
    """-> (idx, counters, passes, pass0, closed, stop): closed is the final closed set; stop is 'rounds' (max_rounds reached),
    'balanced' (no node over) or 'closed' (no node open)."""
    keys = np.asarray(keys, dtype=np.uint64)
    weights = np.asarray(weights, dtype=np.uint64)
    live = np.asarray(live, bool)
    active = live if active is None else np.asarray(active, bool)
    n, M = len(keys), len(weights)
    N = n_total or n
    W = int(weights[live].sum())
    cap = np.array([capacity(N, int(weights[j]), W, num, den) if live[j] else 0 for j in range(M)], dtype=np.int64)
    idx = argmin(np.arange(n), live).astype(np.uint32)
    pass0 = idx.copy()
    closed = np.zeros(M, bool)
    passes, stop = 1, "rounds"
    for r in range(1, max_rounds):
        c = counts(idx, M).astype(np.int64)
        over = active & (c > cap)
        closed |= over
        if not over.any():
            stop = "balanced"
            break
        if not (active & ~closed).any():
            stop = "closed"
            break
        thr = np.zeros(M, dtype=np.uint64)
        thr[over] = [((int(c[j]) - int(cap[j])) << 32) // int(c[j]) for j in np.flatnonzero(over)]
        placed = idx != NONE
        on_over = np.zeros(n, bool)
        on_over[placed] = over[idx[placed]]
        spill = on_over & (spill_hash(keys, r) < thr[np.where(placed, idx, 0)])
        rows = np.flatnonzero(spill)
        if len(rows):
            idx[rows] = argmin(rows, live & ~closed)
        passes += 1
    return idx, counts(idx, M), passes, pass0, closed, stop

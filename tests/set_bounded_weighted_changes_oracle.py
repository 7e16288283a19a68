"""A weighted bounded set kept within load capacity (DESIGN.md 3.21), restated from the document (test infrastructure): pass 0 of the
recorded kind on the current assignment, then the weighted rounds of 3.19 from the loads it leaves, closed set empty, rounds numbered
from 1.

Pass 0:
* flat HRW (3.10): R1 -- an object on NONE, past the table or on a REPLACE node takes the flat placement over the live set; R2 -- any
  other object takes the best of {its node} u CANDIDATES under the flat score (spec_py.hrw over those nodes alone);
* HRW2: S1 as R1 but with the walk (spec_py.hrw2); S2 -- an object moves to its walk's answer iff that node is a CANDIDATE;
* affinity: tests/affinity_set_bounded_oracle.py's pass 0 (its call with max_rounds = 1).
The rounds are tests/bounded_weighted_oracle.py's, entered with the pass-0 result in place of its own pass 0.  Nothing here is shared
with the engine."""
import numpy as np

import affinity_set_bounded_oracle as ASB
import bounded_weighted_oracle as BW
import spec_py as S

NONE = BW.NONE
M32 = 0xFFFFFFFF


def change_set(policy, changed, prev_weight, weights, live, refeatured=()):
    """-> (replace: bool per interned node, cand: sorted node list) of a change set under `policy` ('hrw', 'hrw2' or 'affinity')."""
    live = np.asarray(live, bool)
    replace = ~live
    cand = set()
    for j, pw in zip(changed, prev_weight):
        j, pw, w = int(j), int(pw), int(weights[j])
        if not live[j]:
            continue
        if policy == "affinity":
            if pw == 0:
                cand.add(j)
        elif policy == "hrw":
            r_prev, r_now = S.inv_weight(pw), S.inv_weight(w)
            if r_prev and r_now > r_prev:
                replace[j] = True
            elif not r_prev or r_now < r_prev:
                cand.add(j)
        else:
            if pw and w < pw:
                replace[j] = True
            elif not pw or w > pw:
                cand.add(j)
    for j in refeatured:
        if live[j]:
            replace[j] = True
            cand.add(int(j))
    return replace, sorted(cand)


def hash_pass0(policy, keys, idx, seeds, weights, live, replace, cand, bits=12):
    """-> (idx after pass 0, s1, beaten) under flat HRW or HRW2."""
    keys = np.asarray(keys, np.uint64)
    prev = np.asarray(idx, np.uint32)
    M = len(weights)
    sd, wl = [int(x) for x in seeds], [int(x) for x in weights]
    closed = set(np.flatnonzero(~np.asarray(live, bool)).tolist())
    out = prev.copy()
    s1 = prev >= M
    s1[~s1] = replace[prev[~s1]]
    beaten = np.zeros(len(keys), bool)
    cset = set(cand)
    for i in range(len(keys)):
        k, y = int(keys[i]), int(prev[i])
        if policy == "hrw":
            if s1[i]:
                out[i] = S.hrw(k, sd, wl, closed)
            elif cand:
                wr = [wl[j] if (j == y or j in cset) else 0 for j in range(M)]
                out[i] = S.hrw(k, sd, wr)
        elif s1[i] or cand:
            f = S.hrw2(k, sd, wl, closed, bits)
            if s1[i] or f in cset:
                out[i] = f
    beaten[~s1] = out[~s1] != prev[~s1]
    return out, s1, beaten


def rebalance(policy, keys, idx, obj_w, weights, live, active, changed, prev_weight, argmin, load_total=0, num=5, den=4, max_rounds=4,
              seeds=None, bits=12, fo=None, fn=None, refeatured=()):
    """-> dict: idx, counters, loads, passes, moved, pass0, s1, beaten, closed (nodes over capacity in some round), stop.

    `argmin(rows, mask)` is the re-placement of the rounds, as in bounded_weighted_oracle; for affinity it also re-places the S1 objects
    of pass 0.  Under the hash policies an empty change set leaves pass 0 out."""
    prev = np.asarray(idx, np.uint32)
    replace, cand = change_set(policy, changed, prev_weight, weights, live, refeatured)
    if policy == "affinity":
        r = ASB.rebalance(keys, prev, fo, fn, argmin, replace, cand, weights, live, active, max_rounds=1)
        p0, s1, beaten = r["idx"], r["s1"], r["beaten"]
    elif len(changed):
        p0, s1, beaten = hash_pass0(policy, keys, prev, seeds, weights, live, replace, cand, bits)
    else:
        p0, s1, beaten = prev.copy(), np.zeros(len(prev), bool), np.zeros(len(prev), bool)
    entered = [False]

    def rounds_argmin(rows, mask):   # the rounds' own pass 0 is the pass-0 result above
        if not entered[0]:
            entered[0] = True
            return p0.copy()
        return argmin(rows, mask)

    out = BW.assign_bounded_weighted(keys, obj_w, rounds_argmin, weights, live, active, load_total, num, den, max_rounds)
    out["moved"] = int((out["idx"] != prev).sum())
    out.update(s1=s1, beaten=beaten, replace=replace, cand=cand)
    return out

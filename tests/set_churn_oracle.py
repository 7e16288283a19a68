"""Object churn in a resident set (DESIGN.md 3.18), restated from the document (test infrastructure).

A Shadow holds a set's columns as numpy arrays -- keys (n,), idx (n,), lists (n, R) or None, feats (n, K) or None -- its per-node
counters and whether it is assigned.  insert appends rows placed by `place(keys, feats) -> (idx, lists)`, the batch call of the set's
kind (the caller passes the engine's own batch call of the same handle, tested elsewhere against its own oracle); erase removes every
row whose key is in the erase list and fills the holes below the new size with the surviving rows at or above it, both in increasing
order."""
import numpy as np

NONE = 0xFFFFFFFF


def counts(idx, M):
    idx = np.asarray(idx, dtype=np.int64)
    idx = idx[(idx >= 0) & (idx < M)]
    return np.bincount(idx, minlength=M).astype(np.int64)


class Shadow:
    def __init__(self, keys, idx, lists, feats, counters, assigned):
        self.keys = np.asarray(keys, dtype=np.uint64).copy()
        self.idx = np.asarray(idx, dtype=np.uint32).copy()
        self.lists = None if lists is None else np.asarray(lists, dtype=np.uint32).copy()
        self.feats = None if feats is None else np.asarray(feats, dtype=np.float32).copy()
        self.counters = np.asarray(counters, dtype=np.int64).copy()
        self.assigned = assigned

    @property
    def n(self):
        return len(self.keys)

    def grow_counters(self, M):
        if len(self.counters) < M:
            self.counters = np.concatenate([self.counters, np.zeros(M - len(self.counters), np.int64)])

    def insert(self, keys, feats, place, M):
        """-> first new row"""
        keys = np.asarray(keys, dtype=np.uint64)
        first = self.n
        if not len(keys):
            return first
        self.grow_counters(M)
        lists = None
        if self.assigned:
            idx, lists = place(keys, feats)
            idx = np.asarray(idx, dtype=np.uint32)
            self.counters += counts(idx, len(self.counters))
        else:
            idx = np.full(len(keys), NONE, np.uint32)
        self.keys = np.concatenate([self.keys, keys])
        self.idx = np.concatenate([self.idx, idx])
        if self.lists is not None:
            self.lists = np.concatenate([self.lists, lists])
        if self.feats is not None:
            self.feats = np.concatenate([self.feats, np.asarray(feats, np.float32)])
        return first

    def layout(self, erase_keys):
        """-> (flag, n_new, holes, movers) of DESIGN.md 3.18"""
        flag = np.isin(self.keys, np.asarray(erase_keys, dtype=np.uint64))
        n_new = self.n - int(flag.sum())
        holes = np.flatnonzero(flag[:n_new])
        movers = n_new + np.flatnonzero(~flag[n_new:])
        assert len(holes) == len(movers)
        return flag, n_new, holes, movers

    def erase(self, erase_keys, M):
        """-> rows removed"""
        if not len(erase_keys):
            return 0
        flag, n_new, holes, movers = self.layout(erase_keys)
        self.grow_counters(M)
        if self.assigned:
            self.counters -= counts(self.idx[flag], len(self.counters))
        for name in ("keys", "idx", "lists", "feats"):
            col = getattr(self, name)
            if col is None:
                continue
            col = col.copy()
            col[holes] = col[movers]
            setattr(self, name, col[:n_new])
        return int(flag.sum())

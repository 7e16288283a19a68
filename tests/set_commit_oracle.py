"""Delta commit of a resident set (DESIGN.md 3.20), restated from the document (test infrastructure).

A Directory is a dict model of the placement directory: normalised key -> node, RIO_NONE for a removed key, filled from the
directory's own lookup_many answers for the keys a test looks at.  commit(keys, idx, dry_run) selects every row whose idx differs
from the model's answer for its key at the start of the call, returns the manifest (rows, keys as stored, from, to) in increasing row
order and, unless dry_run, writes the selected rows into the model in row order, so the last selected row of a key wins."""
import numpy as np

NONE = 0xFFFFFFFF
EMPTY = 0xFFFFFFFFFFFFFFFF


def norm(k):
    """the directory folds its reserved empty key onto its neighbour (DESIGN.md 4.2)"""
    k = int(k)
    return EMPTY - 1 if k == EMPTY else k


class Directory:
    def __init__(self, keys, answers):
        self.d = {}
        for k, a in zip(np.asarray(keys, np.uint64).tolist(), np.asarray(answers, np.uint32).tolist()):
            self.d[norm(k)] = a

    def answer(self, keys):
        return np.array([self.d.get(norm(k), NONE) for k in np.asarray(keys, np.uint64).tolist()], dtype=np.uint32)

    def commit(self, keys, idx, dry_run=False):
        """-> (rows u64, keys u64, from u32, to u32)"""
        keys = np.asarray(keys, np.uint64)
        idx = np.asarray(idx, np.uint32)
        frm = self.answer(keys)
        rows = np.flatnonzero(idx != frm)
        manifest = (rows.astype(np.uint64), keys[rows], frm[rows], idx[rows])
        if not dry_run:
            for k, t in zip(manifest[1].tolist(), manifest[3].tolist()):
                self.d[norm(k)] = t
        return manifest

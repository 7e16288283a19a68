"""fp64 oracle of the failure-domain affinity lists (DESIGN.md 3.14; test infrastructure) and the acceptance rule the tests and
tools/bench_affinity_spread.py apply to a list returned by the engine.

The exact list is the greedy pass over each object's live nodes in (fp64 cost, node index) order, cost = -sum_k F_obj[i,k] F_node[j,k],
that keeps the first node of each domain not listed yet.  The engine computes in fp32 (on the tensor cores from a three-piece bf16
split), so one near-tie can change a rank and, through its domain, every later rank.  The rule is therefore conditioned on the
engine's own earlier ranks: for rank r, S_r is the set of live nodes outside the domains of got[:, :r], and a list is accepted when
  (a) its entries are live, lie in distinct domains, and are RIO_NONE exactly past the number of live domains;
  (b) the fp64 cost of got[:, r] is within tau(got) + tau(want) of the minimum over S_r (want: the argmin over S_r);
  (c) got[:, r] is that argmin wherever the fp64 gap to the second-best node of S_r exceeds the same tolerance.
tau is the condition-aware tolerance of affinity_ranked_oracle.  A label of RIO_NONE is a domain of its own."""
import numpy as np

from affinity_ranked_oracle import cost_of, tau

NONE = 0xFFFFFFFF


def domain_ids(labels, M):
    """int64 domain per node: the label, or a unique negative id for RIO_NONE (and for every node when labels is None)."""
    own = -1 - np.arange(M, dtype=np.int64)
    if labels is None:
        return own
    lab = np.asarray(labels, dtype=np.uint32).astype(np.int64)
    return np.where(lab == NONE, own, lab)


def check(got, fo, fn, live, labels, chunk=8192):
    """Asserts (a)-(c) for the engine's (n, R) lists.  Returns the number of entries that differ from the conditioned argmin (all of
    them near-ties)."""
    got = np.asarray(got)
    n, R = got.shape
    live = np.asarray(live, dtype=bool)
    M = len(live)
    dom_all = domain_ids(labels, M)
    live_idx = np.flatnonzero(live)
    n_dom = len(np.unique(dom_all[live_idx]))
    d = min(R, n_dom)
    # (a)
    assert (got[:, d:] == NONE).all(), "entries past the live domains are not RIO_NONE"
    head = got[:, :d]
    assert (head != NONE).all() and (head < M).all(), "RIO_NONE inside the live domain count"
    assert live[head].all(), "a node that is not live"
    hd = dom_all[head]
    for a in range(d):
        for b in range(a + 1, d):
            assert (hd[:, a] != hd[:, b]).all(), ("two ranks in one domain", a, b)
    if not d:
        return 0
    dom_live = dom_all[live_idx]
    fl = np.asarray(fn, dtype=np.float64)[live_idx]
    differ = 0
    for lo in range(0, n, chunk):
        hi = min(n, lo + chunk)
        c = -(np.asarray(fo[lo:hi], dtype=np.float64) @ fl.T)
        excluded = np.zeros(c.shape, dtype=bool)
        for r in range(d):
            cm = np.where(excluded, np.inf, c)
            arg = np.argmin(cm, axis=1)   # the first live position of the minimum: the lowest node index
            best = cm[np.arange(hi - lo), arg]
            cm[np.arange(hi - lo), arg] = np.inf
            second = cm.min(axis=1)
            want = live_idx[arg].astype(np.uint32)
            g = head[lo:hi, r]
            tol = tau(fo[lo:hi], fn, g[:, None])[:, 0] + tau(fo[lo:hi], fn, want[:, None])[:, 0]
            err = cost_of(fo[lo:hi], fn, g[:, None])[:, 0] - best
            # (b)
            assert (np.abs(err) <= tol).all(), ("cost off by more than the tolerance", r, float((np.abs(err) - tol).max()),
                                                 (lo + np.flatnonzero(np.abs(err) > tol)[:5]).tolist())
            # (c)
            clear = second - best > tol
            wrong = clear & (g != want)
            assert not wrong.any(), ("index differs where the order is clear", r, (lo + np.flatnonzero(wrong)[:5]).tolist())
            differ += int((g != want).sum())
            excluded |= dom_live[None, :] == hd[lo:hi, r][:, None]
    return differ

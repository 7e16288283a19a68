"""fp64 oracle of the ranked affinity lists (DESIGN.md 3.9; test infrastructure) and the acceptance rule the tests and
tools/bench_affinity_ranked.py apply to a list returned by the engine.

The oracle sorts every object's live nodes fully by (fp64 cost, node index), cost = -sum_k F_obj[i,k] F_node[j,k], in chunks of
objects.  The engine computes in fp32 (and, on the tensor cores, from a three-piece bf16 split), so its lists are compared under a
condition-aware tolerance instead of bit for bit:

    tau(i, j) = 1e-5 * sum_k |F_obj[i,k] F_node[j,k]| + 1e-12

A list is accepted when
  (a) its entries are distinct live nodes and it is RIO_NONE exactly past the live count;
  (b) at every rank the fp64 cost of the returned node is within tau(got) + tau(want) of the oracle's cost at that rank;
  (c) the index is the oracle's wherever the oracle's fp64 gaps to both neighbouring ranks exceed that tolerance."""
import numpy as np

NONE = 0xFFFFFFFF


def tau(fo, fn, idx):
    """tau(i, idx[i, r]) for an (n, R) index array (entries past the live set are ignored by the callers)."""
    safe = np.where(idx == NONE, 0, idx).astype(np.int64)
    return 1e-5 * np.einsum("nk,nrk->nr", np.abs(fo.astype(np.float64)), np.abs(fn.astype(np.float64))[safe]) + 1e-12


def cost_of(fo, fn, idx):
    safe = np.where(idx == NONE, 0, idx).astype(np.int64)
    return -np.einsum("nk,nrk->nr", fo.astype(np.float64), fn.astype(np.float64)[safe])


def ranked(fo, fn, live, depth, chunk=8192):
    """(idx, cost): each object's first `depth` live nodes in increasing (fp64 cost, node index) order and their fp64 costs;
    RIO_NONE / +inf past the live set."""
    fo = np.asarray(fo, dtype=np.float64)
    live_idx = np.flatnonzero(np.asarray(live))
    fl = np.asarray(fn, dtype=np.float64)[live_idx]
    n = fo.shape[0]
    idx = np.full((n, depth), NONE, dtype=np.uint32)
    cost = np.full((n, depth), np.inf)
    d = min(depth, len(live_idx))
    if not d:
        return idx, cost
    for lo in range(0, n, chunk):
        c = -(fo[lo:lo + chunk] @ fl.T)
        order = np.argsort(c, axis=1, kind="stable")[:, :d]   # live_idx is increasing: stable order breaks ties by node index
        idx[lo:lo + chunk, :d] = live_idx[order]
        cost[lo:lo + chunk, :d] = np.take_along_axis(c, order, axis=1)
    return idx, cost


def check(got, fo, fn, live, want=None):
    """Asserts (a)-(c) for the engine's (n, R) lists; `want` = ranked(fo, fn, live, R + 1) when already computed (it may be deeper).
    Returns the number of entries whose index differs from the oracle's (all of them near-ties)."""
    got = np.asarray(got)
    n, R = got.shape
    live = np.asarray(live, dtype=bool)
    n_live = int(live.sum())
    if want is None:
        want = ranked(fo, fn, live, R + 1)
    w_idx, w_cost = want[0][:, :R + 1], want[1][:, :R + 1]
    if w_idx.shape[1] < R + 1:   # the oracle went exactly R deep: no rank past the list
        w_idx = np.concatenate([w_idx, np.full((n, 1), NONE, np.uint32)], axis=1)
        w_cost = np.concatenate([w_cost, np.full((n, 1), np.inf)], axis=1)
    d = min(R, n_live)
    # (a)
    assert (got[:, d:] == NONE).all(), "entries past the live set are not RIO_NONE"
    head = got[:, :d]
    assert (head != NONE).all() and (head < len(live)).all(), "RIO_NONE inside the live count"
    assert live[head].all(), "a node that is not live"
    for a in range(d):
        for b in range(a + 1, d):
            assert (head[:, a] != head[:, b]).all(), ("repeated node", a, b)
    if not d:
        return 0
    # (b)
    tol = tau(fo, fn, head) + tau(fo, fn, w_idx[:, :d])
    c_got = cost_of(fo, fn, head)
    err = np.abs(c_got - w_cost[:, :d])
    assert (err <= tol).all(), ("cost off by more than the tolerance", float((err - tol).max()), np.argwhere(err > tol)[:5].tolist())
    # (c)
    prev = np.concatenate([np.full((n, 1), np.inf), np.diff(w_cost[:, :d], axis=1)], axis=1)
    nxt = w_cost[:, 1:d + 1] - w_cost[:, :d]
    nxt = np.where(np.isfinite(nxt), nxt, np.inf)
    clear = (prev > tol) & (nxt > tol)
    wrong = clear & (head != w_idx[:, :d])
    assert not wrong.any(), ("index differs where the oracle's order is clear", np.argwhere(wrong)[:5].tolist())
    return int((head != w_idx[:, :d]).sum())

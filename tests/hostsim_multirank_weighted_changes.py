"""N ranks of the engine in ONE process keeping weighted bounded sets within load capacity (DESIGN.md 3.21); run only against the
host-sim library, by tests/test_gpu_set_bounded_weighted_changes.py:

    RIO_HOSTSIM_LIBRARY=<host-sim .so with the weighted doubles> python tests/hostsim_multirank_weighted_changes.py <world>

Every rank is a thread with its own handle, attached as in tests/hostsim_multirank_weighted.py, and holds an id-range shard with its own
weights.  Each rank runs the same sequence: a weighted assign, a leave, a weight drift written by key with the GLOBAL key list (every
rank ignores the keys it does not hold), a rejoin and a weight increase, each followed by the change-set call, under the hash policies
and the affinity cost, with load_total defaulted and given.  Checked: every rank's shard, counters, loads, moved count summed over the
ranks and passes equal one rank holding the whole set; and a weight total past 2^32 - 1 that no single shard reaches is refused on every
rank, with every shard unchanged."""
import os
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from rio_rs_b200 import _native  # noqa: E402

_native.library_path = lambda: os.environ["RIO_HOSTSIM_LIBRARY"]
_native._lib = None

import rio_rs_b200 as R  # noqa: E402
from rio_rs_b200 import parallel  # noqa: E402

KINDS = [("hrw", False), ("hrw2", False), ("hrw", True)]


def addresses(M):
    return ["10.7.%d.%d:7000" % (j >> 8, j & 255) for j in range(M)]


def sequence(p, s, ow, w, fn, drift_keys, drift_w, total):
    """The calls of one rank (or of the one-rank reference): {(solver, affinity, lt, step): (moved, passes, idx, counters, loads)}."""
    out = {}
    addrs = addresses(len(w))
    for solver, aff in KINDS:
        for lt in (0, total + 5000):
            p.set_solver(solver, 12)
            p.set_nodes(addrs, w, fn)
            s.write_weights(ow)
            s.assign_bounded_weighted(aff, lt, 5, 4, 8)

            def step(t, idx, prev):
                moved, passes = s.rebalance_changes_bounded_weighted(idx, prev, lt, 1, 1, 8)
                out[solver, aff, lt, t] = (moved, passes, s.read(), s.counters(), s.loads())

            p.node_set_active(3, False)
            step(0, [3], [int(w[3])])
            s.write_weights_by_key(drift_keys, drift_w)
            step(1, [], [])
            p.node_set_active(3, True)
            p.node_upsert(addrs[7], int(w[7]) * 3)
            step(2, [3, 7], [0, int(w[7])])
    return out


def main():
    world = int(sys.argv[1])
    n, M, K = 30_000, 40, 8
    rng = np.random.default_rng(23)
    w = rng.integers(1, 17, M).astype(np.uint32)
    fn = rng.uniform(-1, 1, (M, K)).astype(np.float32)
    fo = rng.uniform(-1, 1, (n, K)).astype(np.float32)
    keys = rng.integers(0, 2**63, n, dtype=np.uint64)
    ow = np.clip(np.round(np.exp(rng.normal(0.0, 1.5, n)) * 4), 1, 20000).astype(np.uint32)
    drift = rng.choice(n, n // 20, replace=False)
    drift_keys, drift_w = keys[drift], rng.integers(1, 200, len(drift)).astype(np.uint32)
    total = int(ow.astype(np.int64).sum()) - int(ow[drift].astype(np.int64).sum()) + int(drift_w.astype(np.int64).sum())
    handles, results, errors = [None] * world, [None] * world, []
    bar = threading.Barrier(world)

    def rank_main(rank):
        try:
            p = R.GpuObjectPlacement()
            handles[rank] = p.comm_ipc_export(world)
            bar.wait()
            p.comm_ipc_attach(rank, world, handles)
            bar.wait()
            p.set_nodes(addresses(M), w, fn)
            lo, hi = parallel.shard_range(n, rank, world)
            s = p.new_set(hi - lo)
            s.load_keys(keys[lo:hi])
            s.load_feats(fo[lo:hi])
            out = sequence(p, s, ow[lo:hi], w, fn, drift_keys, drift_w, total)
            # every shard stays below 2^32 - 1, their sum does not: every rank refuses, before anything is written
            before = (s.read().tobytes(), s.counters().tobytes())
            big = np.zeros(hi - lo, np.uint32)
            big[0] = 0xFFFFFFFF // world + 1
            s.write_weights(big)
            try:
                s.rebalance_changes_bounded_weighted([], [])
                refused = False
            except R.Unknown:
                refused = (s.read().tobytes(), s.counters().tobytes()) == before
            results[rank] = (lo, hi, out, refused)
            bar.wait()
        except Exception as e:  # noqa: BLE001
            errors.append("rank %d: %r" % (rank, e))
            bar.abort()

    th = [threading.Thread(target=rank_main, args=(r,), daemon=True) for r in range(world)]
    for x in th:
        x.start()
    for x in th:
        x.join(timeout=600)
        assert not x.is_alive(), "a rank did not finish"
    assert not errors, errors
    p = R.GpuObjectPlacement()
    p.set_nodes(addresses(M), w, fn)
    s = p.new_set(n)
    s.load_keys(keys)
    s.load_feats(fo)
    want = sequence(p, s, ow, w, fn, drift_keys, drift_w, total)
    fired = 0
    for key, (moved, passes, idx, cnt, ld) in want.items():
        fired += passes > 1
        assert sum(out[key][0] for _, _, out, _ in results) == moved, key
        for lo, hi, out, _ in results:
            _, gp, gi, gc, gl = out[key]
            assert gp == passes and gi.tobytes() == idx[lo:hi].tobytes() and (gc == cnt).all() and (gl == ld).all(), key
    assert fired >= 4, fired
    for *_, refused in results:
        assert refused, "a rank did not refuse the total past 2^32 - 1"
    print("multirank weighted changes ok: world %d" % world)


if __name__ == "__main__":
    main()

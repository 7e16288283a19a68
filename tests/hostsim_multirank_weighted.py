"""N ranks of the engine in ONE process running the weighted bounded-load calls (DESIGN.md 3.19); run only against the host-sim library,
by tests/test_gpu_set_bounded_weighted.py:

    RIO_HOSTSIM_LIBRARY=<host-sim .so with the weighted doubles> python tests/hostsim_multirank_weighted.py <world>

Every rank is a thread with its own handle, attached through rio_cuda_comm_ipc_export / _attach as in tests/hostsim_multirank.py.  Each
holds an id-range shard with its own weights, so the shards' weight sums differ.  Checked: with load_total defaulted (the weight sum of
all ranks) and given explicitly, under the hash policy and the affinity cost, every rank's shard, counters and loads equal one rank
holding the whole set; and a weight total past 2^32 - 1 that no single shard reaches is refused on every rank, so no rank is left in an
exchange alone."""
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

CAPS = [(5, 4), (101, 100), (1, 1)]


def addresses(M):
    return ["10.6.%d.%d:7000" % (j >> 8, j & 255) for j in range(M)]


def calls(p, s, n_loaded, ow):
    """The weighted calls of one rank (or of the one-rank reference): {(affinity, cap, load_total): (passes, idx, counters, loads)}."""
    out = {}
    total = int(ow.astype(np.int64).sum())
    for aff in (False, True):
        for cap in CAPS:
            for lt in (0, total):
                passes = s.assign_bounded_weighted(aff, lt, cap[0], cap[1], 8)
                out[aff, cap, lt] = (passes, s.read(), s.counters(), s.loads())
    return out


def main():
    world = int(sys.argv[1])
    n, M, K = 60_000, 40, 8
    rng = np.random.default_rng(19)
    w = rng.integers(1, 17, M).astype(np.uint32)
    fn = rng.uniform(-1, 1, (M, K)).astype(np.float32)
    fo = rng.uniform(-1, 1, (n, K)).astype(np.float32)
    keys = rng.integers(0, 2**63, n, dtype=np.uint64)
    ow = np.clip(np.round(np.exp(rng.normal(0.0, 1.5, n)) * 4), 1, 20000).astype(np.uint32)
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
            s.write_weights(ow[lo:hi])
            out = calls(p, s, hi - lo, ow)
            # every shard stays below 2^32 - 1, their sum does not: every rank refuses, before any round
            big = np.zeros(hi - lo, np.uint32)
            big[0] = 0xFFFFFFFF // world + 1
            s.write_weights(big)
            refused = []
            for call in (lambda: s.assign_bounded_weighted(False), lambda: s.loads()):
                try:
                    call()
                    refused.append(False)
                except R.Unknown:
                    refused.append(True)
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
    s.write_weights(ow)
    want = calls(p, s, n, ow)
    shard_sums = [int(ow[lo:hi].astype(np.int64).sum()) for lo, hi, _, _ in results]
    assert len(set(shard_sums)) == world, shard_sums   # the default must not come from one shard's sum
    fired = 0
    for key, (passes, idx, cnt, ld) in want.items():
        fired += passes > 1
        for lo, hi, out, _ in results:
            gp, gi, gc, gl = out[key]
            assert gp == passes and gi.tobytes() == idx[lo:hi].tobytes() and (gc == cnt).all() and (gl == ld).all(), key
    assert fired >= 4
    for *_, refused in results:
        assert refused == [True, True], refused
    print("multirank weighted ok: world %d" % world)


if __name__ == "__main__":
    main()

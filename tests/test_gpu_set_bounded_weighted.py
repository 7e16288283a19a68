"""Weighted objects in bounded-load placement (DESIGN.md 3.19): ObjectSet.assign_bounded_weighted, ObjectSet.loads, the weight column
and GpuObjectPlacement.assign_bounded_weighted_batch against tests/bounded_weighted_oracle.py.

* Identity: weights never written, or written as all 1 with load_total = n, give idx, counters and passes of set_assign_bounded (flat
  HRW, HRW2 at 12 and 5 bits) and of set_assign_bounded_affinity (CUDA cores at K = 8, 16, 24, tensor cores at K = 16) bit for bit.
* Oracle, bit for bit (idx, passes, loads, counters): uniform, lognormal, 1 % hot and partly zero weights, caps 5/4, 101/100, 1/1,
  max_rounds 1..16, both hash policies, affinity on the CUDA cores and on the tensor cores (integer features against c32, U(-1, 1)
  features against a twin handle whose closed nodes are inactive), and live counts either side of 64, 256 and 2304.
* Edge cases, the batch form, the weight column through churn, the state a weighted call leaves, every refusal, two ranks.

The CPU tests at the end run this module's GPU bodies, unchanged, against the engine's host logic compiled with g++ (the host-sim
library of tests/test_engine_host_sim.py) with a plain restatement of the new launchers, and check that a build without them refuses
the weighted calls while the weight column and every other call keep working.  There the tensor path is never taken."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import bounded_weighted_oracle as O
import spec_py as S

NONE = 0xFFFFFFFF
U32 = 0xFFFFFFFF
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAPS = [(5, 4), (101, 100), (1, 1)]
ROUNDS = [1, 2, 4, 16]
MIXES = ["uniform", "lognormal", "hot", "zeros"]


@pytest.fixture(scope="module")
def gp():
    from rio_rs_b200 import build

    build.build()
    import rio_rs_b200 as R

    return R


class variant:
    """RIO_AFFINITY_VARIANT for the calls inside the block: 'ffma' keeps every K = 16 call on the CUDA cores."""

    def __init__(self, v):
        self.v = v

    def __enter__(self):
        os.environ["RIO_AFFINITY_VARIANT"] = self.v

    def __exit__(self, *a):
        os.environ.pop("RIO_AFFINITY_VARIANT", None)


def host_sim(p):
    return p.device_info()["name"].startswith("host-sim")


def addresses(M):
    return ["10.4.%d.%d:7000" % (j >> 8, j & 255) for j in range(M)]


def int_feats(rng, shape):
    return rng.integers(-4, 5, shape).astype(np.float32)


def weight_mix(kind, n, rng):
    if kind == "ones":
        return np.ones(n, np.uint32)
    if kind == "uniform":
        return rng.integers(1, 65, n).astype(np.uint32)
    if kind == "lognormal":
        return np.clip(np.round(np.exp(rng.normal(0.0, 1.5, n)) * 4), 1, 20000).astype(np.uint32)
    if kind == "hot":
        w = np.ones(n, np.uint32)
        w[rng.choice(n, max(n // 100, 1), replace=False)] = 100
        return w
    if kind == "zeros":
        w = rng.integers(1, 9, n).astype(np.uint32)
        w[rng.random(n) < 0.2] = 0
        return w
    raise ValueError(kind)


class Cluster:
    """A handle with M nodes (weights 1..wmax, some inactive, some active with weight 0) and a set of n objects with keys and, for
    K > 0, features, mirrored here for the oracle."""

    def __init__(self, gp, M, n, K=0, seed=0, solver="hrw", bits=12, fo=None, fn=None, dead=(), zero_weight=(), wmax=16):
        rng = np.random.default_rng(2000 + seed)
        self.rng = rng
        self.gp, self.M, self.n, self.K, self.solver, self.bits = gp, M, n, K, solver, bits
        self.fo = (rng.uniform(-1, 1, (n, K)).astype(np.float32) if fo is None else np.asarray(fo, np.float32)) if K else None
        self.fn = (rng.uniform(-1, 1, (M, K)).astype(np.float32) if fn is None else np.asarray(fn, np.float32)) if K else None
        self.w = rng.integers(1, wmax + 1, M).astype(np.uint32)
        self.w[list(zero_weight)] = 0
        self.active = np.ones(M, bool)
        self.active[list(dead)] = False
        self.live = self.active & (self.w > 0)
        self.seeds = [S.node_seed(a) for a in addresses(M)]
        self.keys = rng.integers(0, 2**63, n, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, n, dtype=np.uint64)
        self.p = self.handle(self.active)
        self.s = self.p.new_set(n + 64)
        self.s.load_keys(self.keys)
        if K:
            self.s.load_feats(self.fo)

    def handle(self, mask):
        p = self.gp.GpuObjectPlacement()
        p.set_solver(self.solver, self.bits)
        p.set_nodes(addresses(self.M), self.w, self.fn)
        for j in np.flatnonzero(~np.asarray(mask, bool)):
            p.node_set_active(int(j), False)
        return p

    def argmin(self, affinity, engine=False):
        if not affinity:
            return O.hash_argmin(self.keys, self.seeds, self.w, self.solver, self.bits)
        if engine:   # the engine as its own primitive: assign_batch on a twin handle whose nodes outside `mask` are inactive
            return lambda rows, mask: self.handle(mask).assign_batch(obj_feats=self.fo[rows])
        return O.c32_argmin(self.fo, self.fn)

    def oracle(self, ow, affinity, cap, rounds, engine=False, load_total=0):
        return O.assign_bounded_weighted(self.keys, ow, self.argmin(affinity, engine), self.w, self.live, self.active, load_total, cap[0], cap[1], rounds)

    def run(self, ow, affinity, cap, rounds, var="umma", want=None, load_total=0):
        """The set call (weights written as ow, or never written for ow None) and the batch call, checked against each other, the
        invariants of 3.19 and `want` (the oracle's dict)."""
        s = self.s
        if ow is not None:
            s.write_weights(ow)
        with variant(var):
            s.assign(affinity)
            plain = s.read()
            if affinity:
                s.assign_ranked_affinity(2)
            else:
                s.assign_ranked(2)
            passes = s.assign_bounded_weighted(affinity, load_total, cap[0], cap[1], rounds)
            got, cnt, ld = s.read(), s.counters(), s.loads()
            bidx, bpasses = self.p.assign_bounded_weighted_batch(self.keys, ow, self.fo if affinity else None, load_total, cap[0], cap[1], rounds)
        with pytest.raises(self.gp.Unknown):
            s.read_ranked()
        wv = np.ones(self.n, np.int64) if ow is None else ow.astype(np.int64)
        assert (cnt == O.counts(got, self.M)).all()
        assert (ld == O.loads(got, wv, self.M)).all()
        assert bidx.tobytes() == got.tobytes() and bpasses == passes
        if want is not None:
            assert plain.tobytes() == want["pass0"].tobytes()
            assert passes == want["passes"], (passes, want["passes"])
            assert got.tobytes() == want["idx"].tobytes(), int((got != want["idx"]).sum())
            assert (cnt == want["counters"]).all() and (ld == want["loads"]).all()
            moved = got != plain
            assert want["closed"][plain[moved]].all() and (wv[moved] > 0).all()
        return got, cnt, passes


# ---- identity with the count-based calls --------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("solver,bits", [("hrw", 12), ("hrw2", 12), ("hrw2", 5)])
def test_all_ones_equal_the_count_based_hash_call(gp, solver, bits):
    c = Cluster(gp, 48, 20000, seed=bits, solver=solver, bits=bits, dead=(3,), zero_weight=(7,))
    fired = 0
    for cap in CAPS:
        for rounds in ROUNDS:
            passes = c.s.assign_bounded(0, cap[0], cap[1], rounds)
            want = (c.s.read(), c.s.counters(), passes)
            fired += passes > 1
            c.s.load_keys(c.keys)   # weights never written
            got = c.run(None, False, cap, rounds)
            c.s.write_weights(np.ones(c.n, np.uint32))
            got1 = c.run(None, False, cap, rounds, load_total=c.n)
            for g in (got, got1):
                assert g[0].tobytes() == want[0].tobytes() and (g[1] == want[1]).all() and g[2] == want[2], (cap, rounds)
    assert fired >= 3


@pytest.mark.gpu
@pytest.mark.parametrize("K,var", [(8, "ffma"), (24, "ffma"), (16, "ffma"), (16, "umma")])
def test_all_ones_equal_the_count_based_affinity_call(gp, K, var):
    c = Cluster(gp, 48, 20000, K, seed=K, dead=(5,), zero_weight=(30,))
    fired = 0
    for cap in CAPS:
        for rounds in (2, 4, 16):
            with variant(var):
                passes = c.s.assign_bounded_affinity(0, cap[0], cap[1], rounds)
            want = (c.s.read(), c.s.counters(), passes)
            fired += passes > 1
            got = c.run(None, True, cap, rounds, var)
            c.s.write_weights(np.ones(c.n, np.uint32))
            got1 = c.run(None, True, cap, rounds, var, load_total=c.n)
            for g in (got, got1):
                assert g[0].tobytes() == want[0].tobytes() and (g[1] == want[1]).all() and g[2] == want[2], (cap, rounds)
            c.s.load_keys(c.keys)
            c.s.load_feats(c.fo)
    assert fired >= 3


# ---- against the oracle ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("solver,bits", [("hrw", 12), ("hrw2", 12), ("hrw2", 5)])
@pytest.mark.parametrize("mix", MIXES)
def test_hash_equals_the_oracle(gp, solver, bits, mix):
    c = Cluster(gp, 40, 1500, seed=7, solver=solver, bits=bits, dead=(2,), zero_weight=(9,))
    ow = weight_mix(mix, c.n, c.rng)
    fired = 0
    for cap, rounds in [((5, 4), 4), ((101, 100), 16), ((1, 1), 2), ((1, 1), 1), ((5, 4), 16)]:
        want = c.oracle(ow, False, cap, rounds)
        fired += c.run(ow, False, cap, rounds, want=want)[2] > 1
    assert fired >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("K,var", [(8, "ffma"), (16, "ffma"), (24, "ffma")])
@pytest.mark.parametrize("mix", MIXES)
def test_cuda_cores_equal_the_oracle(gp, K, var, mix):
    c = Cluster(gp, 48, 8000, K, seed=K, dead=(5, 17), zero_weight=(30,))
    ow = weight_mix(mix, c.n, c.rng)
    fired = 0
    for cap in CAPS:
        for rounds in ROUNDS:
            fired += c.run(ow, True, cap, rounds, var, want=c.oracle(ow, True, cap, rounds))[2] > 1
    assert fired >= 4


@pytest.mark.gpu
@pytest.mark.parametrize("M", [48, 64, 65, 256, 257])
@pytest.mark.parametrize("mix", MIXES)
def test_tensor_cores_equal_the_oracle_on_integer_features(gp, M, mix):
    rng = np.random.default_rng(M)
    n = 8000
    c = Cluster(gp, M, n, 16, seed=M, fo=int_feats(rng, (n, 16)), fn=int_feats(rng, (M, 16)))
    ow = weight_mix(mix, n, rng)
    fired = 0
    for cap, rounds in [((5, 4), 4), ((101, 100), 16), ((1, 1), 16), ((5, 4), 1)]:
        fired += c.run(ow, True, cap, rounds, "umma", want=c.oracle(ow, True, cap, rounds))[2] > 1
    assert fired >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("M", [2304, 2305])
def test_live_count_at_the_tensor_core_limit(gp, M):
    rng = np.random.default_rng(M)
    n = 6000
    c = Cluster(gp, M, n, 16, seed=M, fo=int_feats(rng, (n, 16)), fn=int_feats(rng, (M, 16)))
    ow = weight_mix("lognormal", n, rng)
    for cap, rounds in [((5, 4), 4), ((1, 1), 16)]:
        c.run(ow, True, cap, rounds, "umma", want=c.oracle(ow, True, cap, rounds))


@pytest.mark.gpu
@pytest.mark.parametrize("mix", ["uniform", "hot"])
def test_tensor_cores_equal_the_engine_restatement(gp, mix):
    c = Cluster(gp, 200, 30000, 16, seed=11, dead=(3,))
    ow = weight_mix(mix, c.n, c.rng)
    fired = 0
    for cap in CAPS:
        want = c.oracle(ow, True, cap, 8, engine=True)
        first = c.run(ow, True, cap, 8, "umma", want)
        again = c.run(ow, True, cap, 8, "umma", want)
        assert first[0].tobytes() == again[0].tobytes() and first[2] == again[2]
        fired += first[2] > 1
    assert fired >= 2


# ---- edge cases -----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("affinity", [False, True])
def test_edge_cases(gp, affinity):
    K = 8 if affinity else 0
    c = Cluster(gp, 24, 1200, K, seed=3, dead=(4, 9), zero_weight=(11,))
    rng = c.rng
    # an object heavier than every capacity
    ow = rng.integers(1, 5, c.n).astype(np.uint32)
    ow[17] = 100000
    for cap, rounds in [((5, 4), 16), ((1, 1), 16)]:
        c.run(ow, affinity, cap, rounds, "ffma", c.oracle(ow, affinity, cap, rounds))
    # all weights 0: every load is 0, pass 0 only
    z = np.zeros(c.n, np.uint32)
    got, _, passes = c.run(z, affinity, (5, 4), 16, "ffma", c.oracle(z, affinity, (5, 4), 16))
    assert passes == 1
    # weight-0 objects keep their pass-0 node
    ow = weight_mix("zeros", c.n, rng)
    want = c.oracle(ow, affinity, (1, 1), 16)
    got, _, passes = c.run(ow, affinity, (1, 1), 16, "ffma", want)
    assert passes > 1 and (got[ow == 0] == want["pass0"][ow == 0]).all()
    # explicit against defaulted load_total
    ow = weight_mix("uniform", c.n, rng)
    a = c.run(ow, affinity, (5, 4), 4, "ffma", c.oracle(ow, affinity, (5, 4), 4))
    b = c.run(ow, affinity, (5, 4), 4, "ffma", c.oracle(ow, affinity, (5, 4), 4), load_total=int(ow.sum()))
    assert a[0].tobytes() == b[0].tobytes() and a[2] == b[2]
    big = int(ow.sum()) * 3   # a larger total: larger capacities, fewer spills
    c.run(ow, affinity, (5, 4), 4, "ffma", c.oracle(ow, affinity, (5, 4), 4, load_total=big), load_total=big)


@pytest.mark.gpu
@pytest.mark.parametrize("affinity", [False, True])
def test_no_live_node(gp, affinity):
    K = 8 if affinity else 0
    c = Cluster(gp, 6, 500, K, seed=4, dead=range(6))
    ow = weight_mix("uniform", c.n, c.rng)
    got, cnt, passes = c.run(ow, affinity, (5, 4), 4, "ffma", c.oracle(ow, affinity, (5, 4), 4))
    assert (got == NONE).all() and passes == 1 and not cnt.any()


# ---- the weight column ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_weight_column_through_churn(gp):
    c = Cluster(gp, 32, 3000, seed=5)
    s, rng = c.s, c.rng
    assert (s.read_weights() == 1).all()
    assert (s.loads() == 0).all()   # unassigned
    s.assign()
    assert (s.loads() == s.counters()).all()
    w = np.ones(c.n, np.uint32)
    w[100:400] = rng.integers(0, 1000, 300)
    s.write_weights(w[100:400], first=100)
    w[2900:] = 7
    s.write_weights(w[2900:], first=2900)
    assert s.read_weights().tobytes() == w.tobytes()
    assert s.read_weights(150, 50).tobytes() == w[150:200].tobytes()

    def check(tag):
        keys, idx = s.read(want_keys=True)
        assert s.read_weights().tobytes() == w.tobytes(), tag
        assert (s.loads() == O.loads(idx, w, c.M)).all(), tag
        return keys, idx

    check("written")
    s.assign_bounded_weighted(False, 0, 1, 1, 8)
    check("weighted assign")
    s.assign_bounded(0, 5, 4, 4)
    check("count-based assign")
    c.p.node_set_active(3, False)
    s.rebalance_changes([3], [int(c.w[3])])
    check("change set")
    new = c.keys[:40] + np.uint64(1)
    first = s.insert(new)
    w = np.concatenate([w, np.ones(40, np.uint32)])
    keys, _ = check("insert gives 1")
    s.write_weights(np.full(40, 9, np.uint32), first=first)
    w[first:] = 9
    keys, _ = check("new rows written")
    gone = np.concatenate([keys[rng.choice(len(keys), 500, replace=False)], np.array([12345], np.uint64)])
    rows = O.erase_pairing(keys, gone)
    assert s.erase(gone) == 500
    w = w[rows]
    keys2, _ = check("erase carries the weights")
    assert keys2.tobytes() == keys[rows].tobytes()
    s.load_keys(c.keys)
    assert (s.read_weights() == 1).all()
    s.write_weights(np.full(10, 3, np.uint32))
    s.synth_keys(0, 100, 7)
    assert (s.read_weights() == 1).all()


@pytest.mark.gpu
@pytest.mark.parametrize("affinity", [False, True])
def test_state_after_a_weighted_call(gp, affinity):
    """Counters are object counts, lists and the bounded affinity record are gone, and insert places by the recorded plain kind."""
    K = 16 if affinity else 0
    c = Cluster(gp, 48, 5000, K, seed=6)
    s = c.s
    ow = weight_mix("hot", c.n, c.rng)
    s.write_weights(ow)
    with variant("ffma"):
        if affinity:
            s.assign_bounded_affinity(0, 5, 4, 4)
        s.assign_bounded_weighted(affinity, 0, 1, 1, 8)
        assert (s.counters() == O.counts(s.read(), c.M)).all()
        if affinity:
            with pytest.raises(gp.Unknown):
                s.rebalance_changes_bounded_affinity([], [])
        new = c.rng.integers(0, 2**63, 30, dtype=np.uint64)
        fo = c.rng.uniform(-1, 1, (30, K)).astype(np.float32) if K else None
        first = s.insert(new, fo)
        want = c.p.assign_batch(obj_feats=fo) if affinity else c.p.assign_batch(new)
    assert s.read(first).tobytes() == want.tobytes()
    assert (s.read_weights(first) == 1).all()


# ---- refusals --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_errors_change_nothing(gp):
    R = gp
    c = Cluster(gp, 16, 400, 16, seed=8)
    s, p, L = c.s, c.p, c.p.L
    ow = weight_mix("uniform", c.n, c.rng)
    s.write_weights(ow)
    s.assign_bounded_affinity(0, 5, 4, 4)
    s.assign_ranked(2)

    def state():
        k, idx = s.read(want_keys=True)
        try:
            lists = s.read_ranked().tobytes()
        except R.Unknown:   # a bounded call in flight dropped them
            lists = None
        return s.size(), k.tobytes(), idx.tobytes(), s.counters().tobytes(), s.read_weights().tobytes(), lists

    def refused(call, tag, exc=R.Unknown):
        before = state()
        with pytest.raises(exc):
            call()
        assert state() == before, tag

    assert L.rio_cuda_set_assign_bounded_weighted(None, 0, 0, 5, 4, 4, None) != 0
    assert L.rio_cuda_set_loads(None, None, 0) != 0
    assert L.rio_cuda_set_write_weights(None, 0, 0, None) != 0
    refused(lambda: s.assign_bounded_weighted(False, 0, 5, 0, 4), "cap_den 0")
    refused(lambda: s.assign_bounded_weighted(False, 0, 5, 4, 0), "max_rounds 0")
    refused(lambda: s.assign_bounded_weighted(2), "use_affinity 2")
    refused(lambda: s.write_weights(np.ones(5, np.uint32), first=c.n - 4), "write past the end")
    refused(lambda: s.read_weights(c.n - 4, 5), "read past the end")
    refused(lambda: s._ck(L.rio_cuda_set_write_weights(s.s, 0, 3, None)), "null weights")
    refused(lambda: s.assign_bounded_weighted(False, int(ow.sum()) - 1), "load_total below the local sum")
    refused(lambda: s.assign_bounded_weighted(False, 1 << 32), "load_total past u32")
    # a bounded call in flight
    s.assign_bounded_begin(0, 5, 4, 4)
    refused(lambda: s.assign_bounded_weighted(False), "bounded call in flight")
    s.assign_bounded_end()
    s.assign_ranked(2)
    # affinity: set features of another K, then a handle without node features
    s.load_feats(c.fo[:, :8])
    refused(lambda: s.assign_bounded_weighted(True), "set features of another K")
    s.load_feats(c.fo)
    s.assign_ranked(2)
    q = R.GpuObjectPlacement()
    q.set_nodes(addresses(8))
    t = q.new_set(100)
    t.load_keys(c.keys[:100])
    t.load_feats(c.fo[:100])
    with pytest.raises(R.Unknown):
        t.assign_bounded_weighted(True)
    with pytest.raises(R.Unknown):
        q.assign_bounded_weighted_batch(c.keys[:100], None, c.fo[:100])
    # the u32 rule: a local weight sum of exactly 2^32 - 1 runs, one more is refused by the weighted call and by loads()
    big = np.zeros(c.n, np.uint32)
    big[0], big[1] = U32 - 5, 5
    s.write_weights(big)
    s.assign_ranked(2)
    assert s.assign_bounded_weighted(False) >= 1
    assert int(s.loads().astype(np.int64).sum()) == U32
    assert p.assign_bounded_weighted_batch(c.keys, big)[1] >= 1
    big[2] = 1
    s.write_weights(big)
    s.assign_ranked(2)
    refused(lambda: s.assign_bounded_weighted(False), "weight sum past u32")
    refused(lambda: s.assign_bounded_weighted(True, U32), "weight sum past u32 (affinity, explicit total)")
    refused(lambda: s.loads(), "loads past u32")
    with pytest.raises(R.Unknown):
        p.assign_bounded_weighted_batch(c.keys, big)
    # NULL buffers of the batch call; n = 0 answers OK with no pass
    out = np.empty(c.n, np.uint32)
    assert L.rio_cuda_assign_bounded_weighted_batch(p.h, None, None, None, c.n, 0, 5, 4, 4, out.ctypes.data, None) != 0
    assert L.rio_cuda_assign_bounded_weighted_batch(p.h, c.keys.ctypes.data, None, None, c.n, 0, 5, 4, 4, None, None) != 0
    assert p.assign_bounded_weighted_batch(c.keys[:0])[1] == 0


# ---- two ranks -------------------------------------------------------------------------------------------------------------------
def _worker(rank, world, port, n, M, q, comm):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    os.environ["RIO_COMM"] = comm
    import torch.distributed as dist

    import rio_rs_b200 as R
    from rio_rs_b200 import parallel

    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)  # bootstrap only
    rng = np.random.default_rng(78)
    fo = rng.uniform(-1, 1, (n, 16)).astype(np.float32)
    fn = rng.uniform(-1, 1, (M, 16)).astype(np.float32)
    w = rng.integers(1, 17, M).astype(np.uint32)
    ow = weight_mix("lognormal", n, rng)
    keys = rng.integers(0, 2**63, n, dtype=np.uint64)
    p = R.GpuObjectPlacement(device=rank)
    parallel.init_comm(p, dist)
    p.set_nodes(addresses(M), w, fn)
    lo, hi = parallel.shard_range(n, rank, world)
    s = p.new_set(hi - lo)
    s.load_keys(keys[lo:hi])
    s.load_feats(fo[lo:hi])
    s.write_weights(ow[lo:hi])
    out = {}
    total = int(ow.astype(np.int64).sum())   # the same explicit total on every rank, and the default (the sum over all ranks)
    for aff in (False, True):
        for cap in CAPS:
            for lt in (0, total):
                passes = s.assign_bounded_weighted(aff, lt, cap[0], cap[1], 8)
                out[aff, cap, lt] = (passes, s.read().tolist(), s.counters().tolist(), s.loads().tolist())
    q.put((rank, lo, hi, out))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("comm", ["p2p", "nccl"])
def test_two_ranks_equal_one_rank_on_the_global_set(gp, comm):
    """Two ranks, each with one shard and its weights (the shards' weight sums differ): with load_total given as the global weight
    sum on every rank, and with it defaulted (the engine then sums the shards' weights across ranks), every shard equals the one-rank
    call on the global set, and every rank holds the global counters and loads.  Skipped with fewer than two GPUs."""
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp

    n, M, world = 200_000, 96, 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 30500 + os.getpid() % 500 + (11 if comm == "nccl" else 0)
    procs = [ctx.Process(target=_worker, args=(r, world, port, n, M, q, comm)) for r in range(world)]
    try:
        for pr in procs:
            pr.start()
        res = sorted(q.get(timeout=600) for _ in range(world))
        for pr in procs:
            pr.join(timeout=120)
    finally:   # a worker that failed or got stuck must not outlive the test
        for pr in procs:
            if pr.is_alive():
                pr.kill()
                pr.join(timeout=30)
    rng = np.random.default_rng(78)
    fo = rng.uniform(-1, 1, (n, 16)).astype(np.float32)
    fn = rng.uniform(-1, 1, (M, 16)).astype(np.float32)
    w = rng.integers(1, 17, M).astype(np.uint32)
    ow = weight_mix("lognormal", n, rng)
    keys = rng.integers(0, 2**63, n, dtype=np.uint64)
    p = gp.GpuObjectPlacement()
    p.set_nodes(addresses(M), w, fn)
    s = p.new_set(n)
    s.load_keys(keys)
    s.load_feats(fo)
    s.write_weights(ow)
    total = int(ow.astype(np.int64).sum())
    for aff in (False, True):
        for cap in CAPS:
            for lt in (0, total):
                passes = s.assign_bounded_weighted(aff, lt, cap[0], cap[1], 8)
                idx, cnt, ld = s.read().tolist(), s.counters().tolist(), s.loads().tolist()
                for _, lo, hi, out in res:
                    assert out[aff, cap, lt] == (passes, idx[lo:hi], cnt, ld), (aff, cap, lt)


# ---- host-sim --------------------------------------------------------------------------------------------------------------------
DOUBLES = os.path.join(ROOT, "tests", "cpp", "hostsim", "bounded_weighted_launchers.cpp")
OTHER_DOUBLES = [os.path.join(ROOT, "tests", "cpp", "hostsim", f) for f in ("ranked_launchers.cpp", "change_launchers.cpp", "ranked_change_launchers.cpp",
                                                                              "spread_launchers.cpp", "spread_change_launchers.cpp",
                                                                              "affinity_ranked_launchers.cpp", "affinity_spread_launchers.cpp",
                                                                              "affinity_set_launchers.cpp", "affinity_bounded_launchers.cpp",
                                                                              "set_bounded_affinity_launchers.cpp", "set_churn_launchers.cpp")]


def test_the_doubles_cover_the_new_launchers():
    decl = set(re.findall(r"\b(launch_[a-z0-9_]+)\s*\(", open(os.path.join(ROOT, "rio_rs_b200", "csrc", "k_bounded_weighted.cuh")).read()))
    have = set(re.findall(r"^void\s+([a-z0-9_]+)\s*\(", open(DOUBLES).read(), flags=re.M))
    assert len(decl) == 5 and decl <= have, decl - have


def _hostsim_library(HS, name, doubles):
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, name)
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + doubles + ["-o", so, "-ldl", "-lpthread"])
    return so


def test_bounded_weighted_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + every double, the new one
    included)."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_bounded_weighted.so", OTHER_DOUBLES + [DOUBLES])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider",
           "-k", "not two_ranks"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=3000, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 50 and "failed" not in r.stdout, tail


@pytest.mark.parametrize("world", [2, 4])
def test_ranks_with_unequal_shard_weights_equal_one_rank_on_the_host_logic(world):
    """tests/hostsim_multirank_weighted.py: `world` ranks as threads of one process over the host-sim library, each shard with its own
    weight sum.  Defaulted and explicit load_total give every rank the one-rank result, and a weight total past 2^32 - 1 that no shard
    reaches alone is refused on every rank."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_bounded_weighted_mr.so", OTHER_DOUBLES + [DOUBLES])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "hostsim_multirank_weighted.py"), str(world)], capture_output=True, text=True,
                       timeout=900, env=env, cwd=ROOT)
    assert r.returncode == 0 and "multirank weighted ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


def test_the_weighted_calls_report_an_error_where_their_kernels_are_not_linked():
    """The engine's host code built WITHOUT the new launchers loads and refuses the weighted calls, set_loads and erase on a set with
    a weight column with RIO_ERR_UPSTREAM; the weight column's own calls, erase on a set without one and every other call keep
    working."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    so = _hostsim_library(HS, "librio_cuda_hostsim_no_bounded_weighted.so", OTHER_DOUBLES)
    code = (
        "import sys, numpy as np\n"
        "from rio_rs_b200 import _native as N\n"
        "N.library_path = lambda: sys.argv[1]\n"
        "import rio_rs_b200 as R\n"
        "p = R.GpuObjectPlacement()\n"
        "p.set_nodes(['10.0.0.%d:5000' % j for j in range(8)])\n"
        "keys = np.arange(100, dtype=np.uint64)\n"
        "s = p.new_set(200); s.load_keys(keys); s.assign_bounded(0, 5, 4, 4)\n"
        "assert s.erase(keys[90:]) == 10 and s.insert(keys[90:]) == 90\n"
        "s.write_weights(np.arange(100, dtype=np.uint32))\n"
        "assert (s.read_weights() == np.arange(100)).all()\n"
        "assert s.insert(keys[:2] + 1000) == 100 and (s.read_weights(100) == 1).all()\n"
        "calls = (lambda: s.assign_bounded_weighted(), lambda: s.loads(), lambda: s.erase(keys[:3]),\n"
        "         lambda: p.assign_bounded_weighted_batch(keys))\n"
        "for call in calls:\n"
        "    try:\n"
        "        call()\n"
        "        raise SystemExit('ran without kernels')\n"
        "    except R.Upstream as e:\n"
        "        assert 'weighted bounded kernels' in str(e), e\n"
        "assert s.size() == 102 and (s.read_weights()[:100] == np.arange(100)).all()\n"
        "assert s.assign_bounded(0, 5, 4, 4) >= 1 and (s.counters().sum() == 102)\n"
        "s.load_keys(keys)\n"
        "assert s.erase(keys[:3]) == 3\n"
        "print('refused ok')\n"
    )
    r = subprocess.run([sys.executable, "-c", code, so], capture_output=True, text=True, timeout=300, cwd=HS.ROOT)
    assert r.returncode == 0 and "refused ok" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]

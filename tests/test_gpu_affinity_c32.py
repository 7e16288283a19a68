"""Every affinity kernel against the exact fp32 reference of tests/affinity_c32_ref.c (DESIGN.md 3.6), on inputs built to sit where
fp32 kernels go wrong: exact c32 ties that fp64 separates, pairs whose c32 order is the opposite of their fp64 order, cancellation,
signed zeros, twins on every boundary the launchers branch on, magnitudes from 2^-40 to 2^40, and near-ties that a plain bf16
product gets wrong.

* CUDA cores (RIO_AFFINITY_VARIANT=ffma, and K = 16 past the tensor-core limit): assign_batch, ObjectSet.assign(True), the ranked and
  failure-domain lists at ranks 1..8 and the affinity resident sets after every change set equal the reference bit for bit.
* Tensor cores (K = 16, padded live count <= 2304): T1, rank 1 is the exact (c32, j) minimum of its own group of 8 positions and ranks
  2.. are strictly increasing in (c32, j); T2, every rank is within beta of the reference conditioned on the engine's earlier ranks,
  and equal to it wherever the gap exceeds that bound; T3, rank 1 equals the CUDA cores' wherever the rank-1 gap exceeds the bound.
* The fixtures are seeded and check their own construction with the reference; test_fixtures_catch_every_mutant shows that each
  plausible way of computing the cost wrongly changes at least one row the tests above demand exactly.

The CPU test at the end runs this module's GPU bodies, unchanged, against the host-sim library (engine.cu with every affinity double);
there the tensor-core path is never selected."""
import functools
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import affinity_c32_ref as REF

NONE = REF.NONE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
K_TC = 16
# DESIGN.md 3.6: the bf16 split drops ml, lm and ll (<= 2^-22 S with the split's own rounding), the wgmma accumulator adds 6 K exact
# bf16 products in fp32 in an unspecified order (<= 6 K 2^-23 (1 + 2^-7) S under any faithful rounding), and c32 itself is K
# rounded fmaf steps (<= K 2^-24 S).
BETA = 2.0**-22 + 6 * K_TC * 2.0**-23 * (1 + 2.0**-7) + K_TC * 2.0**-24
MEASURED = {}   # largest |c32(got) - c32(ref)| / (S_got + S_ref) seen by T2, per test


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


def tensor_cores(p, K, n_live):
    padded = 64 if n_live <= 64 else (n_live + 255) // 256 * 256
    return K == 16 and 0 < padded <= 2304 and not host_sim(p)


# ---- fixtures ----------------------------------------------------------------------------------------------------------------------
class Fix:
    """Object rows, node rows, the live mask and failure-domain labels (NONE: a domain of its own) of one hard input."""

    def __init__(self, name, fo, fn, live=None, dom=None):
        self.name, self.fo, self.fn = name, np.ascontiguousarray(fo, np.float32), np.ascontiguousarray(fn, np.float32)
        M = len(self.fn)
        self.live = np.ones(M, bool) if live is None else np.asarray(live, bool)
        self.dom = (np.arange(M, dtype=np.uint32) // 8 + 1000) if dom is None else np.asarray(dom, np.uint32)

    @property
    def K(self):
        return self.fn.shape[1]


def _strong(rng, fn, pairs):
    """the pairs' first nodes get components of magnitude 1.5 to 2 (the other nodes have at most 1), so that objects close to them
    see the pair at ranks 1 and 2 at small K too"""
    for a, _ in pairs:
        fn[a] = (np.where(fn[a] < 0, -1, 1) * rng.uniform(1.5, 2, fn.shape[1])).astype(np.float32)


def _aligned(rng, fn, pairs, n, noise):
    """n object rows, each close to the first node of one of the pairs, so that the pair competes for rank 1"""
    who = np.arange(n) % len(pairs)
    a = np.array([p[0] for p in pairs])[who]
    return (fn[a] + noise * rng.uniform(-1, 1, (n, fn.shape[1]))).astype(np.float32), who


def _dot64(fo, fn):
    return np.asarray(fo, np.float64) @ np.asarray(fn, np.float64).T


@functools.lru_cache(maxsize=None)
def ulp_twins(K, seed=1):
    """Node b is node a with component k* one ulp larger; every object's feature k* is positive and about 2^-20, so the product change
    is absorbed in c32 (an exact tie, the lower index first) while fp64 puts b first."""
    assert K >= 2
    rng = np.random.default_rng(seed)
    M, n = 96, 1536
    fn = rng.uniform(-1, 1, (M, K)).astype(np.float32)
    pairs = [(a, a + 37) for a in range(3, 51, 6)]
    _strong(rng, fn, pairs)
    ks = [int(x) for x in rng.integers(0, K, len(pairs))]
    fo, who = _aligned(rng, fn, pairs, n, 0.05)
    for (a, b), k in zip(pairs, ks):
        fn[b] = fn[a]
        fn[b, k] = np.nextafter(fn[a, k], np.float32(np.inf))
    fo[np.arange(n), np.array(ks)[who]] = rng.uniform(0.5, 1, n).astype(np.float32) * np.float32(2.0**-20)
    f = Fix("ulp twins K=%d" % K, fo, fn)
    c, d = REF.c32(fo, fn), _dot64(fo, fn)
    a = np.array([p[0] for p in pairs])[who]
    b = np.array([p[1] for p in pairs])[who]
    r = np.arange(n)
    tie = (c[r, a] == c[r, b]) & (d[r, b] > d[r, a]) & (REF.ranked(fo, fn, f.live, 2) == np.stack([a, b], 1)).all(1)
    assert tie.sum() >= n // 2, ("the c32 ties did not happen", int(tie.sum()))
    return f


@functools.lru_cache(maxsize=None)
def order_flips(K, seed=2):
    """Near-twins (a few components of b one or two ulps away from a's) and objects close to a: a seeded search keeps the node
    table in which the most rows see a and b in opposite c32 and fp64 orders."""
    best = None
    for s in range(8):
        rng = np.random.default_rng(1000 * seed + s)
        M, n = 80, 1200
        fn = rng.uniform(-1, 1, (M, K)).astype(np.float32)
        pairs = [(a, a + 29) for a in range(2, 42, 5)]
        _strong(rng, fn, pairs)
        for a, b in pairs:
            fn[b] = fn[a]
            for k in rng.choice(K, max(2, K // 3), replace=False):   # fmaf is monotone: one nudged product cannot flip the order
                for _ in range(int(rng.integers(1, 3))):
                    fn[b, k] = np.nextafter(fn[b, k], np.float32(np.inf if rng.integers(2) else -np.inf))
        fo, who = _aligned(rng, fn, pairs, n, 0.3)
        c, d = REF.c32(fo, fn), _dot64(fo, fn)
        r = np.arange(n)
        a = np.array([p[0] for p in pairs])[who]
        b = np.array([p[1] for p in pairs])[who]
        flips = int(((c[r, b] < c[r, a]) & (d[r, b] < d[r, a]) | (c[r, b] > c[r, a]) & (d[r, b] > d[r, a])).sum())   # cost = -dot
        if best is None or flips > best[0]:
            best = (flips, Fix("order flips K=%d" % K, fo, fn))
    assert best[0] >= 10, ("too few order flips", best[0])
    return best[1]


@functools.lru_cache(maxsize=None)
def cancellation(K, seed=3):
    """Features 0 and 1 of every node are +-1e4 (they cancel for objects whose first two features are equal), next to O(1) terms that
    differ between nodes by about one ulp of 1e4: the summation order decides the argmin."""
    assert K >= 3
    rng = np.random.default_rng(seed)
    M, n = 64, 1024
    fn = np.empty((M, K), np.float32)
    big = rng.uniform(0.9e4, 1.1e4, M).astype(np.float32)
    fn[:, 0] = big
    fn[:, 1] = -big + 2e-3 * rng.uniform(-1, 1, M).astype(np.float32)
    fn[:, 2:] = rng.uniform(-1, 1, K - 2).astype(np.float32) + 2e-3 * rng.uniform(-1, 1, (M, K - 2)).astype(np.float32)
    fo = rng.uniform(-1, 1, (n, K)).astype(np.float32)
    fo[:, 0] = rng.uniform(0.5, 1.5, n).astype(np.float32)
    fo[:, 1] = fo[:, 0]
    f = Fix("cancellation K=%d" % K, fo, fn)
    r1 = REF.ranked(fo, fn, f.live, 1)
    assert (REF.ranked(fo, fn, f.live, 1, REF.MUTANTS["reversed k order"]) != r1).sum() >= 10, "the summation order decides nothing"
    return f


T0 = np.float32(2.0**-80)


def signed_zero_nodes(M, a, b):
    """Node a's costs are +0 and node b's -0 for every object of signed_zero (products of 2^-80 and 2^-80 underflow); every other node
    costs more than 0.  a < b: the CUDA cores list a first."""
    rng = np.random.default_rng(M + a + b)
    fn = -rng.uniform(0.5, 1, (M, 16)).astype(np.float32)
    fn[a] = T0
    fn[a, 15] = -T0
    fn[b] = T0
    return fn


@functools.lru_cache(maxsize=None)
def signed_zero(M, a, b):
    fo = np.repeat(T0 * np.float32(2.0) ** -np.arange(4, dtype=np.float32)[:, None], 16, axis=1).astype(np.float32)
    fo = np.tile(fo, (64, 1))
    fn = signed_zero_nodes(M, a, b)
    f = Fix("signed zero M=%d a=%d b=%d" % (M, a, b), fo, fn, dom=np.full(M, NONE, np.uint32))
    c = REF.c32(fo, fn)
    assert (c[:, a] == 0).all() and not np.signbit(c[:, a]).any() and np.signbit(c[:, b]).all(), "no signed-zero tie"
    assert ((c[:, a] == c[:, b]) & (np.delete(c, [a, b], axis=1) > 0).all(axis=1)).all()
    assert (REF.ranked(fo, fn, f.live, 2) == [a, b]).all()
    return f


@functools.lru_cache(maxsize=None)
def boundary_twins(M, twins, dead=(), seed=4):
    """Exact twins (identical rows, so identical c32 at any K) at the given interned indices, with `dead` nodes not live; objects
    close to the twins.  The lower index comes first; in failure-domain lists the twins are in domains of their own."""
    rng = np.random.default_rng(seed + M)
    fn = rng.uniform(-1, 1, (M, 16)).astype(np.float32)
    _strong(rng, fn, twins)
    for a, b in twins:
        fn[b] = fn[a]
    live = np.ones(M, bool)
    live[list(dead)] = False
    fo, _ = _aligned(rng, fn, twins, 1024, 0.1)
    dom = np.arange(M, dtype=np.uint32) // 8 + 1000
    for a, b in twins:
        dom[a], dom[b] = NONE, NONE
    f = Fix("twins M=%d %s" % (M, twins), fo, fn, live, dom)
    r = REF.ranked(fo, fn, live, 2)
    for a, b in twins:
        assert ((r[:, 0] == a) & (r[:, 1] == b)).sum() >= 50, ("twins never met", a, b)
    return f


# live positions n-1 | n of the padding steps and the group step, and interned indices 2047 | 2048 (the K = 16 CUDA-core node chunk)
# with dead nodes before and between them, so positions are not indices
BOUNDARIES = [
    (64, ((7, 8), (62, 63))),
    (65, ((63, 64), (0, 8))),
    (256, ((254, 255), (15, 16))),
    (257, ((255, 256), (7, 8))),
    (2100, ((2047, 2048), (2040, 2056)), tuple(range(100, 400)) + tuple(range(2041, 2047)) + tuple(range(2049, 2056))),
]


@functools.lru_cache(maxsize=None)
def magnitude_spread(K, seed=5):
    """Node j's features are uniform(-1, 1) * 2^e_j with e_j in [-40, 40]; objects' in [-20, 20]: every product is a normal fp32."""
    rng = np.random.default_rng(seed)
    M, n = 300, 1024
    fn = (rng.uniform(-1, 1, (M, K)) * 2.0 ** rng.integers(-40, 41, M)[:, None]).astype(np.float32)
    fo = (rng.uniform(-1, 1, (n, K)) * 2.0 ** rng.integers(-20, 21, n)[:, None]).astype(np.float32)
    fn[np.abs(fn) < 2.0**-60] = 2.0**-60
    fo[np.abs(fo) < 2.0**-40] = 2.0**-40
    assert (np.abs(fn).max(axis=1) > 2.0**35).any() and (np.abs(fn).max(axis=1) < 2.0**-35).any()
    return Fix("magnitudes K=%d" % K, fo, fn)


def tensor_rank1(cost, c32, live):
    """Rank 1 of the tensor-core path for costs `cost` of its group pick: the group (8 consecutive live positions) with the smallest
    cost, ties to the smaller group, then the (c32, position) minimum inside it."""
    lidx = np.flatnonzero(live)
    cg = cost[:, lidx]
    pad = (-len(lidx)) % 8
    grp = np.pad(cg, ((0, 0), (0, pad)), constant_values=np.inf).reshape(len(cg), -1, 8).min(axis=2)
    g = np.argmin(grp, axis=1)
    pos = g[:, None] * 8 + np.arange(8)[None, :]
    ok = pos < len(lidx)
    c = np.where(ok, np.take_along_axis(c32[:, lidx], np.minimum(pos, len(lidx) - 1), axis=1), np.inf)
    return lidx[pos[np.arange(len(c)), np.argmin(c, axis=1)]]


@functools.lru_cache(maxsize=None)
def split_has_teeth(seed=6):
    """Rows whose best-versus-second c32 gap lies in [2^-12 S, 100 beta S], the two in different groups: a plain bf16 product picks
    the wrong group on every kept row, the six-term split (exact accumulation) the right one.  Node a's components are bf16 values
    and node b's are 2^-11 to 2^-10 larger in magnitude, less than half a bf16 ulp: in bf16 the two are the same node, and a's earlier
    group wins, while b is the better node by about 2^-10.5 S."""
    rng = np.random.default_rng(seed)
    M, n = 256, 4096
    fn = rng.uniform(-1, 1, (M, 16)).astype(np.float32)
    pairs = [(16 * q, 16 * q + 8 + q % 8) for q in range(16)]
    _strong(rng, fn, pairs)
    for a, b in pairs:
        u = fn[a].view(np.uint32)
        fn[a] = ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32).view(np.float32)   # round to bf16
        fn[b] = fn[a] * (1 + rng.uniform(2.0**-11, 2.0**-10, 16)).astype(np.float32)
    fo, _ = _aligned(rng, fn, pairs, n, 0.02)
    live = np.ones(M, bool)
    c, s = REF.c32(fo, fn), REF.S(fo, fn)
    r = REF.ranked(fo, fn, live, 2)
    i = np.arange(n)
    gap = (c[i, r[:, 1]] - c[i, r[:, 0]]).astype(np.float64)
    sb = s[i, r[:, 0]]
    keep = (gap >= 2.0**-12 * sb) & (gap <= 100 * BETA * sb) & (r[:, 0] // 8 != r[:, 1] // 8)
    keep &= tensor_rank1(REF.c32(fo, fn, REF.MUTANTS["bf16 product only"]), c, live) != r[:, 0]
    keep &= tensor_rank1(REF.c32(fo, fn, REF.SPLIT6), c, live) == r[:, 0]
    assert keep.sum() >= 64, ("too few rows where the split has teeth", int(keep.sum()))
    return Fix("split has teeth", fo[keep], fn, live)


# the inputs the CUDA-core tests demand bit for bit, K = 16 and generic K (built on first use)
EXACT = [lambda: ulp_twins(16), lambda: order_flips(16), lambda: cancellation(16), lambda: magnitude_spread(16),
         lambda: signed_zero(64, 10, 13), lambda: signed_zero(300, 10, 21)]
EXACT += [functools.partial(boundary_twins, *b) for b in BOUNDARIES]
EXACT += [functools.partial(g, K) for K in (3, 5, 8, 17, 64) for g in (ulp_twins, order_flips, cancellation)]
EXACT += [lambda: order_flips(2), lambda: magnitude_spread(1)]


def exact_fixtures():
    return [f() for f in EXACT]


# ---- checks -------------------------------------------------------------------------------------------------------------------------
def handle(gp, oracle, f):
    p = gp.GpuObjectPlacement()
    M = len(f.fn)
    p.set_nodes(oracle.synth_nodes(M)[0], None, f.fn)
    p.set_node_domains(np.arange(M, dtype=np.uint32), f.dom)
    for j in np.flatnonzero(~f.live):
        p.node_set_active(int(j), False)
    return p


def ref_list(f, R, kind, fo=None):
    fo = f.fo if fo is None else fo
    return REF.spread(fo, f.fn, f.live, f.dom, R) if kind == "spread" else REF.ranked(fo, f.fn, f.live, R)


def call(p, kind, fo, R):
    return p.assign_ranked_affinity_spread(fo, R) if kind == "spread" else p.assign_ranked_affinity(fo, R)


def assert_exact(got, want, tag):
    bad = np.flatnonzero((got != want).any(axis=1))
    assert not len(bad), (tag, len(bad), [(int(i), got[i].tolist(), want[i].tolist()) for i in bad[:3]])


def dom_ids(f):
    own = -1 - np.arange(len(f.fn), dtype=np.int64)
    lab = f.dom.astype(np.int64)
    return np.where(f.dom == NONE, own, lab)


def tensor_checks(f, got, kind, tag):
    """T1 and T2 for an (n, R) tensor-core list; returns the rows whose rank-1 gap exceeds the T2 bound"""
    n, R = got.shape
    c, s = REF.c32(f.fo, f.fn), REF.S(f.fo, f.fn)
    lidx = np.flatnonzero(f.live)
    pos = np.full(len(f.fn), -1, np.int64)
    pos[lidx] = np.arange(len(lidx))
    rows = np.arange(n)
    d = dom_ids(f)
    n_dom = len(np.unique(d[lidx]))
    depth = min(R, len(lidx) if kind == "ranked" else n_dom)
    assert (got[:, depth:] == NONE).all() and (got[:, :depth] != NONE).all(), tag
    head = got[:, :depth].astype(np.int64)
    assert f.live[head].all(), tag
    if kind == "spread":
        for a in range(depth):
            for b in range(a + 1, depth):
                assert (d[head[:, a]] != d[head[:, b]]).all(), (tag, "two ranks in one domain")
    else:
        for a in range(depth):
            for b in range(a + 1, depth):
                assert (head[:, a] != head[:, b]).all(), (tag, "a node listed twice")
    # T1: rank 1 is the (c32, j) minimum of the live nodes of its own group
    g0 = pos[head[:, 0]] // 8
    gpos = g0[:, None] * 8 + np.arange(8)[None, :]
    ok = gpos < len(lidx)
    gj = lidx[np.minimum(gpos, len(lidx) - 1)]
    gc = np.where(ok, c[rows[:, None], gj], np.inf)
    want1 = gj[rows, np.argmin(gc, axis=1)]
    bad = np.flatnonzero(want1 != head[:, 0])
    assert not len(bad), (tag, "T1: rank 1 is not its group's c32 minimum", [(int(i), int(head[i, 0]), int(want1[i])) for i in bad[:3]])
    # ... and ranks 2.. strictly increase in (c32, j)
    for r in range(1, depth - 1):
        ca, cb = c[rows, head[:, r]], c[rows, head[:, r + 1]]
        assert ((ca < cb) | (ca == cb) & (head[:, r] < head[:, r + 1])).all(), (tag, "T1: ranks out of (c32, j) order", r)
    # T2: each rank against the reference conditioned on the engine's earlier ranks.  S_got is the largest S of the groups the row's
    # list came from: the tensor core compares groups by their best column, which need not be the node the fp32 re-cost keeps.
    hg = pos[head] // 8
    s_grp = np.zeros(n)
    for r in range(depth):
        gp_ = hg[:, r][:, None] * 8 + np.arange(8)[None, :]
        okr = gp_ < len(lidx)
        s_grp = np.maximum(s_grp, np.where(okr, s[rows[:, None], lidx[np.minimum(gp_, len(lidx) - 1)]], 0).max(axis=1))
    excluded = np.zeros(c.shape, bool)
    excluded[:, ~f.live] = True
    worst, clear1 = 0.0, None
    for r in range(depth):
        cm = np.where(excluded, np.inf, c).astype(np.float64)
        ref = np.argmin(cm, axis=1)
        best = cm[rows, ref]
        cm[rows, ref] = np.inf
        gap = cm.min(axis=1) - best
        g = head[:, r]
        delta = c[rows, g].astype(np.float64) - best
        bound = BETA * (np.maximum(s[rows, g], s_grp) + s[rows, ref])
        worst = max(worst, float((np.abs(delta) / (s[rows, g] + s[rows, ref] + 1e-300)).max()))
        over = np.flatnonzero(np.abs(delta) > bound)
        assert not len(over), (tag, "T2: rank %d off by more than beta" % r, [(int(i), int(g[i]), int(ref[i])) for i in over[:3]])
        wrong = np.flatnonzero((gap > bound) & (g != ref))
        assert not len(wrong), (tag, "T2: rank %d differs where the gap is clear" % r, [(int(i), int(g[i]), int(ref[i])) for i in wrong[:3]])
        if r == 0:
            clear1 = gap > bound
        if kind == "spread":
            excluded |= d[None, :] == d[g][:, None]
        else:
            excluded[rows, g] = True
    MEASURED[tag] = max(MEASURED.get(tag, 0.0), worst)
    return clear1


# ---- CUDA cores: the whole list, bit for bit -------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fi", range(len(EXACT)))
def test_cuda_cores_equal_the_reference(gp, oracle, fi):
    """assign_batch, ObjectSet.assign(True) and both list kinds at ranks 1..8 equal the reference exactly (ffma)."""
    f = EXACT[fi]()
    p = handle(gp, oracle, f)
    want8 = {k: ref_list(f, 8, k) for k in ("ranked", "spread")}
    with variant("ffma"):
        assert (p.assign_batch(obj_feats=f.fo) == want8["ranked"][:, 0]).all(), f.name
        s = p.new_set(len(f.fo))
        s.synth_keys(0, len(f.fo), 3)
        s.load_feats(f.fo)
        s.assign(True)
        assert (s.read() == want8["ranked"][:, 0]).all(), f.name
        for kind in ("ranked", "spread"):
            for R in range(1, 9):
                want = want8[kind][:, :R] if kind == "ranked" else ref_list(f, R, kind)
                assert_exact(call(p, kind, f.fo, R), want, (f.name, kind, R))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ranked", "spread"])
def test_cuda_cores_above_the_tensor_core_limit(gp, oracle, kind):
    """K = 16 with 2400 live nodes runs on the CUDA cores on the default path; near-twins spread over the whole table."""
    rng = np.random.default_rng(9)
    M = 2400
    fn = rng.uniform(-1, 1, (M, 16)).astype(np.float32)
    pairs = [(a, a + 1031) for a in range(5, 1300, 97)]
    _strong(rng, fn, pairs)
    for a, b in pairs:
        fn[b] = fn[a]
        fn[b, a % 16] = np.nextafter(fn[a, a % 16], np.float32(np.inf))
    fo, _ = _aligned(rng, fn, pairs, 3000, 0.05)
    f = Fix("2400 live", fo, fn)
    p = handle(gp, oracle, f)
    assert not tensor_cores(p, 16, M)
    assert (p.assign_batch(obj_feats=fo) == ref_list(f, 1, "ranked")[:, 0]).all()
    for R in (1, 3, 8):
        assert_exact(call(p, kind, fo, R), ref_list(f, R, kind), (kind, R))


class ExactSet:
    """An affinity resident set on the CUDA cores whose node table is mirrored here; every state is compared with the reference."""

    def __init__(self, gp, oracle, f, R, kind):
        self.f = Fix(f.name, f.fo, f.fn.copy(), f.live.copy(), f.dom.copy())
        self.R, self.kind = R, kind
        M = len(f.fn)
        self.addrs = oracle.synth_nodes(M)[0]
        self.w = np.full(M, 2, np.uint32)
        self.p = handle(gp, oracle, self.f)
        self.s = self.p.new_set(len(f.fo))
        self.s.synth_keys(0, len(f.fo), 5)
        self.s.load_feats(f.fo)
        with variant("ffma"):
            (self.s.assign_ranked_affinity_spread if kind == "spread" else self.s.assign_ranked_affinity)(R)
        self.check("assign")

    def check(self, tag):
        self.cur = self.s.read_ranked()
        assert_exact(self.cur, ref_list(self.f, self.R, self.kind), (self.f.name, self.kind, tag))
        assert (self.s.read() == self.cur[:, 0]).all(), tag

    def step(self, idx, prev, tag):
        self.s.rebalance_changes_ranked(idx, prev)
        self.check(tag)

    def leave(self, js):
        prev = [int(self.w[j]) if self.f.live[j] else 0 for j in js]
        for j in js:
            self.p.node_set_active(int(j), False)
            self.f.live[j] = False
        self.step(list(js), prev, "leave %d" % len(js))

    def join(self, js):
        prev = [int(self.w[j]) if self.f.live[j] else 0 for j in js]
        for j in js:
            self.p.node_upsert(self.addrs[j], int(self.w[j]))
            self.f.live[j] = True
        self.step(list(js), prev, "join %d" % len(js))

    def reweight(self, js):
        prev = [int(self.w[j]) for j in js]
        for j in js:
            self.w[j] += 3
            self.p.node_upsert(self.addrs[j], int(self.w[j]))
        self.step(list(js), prev, "weights")

    def refeature(self, j, row, tag):
        self.f.fn[j] = row
        self.p.node_upsert(self.addrs[j], int(self.w[j]), self.f.fn[j])
        self.step([], [], tag)


def listed_pair(es, col):
    """(row i, listed node y, unlisted node z) with z < y, so a copy of y's row at z goes before y"""
    for i in range(len(es.cur)):
        y = int(es.cur[i, col])
        zs = [z for z in range(y) if z not in es.cur[i] and es.f.live[z]]
        if y != NONE and zs:
            return i, y, zs[-1]
    raise AssertionError("no listed member with an unlisted lower index")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ranked", "spread"])
@pytest.mark.parametrize("R", [1, 3, 8])
def test_resident_sets_equal_the_reference(gp, oracle, kind, R):
    """Leaves, joins, a weight-only change, a rack leaving, a refeature into an exact c32 tie with a listed member and one into an
    order flip against it: after every change set the lists equal the reference over the current live set, features and labels."""
    f = ulp_twins(16)
    es = ExactSet(gp, oracle, f, R, kind)
    busy = int(np.bincount(es.cur[:, 0].astype(np.int64)).argmax())
    es.leave([busy])
    es.join([busy])
    es.reweight([1, 2, busy])
    rack = [int(j) for j in np.flatnonzero(es.f.dom == es.f.dom[busy])]
    es.leave(rack)
    es.join(rack[:3])
    # an exact tie: z < y gets y's row, so z goes right before y wherever y was listed
    i, y, z = listed_pair(es, min(R, 2) - 1)
    es.refeature(z, es.f.fn[y].copy(), "exact tie")
    assert REF.c32(f.fo[i:i + 1], es.f.fn[[y, z]])[0].tolist() == REF.c32(f.fo[i:i + 1], es.f.fn[[z, y]])[0].tolist()[::-1]
    # an order flip: z's row becomes a near-twin of the rank-1 node whose c32 and fp64 orders against it disagree on some rows
    y = int(es.cur[0, 0])
    z = max(j for j in range(len(es.f.fn)) if es.f.live[j] and j not in es.cur[:, 0] and j != y)
    rows = np.flatnonzero(es.cur[:, 0] == y)
    best = None
    for t in range(40):
        rng = np.random.default_rng(t)
        cand = es.f.fn[y].copy()
        for k in rng.choice(16, 5, replace=False):
            cand[k] = np.nextafter(cand[k], np.float32(np.inf if rng.integers(2) else -np.inf))
        c = REF.c32(f.fo[rows], np.stack([es.f.fn[y], cand]))
        d = _dot64(f.fo[rows], np.stack([es.f.fn[y], cand]))
        flips = int(((c[:, 1] < c[:, 0]) & (d[:, 1] < d[:, 0]) | (c[:, 1] > c[:, 0]) & (d[:, 1] > d[:, 0])).sum())
        if best is None or flips > best[0]:
            best = (flips, cand)
    assert best[0] > 0, "no order flip found"
    es.refeature(z, best[1], "order flip")
    es.leave([int(j) for j in np.flatnonzero(es.f.live)][: len(es.f.fn) // 2])


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["ranked", "spread"])
def test_resident_set_candidates_on_both_sides_of_the_staging_budget(gp, oracle, kind):
    """K = 64, 1000 interned nodes: 300 candidates are staged in shared memory (300 (4K + 4) + 1000 B <= 96 KB), 400 are not."""
    f = order_flips(64)
    rng = np.random.default_rng(3)
    M = 1000
    fn = rng.uniform(-1, 1, (M, 64)).astype(np.float32)
    fn[: len(f.fn)] = f.fn
    es = ExactSet(gp, oracle, Fix("K=64 staging", f.fo[:600], fn), 4, kind)
    out = list(range(500, 900))
    es.leave(out)
    es.join(out[:300])
    es.leave(out[:300])
    es.join(out)


# ---- tensor cores ----------------------------------------------------------------------------------------------------------------
TENSOR = [lambda: ulp_twins(16), lambda: order_flips(16), lambda: cancellation(16), lambda: magnitude_spread(16), split_has_teeth]
TENSOR += [functools.partial(boundary_twins, *b) for b in BOUNDARIES]


@pytest.mark.gpu
@pytest.mark.parametrize("fi", range(len(TENSOR)))
def test_tensor_cores_t1_t2_t3(gp, oracle, fi):
    """T1 and T2 for assign_batch and both list kinds at R = 1, 3, 4, 8; T3: rank 1 equals the CUDA cores' wherever the rank-1 gap
    exceeds the T2 bound, on every row of the split-has-teeth set."""
    f = TENSOR[fi]()
    p = handle(gp, oracle, f)
    assert tensor_cores(p, 16, int(f.live.sum())) == (not host_sim(p))
    with variant("ffma"):
        cuda = p.assign_batch(obj_feats=f.fo)
    assert (cuda == ref_list(f, 1, "ranked")[:, 0]).all()
    with variant("umma"):
        one = p.assign_batch(obj_feats=f.fo)
        clear = tensor_checks(f, one[:, None], "ranked", f.name)
        wrong = np.flatnonzero(clear & (one != cuda))
        assert not len(wrong), ("T3", [(int(i), int(one[i]), int(cuda[i])) for i in wrong[:3]])
        if f.name == "split has teeth":
            assert clear.all() and (one == cuda).all()
        for kind in ("ranked", "spread"):
            for R in (1, 3, 4, 8):
                got = call(p, kind, f.fo, R)
                assert (got[:, 0] == one).all(), (kind, R)
                tensor_checks(f, got, kind, f.name)


@pytest.mark.gpu
@pytest.mark.parametrize("M,a,b", [(64, 10, 13), (300, 10, 13), (64, 10, 21), (300, 250, 290)])
def test_signed_zero_ties_go_to_the_lower_index(gp, oracle, M, a, b):
    """c32 is +0 for node a and -0 for node b; they are equal, so a < b comes first on both paths and in all three resolve kernels,
    whether a and b share a group of 8 or not."""
    f = signed_zero(M, a, b)
    p = handle(gp, oracle, f)
    for var in ("ffma", "umma"):
        with variant(var):
            assert (p.assign_batch(obj_feats=f.fo) == a).all(), var
            for kind in ("ranked", "spread"):
                for R in (2, 3, 8):
                    assert_exact(call(p, kind, f.fo, R), ref_list(f, R, kind), (var, kind, R))


@pytest.mark.gpu
def test_report_t2(gp):
    """Prints the largest |c32(got) - c32(ref)| / (S_got + S_ref) T2 met in this run, next to beta."""
    p = gp.GpuObjectPlacement()
    print("\nT2 on %s: beta = %.3e, largest |dc|/(S_got + S_ref) = %s" % (p.device_info()["name"], BETA,
                                                                          max(MEASURED.values()) if MEASURED else "not measured"))
    for k, v in sorted(MEASURED.items()):
        print("  %-40s %.3e" % (k, v))


# ---- CPU ---------------------------------------------------------------------------------------------------------------------------
def test_fixtures_catch_every_mutant():
    """Each mutant cost changes at least one list on the fixtures the CUDA-core tests demand bit for bit; the bf16-only product
    also changes the tensor path's rank 1 on the split-has-teeth rows, where T3 demands it exactly."""
    caught = {m: [] for m in REF.MUTANTS}
    for f in exact_fixtures():
        for kind in ("ranked", "spread"):
            want = ref_list(f, 8, kind)
            for m, mode in REF.MUTANTS.items():
                lists = REF.spread if kind == "spread" else REF.ranked
                got = lists(f.fo, f.fn, f.live, f.dom, 8, mode) if kind == "spread" else lists(f.fo, f.fn, f.live, 8, mode)
                rows = int((got != want).any(axis=1).sum())
                if rows:
                    caught[m].append("%s/%s: %d" % (f.name, kind, rows))
    t = split_has_teeth()
    c = REF.c32(t.fo, t.fn)
    want = REF.ranked(t.fo, t.fn, t.live, 1)[:, 0]
    teeth = int((tensor_rank1(REF.c32(t.fo, t.fn, REF.MUTANTS["bf16 product only"]), c, t.live) != want).sum())
    assert teeth == len(t.fo)
    caught["bf16 product only"].append("split has teeth (tensor rank 1): %d" % teeth)
    print()
    for m, where in caught.items():
        print("%-28s %s" % (m, "; ".join(where)))
    assert all(caught.values()), [m for m, w in caught.items() if not w]


HOSTSIM_DOUBLES = [os.path.join(ROOT, "tests", "cpp", "hostsim", f) for f in ("ranked_launchers.cpp", "change_launchers.cpp", "ranked_change_launchers.cpp",
                                                                                "spread_launchers.cpp", "spread_change_launchers.cpp", "affinity_ranked_launchers.cpp",
                                                                                "affinity_spread_launchers.cpp", "affinity_set_launchers.cpp")]


def test_bodies_on_the_engine_host_logic():
    """This module's GPU bodies, unchanged, against the host-sim library (engine.cu + tests/cpp/hostsim/ + every affinity double):
    the doubles must compute c32 for the CUDA-core bodies to pass."""
    import test_engine_host_sim as HS

    if HS.GXX is None:
        pytest.skip("no host C++ compiler")
    os.makedirs(HS.OUT, exist_ok=True)
    so = os.path.join(HS.OUT, "librio_cuda_hostsim_affinity_c32.so")
    subprocess.check_call([HS.GXX, "-std=c++17", "-O2", "-g", "-fPIC", "-shared", "-Wall", "-Wextra", "-Werror", "-I" + HS.SIM, "-x", "c++"] + HS.PRODUCT +
                          HS.DOUBLES + HOSTSIM_DOUBLES + ["-o", so, "-ldl", "-lpthread"])
    env = dict(os.environ)
    env["RIO_HOSTSIM_LIBRARY"] = so
    env["PYTHONPATH"] = os.path.join(HS.ROOT, "tests") + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-p", "hostsim_plugin", "-q", "-x", "-p", "no:cacheprovider"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=3000, env=env, cwd=HS.ROOT)
    tail = (r.stdout + r.stderr)[-3000:]
    assert r.returncode == 0, tail
    m = re.search(r"(\d+) passed", r.stdout)
    assert m and int(m.group(1)) >= 50 and "failed" not in r.stdout, tail

"""Excluded points per query (include/hnsw_b200.h "Excluded points per query"): Hnsw.search_flat_excluding and
search_exact_excluding.

Row i must equal, bit for bit, the single-filter call on query i with a resident filter made for that row, admitting
exactly the points its restriction admits minus its list (ids, distance bits, internal ids, PointIds, counts, and with
statistics on the traversal counters).  A row with an empty list must equal the call for its restriction alone, which
for an unrestricted row is the unfiltered search that follows the tie mode.  The graphs are built with default ids, so
that an origin id (what a resident filter is made of) is the insertion rank (what a list holds), also on partitioned
handles."""
import ctypes as C

import numpy as np
import pytest
import torch  # imported first, so that torch's own NCCL is the one the library binds at run time

from answers import same, stats_sum
from graphs import data
from restrict import lists_for
from util import oracle_layers

pytestmark = pytest.mark.gpu

N, M, EFC = 1500, 8, 64
NONE = 0xFFFFFFFF
RANGE_ALL = (-(1 << 63), (1 << 63) - 1)
GRID = [(k, ef) for k in (1, 10, 64) for ef in (k, 64, 200)]
GRAPHS = [(np.float32, "DistL2", 48), (np.float32, "DistCosine", 100), (np.uint8, "DistHamming", 100)]


def build(pkg, po, dtype, metric, d, seed):
    """an oracle graph (MODE_DET, ORDER_GPU, default ids: origin id = insertion rank) imported into the engine"""
    X = data(dtype, metric, N, d, seed)
    o = po.Oracle(M, N, 16, EFC, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X)
    lv, rk, og = o.export_points()
    assert np.array_equal(og, np.arange(N))
    h = pkg.Hnsw(M, N, 16, EFC, metric, dtype=dtype)
    h.import_graph(X, og, lv, o.entry, oracle_layers(o))
    return X, h


class Reference:
    """row i of the defining calls: the unfiltered call for an unrestricted row with an empty list, else the resident
    filter call over adm[i] (None: every point) minus lists[i]; each row's filter is made once"""

    def __init__(self, h, Q, adm, lists, n=N):
        self.h, self.Q, self.rfs = h, Q, []
        for a, e in zip(adm, lists):
            e = np.unique(np.asarray(e, np.int64))
            if a is None and e.size == 0:
                self.rfs.append(None)
                continue
            keep = np.setdiff1d(np.arange(n) if a is None else np.asarray(a, np.int64), e)
            self.rfs.append(h.make_filter(keep.astype(np.uint64)))

    def rows(self, k, ef=None, exact=False):
        parts = []
        for i, rf in enumerate(self.rfs):
            q = self.Q[i:i + 1]
            parts.append(self.h.search_exact(q, k, filter=rf) if exact else self.h.search_flat(q, k, ef, filter=rf))
        return tuple(np.concatenate([p[j] for p in parts]) for j in range(5))

    def stats(self, k, ef):
        """the counters of the defining calls, one row after the other"""
        per = []
        for i, rf in enumerate(self.rfs):
            self.h.get_stats()
            self.h.search_flat(self.Q[i:i + 1], k, ef, filter=rf)
            per.append(self.h.get_stats())
        return stats_sum(per)

    def free(self):
        for rf in self.rfs:
            if rf is not None:
                rf.free()


@pytest.mark.parametrize("dtype,metric,d", GRAPHS, ids=[f"{np.dtype(c[0]).name}-{c[1]}" for c in GRAPHS])
def test_lists_unrestricted(pkg, po, dtype, metric, d):
    X, h = build(pkg, po, dtype, metric, d, seed=d)
    Q = data(dtype, metric, 28, d, d + 100)
    entry = int(h.export_points()[3])
    lists = lists_for(po, X, Q, metric, entry, N, 5)
    ref = Reference(h, Q, [None] * len(Q), lists)
    tidy = [np.unique(x) for x in lists]
    for k, ef in GRID:
        got = h.search_flat_excluding(Q, k, ef, lists)
        same(got, ref.rows(k, ef), f"graph k={k} ef={ef}")
        same(h.search_flat_excluding(Q, k, ef, tidy), got, f"graph k={k} ef={ef}: unsorted lists with repeats")
        assert np.all(got[4][5::7] == 0), "a list of every point leaves nothing"
    for k in (1, 10, 64):
        got = h.search_exact_excluding(Q, k, lists)
        same(got, ref.rows(k, exact=True), f"exact k={k}")
        same(h.search_exact_excluding(Q, k, tidy), got, f"exact k={k}: unsorted lists with repeats")
    # the brute-force top 20 must change the answer, and no row holds an excluded point
    plain = h.search_flat(Q, 10, 64)
    for i in range(2, len(Q), 7):
        assert set(plain[2][i, :plain[4][i]]) & set(lists[i].tolist()), f"row {i}: its top 20 were not in its answer"
    got = h.search_flat_excluding(Q, 10, 64, lists)
    for i in range(len(Q)):
        assert not set(got[2][i, :got[4][i]].tolist()) & set(lists[i].tolist()), f"row {i} holds an excluded point"
    # statistics: the batch adds what the defining calls add
    h.enable_stats(True)
    for k, ef in ((10, 64), (64, 200)):
        h.get_stats()
        h.search_flat_excluding(Q, k, ef, lists)
        s = h.get_stats()
        assert s == ref.stats(k, ef), (k, ef)
    h.enable_stats(False)
    ref.free()


def test_empty_lists_keep_kernels_and_tie_mode(pkg, po):
    X, h = build(pkg, po, np.uint8, "DistHamming", 100, seed=7)
    Q = data(np.uint8, "DistHamming", 64, 100, 8)
    empty = [[] for _ in range(len(Q))]
    h.set_tie_mode(0)
    t0 = h.search_flat(Q, 10, 64)
    h.set_tie_mode(1)
    t1 = h.search_flat(Q, 10, 64)
    assert not np.array_equal(t0[2], t1[2]), "the tie modes give the same rows: the case checks nothing"
    for tie, want in ((0, t0), (1, t1)):
        h.set_tie_mode(tie)
        for k, ef in GRID:
            w = h.search_flat(Q, k, ef)
            kw = pkg.last_kernel()
            same(h.search_flat_excluding(Q, k, ef, empty), w, f"tie {tie} k={k} ef={ef}")
            assert pkg.last_kernel() == kw, (tie, k, ef, pkg.last_kernel(), kw)
        same(h.search_flat_excluding(Q, 10, 64, (np.zeros(len(Q) + 1, np.uint64), np.zeros(0, np.uint64))), want,
             f"tie {tie}: offsets and ranks")
    # tie mode 1: rows with a list ignore it, rows without follow it
    lists = [[] if i % 2 else [int(i)] for i in range(len(Q))]
    ref = Reference(h, Q, [None] * len(Q), lists)
    same(h.search_flat_excluding(Q, 10, 64, lists), ref.rows(10, 64), "tie 1 mixed")
    same(h.search_exact_excluding(Q, 10, lists), ref.rows(10, exact=True), "tie 1 mixed exact")
    ref.free()
    h.set_tie_mode(0)


def test_mixed_restrictions(pkg, po):
    X, h = build(pkg, po, np.float32, "DistL2", 48, seed=3)
    nq = 42
    Q = data(np.float32, "DistL2", nq, 48, 4)
    rng = np.random.default_rng(9)
    lab = rng.integers(0, 5, N).astype(np.uint32)
    lab[rng.random(N) < 0.1] = NONE
    attr = rng.integers(-1000, 1000, N).astype(np.int64)
    attr[rng.random(N) < 0.05] = -(1 << 63)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    lists = lists_for(po, X, Q, "DistL2", int(h.export_points()[3]), N, 6)
    sets = [[NONE] if i % 3 == 0 else [int(i % 5), int((i * 3) % 5)] for i in range(nq)]
    ranges = [RANGE_ALL if i % 4 == 0 else (-600 + 10 * i, 400 + 5 * i) for i in range(nq)]

    def in_sets(i):
        return np.ones(N, bool) if sets[i] == [NONE] else np.isin(lab, sets[i])

    def in_range(i):
        lo, hi = ranges[i]
        return np.ones(N, bool) if ranges[i] == RANGE_ALL else (attr >= lo) & (attr <= hi) & (attr != -(1 << 63))

    def adm_of(mask_fn):
        out = []
        for i in range(nq):
            m = mask_fn(i)
            out.append(None if m is None else np.flatnonzero(m))
        return out

    cases = {
        "none": ({}, [None] * nq),
        "sets": ({"sets": sets}, adm_of(lambda i: None if sets[i] == [NONE] else in_sets(i))),
        "ranges": ({"ranges": ranges}, adm_of(lambda i: None if ranges[i] == RANGE_ALL else in_range(i))),
        "ranges and sets": ({"ranges": ranges, "sets": sets},
                            adm_of(lambda i: None if sets[i] == [NONE] and ranges[i] == RANGE_ALL
                                   else in_sets(i) & in_range(i))),
    }
    for name, (kw, adm) in cases.items():
        ref = Reference(h, Q, adm, lists)
        for k, ef in ((1, 1), (10, 64), (64, 200)):
            same(h.search_flat_excluding(Q, k, ef, lists, **kw), ref.rows(k, ef), f"{name} k={k} ef={ef}")
        same(h.search_exact_excluding(Q, 10, lists, **kw), ref.rows(10, exact=True), f"{name} exact")
        # an empty list gives the row of the restriction's own call
        empty = [[] for _ in range(nq)]
        if name == "none":
            want, wexact = h.search_flat(Q, 10, 64), h.search_exact(Q, 10)
        elif name == "sets":
            want, wexact = h.search_flat_label_sets(Q, 10, 64, sets), h.search_exact_label_sets(Q, 10, sets)
        else:
            s = kw.get("sets")
            want, wexact = h.search_flat_ranges(Q, 10, 64, ranges, sets=s), h.search_exact_ranges(Q, 10, ranges, sets=s)
        same(h.search_flat_excluding(Q, 10, 64, empty, **kw), want, f"{name}: empty lists")
        same(h.search_exact_excluding(Q, 10, empty, **kw), wexact, f"{name}: empty lists, exact")
        ref.free()
    # one resident filter for every row, with the rows' lists on top
    fadm = np.flatnonzero(rng.random(N) < 0.4)
    rf = h.make_filter(fadm.astype(np.uint64))   # origin ids are ranks
    ref = Reference(h, Q, [fadm] * nq, lists)
    for k, ef in ((10, 64), (64, 200)):
        same(h.search_flat_excluding(Q, k, ef, lists, filter=rf), ref.rows(k, ef), f"resident filter k={k}")
    same(h.search_exact_excluding(Q, 10, lists, filter=rf), ref.rows(10, exact=True), "resident filter exact")
    same(h.search_flat_excluding(Q, 10, 64, [[] for _ in range(nq)], filter=rf), h.search_flat(Q, 10, 64, filter=rf),
         "resident filter, empty lists")
    ref.free()
    rf.free()


def test_exact_against_float64(pkg, po):
    X, h = build(pkg, po, np.float32, "DistL2", 48, seed=13)
    Q = data(np.float32, "DistL2", 35, 48, 14)
    lists = lists_for(po, X, Q, "DistL2", int(h.export_points()[3]), N, 15)
    for k in (1, 10, 64):
        _, d, it, _, c = h.search_exact_excluding(Q, k, lists)
        for i in range(len(Q)):
            keep = np.setdiff1d(np.arange(N), lists[i])
            assert c[i] == min(k, keep.size), (k, i)
            if keep.size == 0:
                continue
            d64 = np.sqrt(((X[keep].astype(np.float64) - Q[i].astype(np.float64)) ** 2).sum(1))
            kth = np.sort(d64)[c[i] - 1]
            got = np.sqrt(((X[it[i, :c[i]].astype(np.int64)].astype(np.float64) - Q[i]) ** 2).sum(1))
            assert np.all(np.isin(it[i, :c[i]], keep)), (k, i)
            assert np.all(got <= kth * (1 + 1e-5) + 1e-6), (k, i, got.max(), kth)
            assert np.allclose(d[i, :c[i]], got, rtol=1e-5, atol=1e-6), (k, i)


@pytest.mark.parametrize("P", [2, 3])
def test_partitions_and_views(pkg, po, P):
    d = 48
    X = data(np.float32, "DistL2", N, d, 31)
    h = pkg.Hnsw(M, N, 16, EFC, "DistL2")
    h.partition([0] * P)
    h.insert_flat(X)
    Q =data(np.float32, "DistL2", 28, d, 32)
    lists = lists_for(po, X, Q, "DistL2", 0, N, 33)
    ref = Reference(h, Q, [None] * len(Q), lists)
    for k, ef in ((10, 64), (64, 200), (1, 1)):
        same(h.search_flat_excluding(Q, k, ef, lists), ref.rows(k, ef), f"P={P} k={k} ef={ef}")
    for k in (1, 10):
        same(h.search_exact_excluding(Q, k, lists), ref.rows(k, exact=True), f"P={P} exact k={k}")
    ref.free()
    # a view: local ids.  Its exact row is its exact row of k + |E| without E, cut to k; its graph rows hold no
    # excluded point, and with empty lists equal its own search_flat rows
    v = h.partition_view(1)
    nv = v.get_nb_point()
    rng = np.random.default_rng(P)
    loc = [np.sort(rng.choice(nv, [0, 1, 7, 40][i % 4], replace=False)) for i in range(len(Q))]
    k = 10
    _, d_, it, pid, c = v.search_exact_excluding(Q, k, loc)
    wide = v.search_exact(Q, k + 40)
    for i in range(len(Q)):
        keep = [j for j in range(wide[4][i]) if wide[2][i, j] not in set(loc[i].tolist())][:k]
        assert c[i] == len(keep) and np.array_equal(it[i, :c[i]], wide[2][i, keep]), i
        assert np.array_equal(d_[i, :c[i]].view(np.uint32), wide[1][i, keep].view(np.uint32)), i
    g = v.search_flat_excluding(Q, k, 64, loc)
    for i in range(len(Q)):
        assert not set(g[2][i, :g[4][i]].tolist()) & set(loc[i].tolist()), i
    same(v.search_flat_excluding(Q, k, 64, [[] for _ in Q]), v.search_flat(Q, k, 64), "view, empty lists")
    with pytest.raises(pkg.HnswError, match=rf"qx\[\d+\] = {nv} is not below nb_point = {nv}"):
        v.search_flat_excluding(Q[:1], k, 64, [[nv]])


def test_replicas(pkg, po):
    if torch.cuda.device_count() < 2:
        pytest.skip("replicas need two GPUs: not run")
    X, h = build(pkg, po, np.float32, "DistL2", 48, seed=21)
    Q = data(np.float32, "DistL2", 400, 48, 22)
    lists = lists_for(po, X, Q, "DistL2", 0, N, 23)
    want = h.search_flat_excluding(Q, 10, 64, lists), h.search_exact_excluding(Q, 10, lists)
    h.replicate([0, 1])
    same(h.search_flat_excluding(Q, 10, 64, lists), want[0], "replicated graph")
    same(h.search_exact_excluding(Q, 10, lists), want[1], "replicated exact")


def test_refusals(pkg, po):
    X, h = build(pkg, po, np.float32, "DistL2", 24, seed=47)
    L = h._L
    Q = data(np.float32, "DistL2", 3, 24, 48)
    p = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731

    def call(exact, off, ids, filter=-1, rg=None, so=None, sv=None, nq=3, handle=None):
        """the raw C call on answer arrays filled with a sentinel; returns (rc, message, whether they stayed)"""
        ans = [np.full((3, 10), 7, np.uint64), np.full((3, 10), 7, np.float32), np.full((3, 10), 7, np.uint32),
               np.full((3, 10, 2), 7, np.int32), np.full(3, 7, np.int32)]
        args = [handle if handle is not None else h._h, off, ids, filter, rg, so, sv, p(Q), nq, 24, 10]
        fn = L.hnsw_b200_search_exact_excluding if exact else L.hnsw_b200_search_flat_excluding
        rc = fn(*args, *([] if exact else [64]), *map(p, ans))
        return rc, pkg.last_error(), all(np.all(a == np.array(7).astype(a.dtype)) for a in ans)

    off = np.array([0, 1, 3, 3], np.uint64)
    ids = np.array([5, 9, 2], np.uint64)
    for exact in (False, True):
        assert call(exact, p(off), p(ids))[0] == 0
        rc, msg, kept = call(exact, p(off), p(ids), handle=C.c_void_p(0))
        assert rc != 0 and "NULL handle" in msg and kept
        assert call(exact, None, None, nq=0)[0] == 0
        rc, msg, kept = call(exact, None, p(ids))
        assert rc != 0 and "qx_off is NULL" in msg and kept
        rc, msg, kept = call(exact, p(off), None)
        assert rc != 0 and "qx is NULL" in msg and kept
        bad = np.array([0, 2, 1, 3], np.uint64)
        rc, msg, kept = call(exact, p(bad), p(ids))
        assert rc != 0 and "excluded list 1: qx_off[2] = 1 is below qx_off[1] = 2" in msg and kept, msg
        far = np.array([5, 9, N + 4], np.uint64)
        rc, msg, kept = call(exact, p(off), p(far))
        assert rc != 0 and f"excluded list 1: qx[2] = {N + 4} is not below nb_point = {N}" in msg and kept, msg
        rf = h.make_filter(np.arange(0, N, 2, dtype=np.uint64))
        sets_off, sets = np.array([0, 1, 2, 3], np.uint64), np.array([1, 2, 3], np.uint32)
        rc, msg, kept = call(exact, p(off), p(ids), rf.id, None, p(sets_off), p(sets))
        assert rc != 0 and "cannot be combined" in msg and kept
        bad_sets = np.array([0, 2, 1, 3], np.uint64)
        rc, msg, kept = call(exact, p(off), p(ids), -1, None, p(bad_sets), p(sets))
        assert rc != 0 and "label set 1" in msg and kept, msg
        rf.free()
        rc, msg, kept = call(exact, p(off), p(ids), 123456)   # an unknown filter
        assert rc != 0 and kept
        ans = h._answers(3, 10, True, True)
        assert L.hnsw_b200_search_exact(h._h, 123456, p(Q), 3, 24, 10, *map(p, ans)) != 0
        assert pkg.last_error() == msg
    # a stale filter: refused with the wording of the filtered calls
    h2 = pkg.Hnsw(M, N + 4, 16, EFC, "DistL2")
    h2.insert_flat(X)
    rf2 = h2.make_filter(np.arange(N, dtype=np.uint64))
    h2.insert_flat(X[:1])
    with pytest.raises(pkg.HnswError):
        h2.search_flat_excluding(Q, 10, 64, [[1], [], [2]], filter=rf2)
    msg = pkg.last_error()
    with pytest.raises(pkg.HnswError) as e:
        h2.search_flat(Q, 10, 64, filter=rf2)
    assert str(e.value) == msg
    rf2.free()

"""A filter per query (include/hnsw_b200.h "A filter per query"): Hnsw.search_flat_per_query and search_exact_per_query,
one batch whose query i uses resident filter filters[i] or none (None / -1).

Row i must equal, bit for bit, what the single-filter call returns for query i: search_flat(filter=filters[i]) (the
unfiltered search_flat for None) or search_exact(filter=filters[i]); ids, distance bits, internal ids, PointIds and
counts, and with statistics on the counters of one per-query call equal the sum over the single-filter calls.  Every
refusal names the first bad position and leaves the handle answering as before."""
import threading

import numpy as np
import pytest

from answers import per_group, rows_of, same, same_as_single_filter_calls
from exactref import expected, handle, origin_ids
from graphs import data
from restrict import EFC, M, N, build

pytestmark = pytest.mark.gpu


def graph_filters(h):
    """(name, origin ids admitted) for: none, one point, a third, the tie-heavy twins, all"""
    ids = origin_ids(N)
    sets = [("none", ids[:0]), ("one", ids[1234:1235]), ("third", ids[1::3]), ("twins", ids[:400]), ("all", ids)]
    return [(name, allow, h.make_filter(allow)) for name, allow in sets]


def take(res, rows):
    return tuple(None if x is None else x[rows] for x in res)


GRAPH_CASES = [(np.float32, "DistL2", 24), (np.float32, "DistL2", 100), (np.uint8, "DistHamming", 100)]


@pytest.mark.parametrize("dtype,metric,d", GRAPH_CASES, ids=[f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}" for c in GRAPH_CASES])
def test_graph_rows_equal_single_filter_calls(pkg, po, dtype, metric, d):
    X, Q, o, h = build(pkg, po, dtype, metric, d, seed=d)
    fl = graph_filters(h)
    rfs = [rf for _, _, rf in fl]
    sel = np.random.default_rng(d).integers(-1, len(fl), len(Q))
    filters = [None if g < 0 else rfs[g] for g in sel]
    # tie mode 1 changes the kernel of the -1 rows only
    same_as_single_filter_calls(h, Q, sel, rfs, lambda k, ef: h.search_flat_per_query(Q, k, ef, filters))
    # one group straight against the oracle's filtered search
    h.set_tie_mode(0)
    name, allow, rf = fl[2]
    rows = rows_of(sel, 2)
    got = h.search_flat_per_query(Q, 10, 64, filters)
    oo = o.search_batch(Q[rows], 10, 64, filter_ids=allow)
    assert np.array_equal(got[4][rows], oo[4]) and np.array_equal(got[2][rows], oo[2])
    assert np.array_equal(got[1][rows].view(np.uint32), oo[1].view(np.uint32))
    for rf in rfs:
        rf.free()


def exact_filters(h, n, seed):
    """filters over internal ids: one point, three, ~5 %, ~50 %, all"""
    rng = np.random.default_rng(seed)
    og = origin_ids(n)
    sets = [np.array([n // 2]), np.array([0, n // 3, n - 1]), np.sort(rng.choice(n, n // 20, replace=False)),
            np.sort(rng.choice(n, n // 2, replace=False)), np.arange(n)]
    return sets, [h.make_filter(og[a]) for a in sets]


@pytest.mark.parametrize("k", [1, 10, 100])
def test_exact_rows_equal_single_filter_calls(pkg, po, k):
    """groups of 1, 31, 32, 33 and 70 rows (tiles of up to 32 straddle them) and a -1 group, shuffled"""
    n, d = 1500, 24
    X = data(np.float32, "DistL2", n, d, 3)
    h = handle(pkg, X, "DistL2")
    sets, rfs = exact_filters(h, n, k)
    sizes = [1, 31, 32, 33, 70, 45]   # the last group is the unfiltered one
    sel = np.concatenate([np.full(s, g if g < len(rfs) else -1) for g, s in enumerate(sizes)])
    np.random.default_rng(k).shuffle(sel)
    Q = data(np.float32, "DistL2", len(sel), d, 103)
    Q[:10] = X[:10]
    filters = [None if g < 0 else rfs[g] for g in sel]
    got = h.search_exact_per_query(Q, k, filters)
    kern = pkg.last_kernel()
    same(got, per_group(lambda q, rf: h.search_exact(q, k, filter=rf), Q, sel, rfs), f"k={k}")
    h.search_exact(Q[:4], k, filter=rfs[0])
    assert "exact_knn_kernel" in kern and pkg.last_kernel() == kern
    for g in np.unique(sel):
        rows = rows_of(sel, g)
        adm = np.arange(n) if g < 0 else sets[g]
        same(take(got, rows), expected(po, h, X, Q[rows], k, "DistL2", adm), f"k={k} group {g} vs oracle")
    for rf in rfs:
        rf.free()


def test_exact_split_and_unsplit_launches(pkg, po):
    """Eight rows over 60 000 points (four unfiltered, four on a ~50 % filter): two tiles, so the points are split over
    many CTAs whose lists are merged in the kernel.  Rows whose filters all admit < 2 048 points are never split (a slice
    of the widest tile keeps >= 1 024 points).  Both equal the oracle."""
    n, d = 60000, 24
    X = data(np.float32, "DistL2", n, d, 21)
    h = handle(pkg, X, "DistL2")
    rng = np.random.default_rng(2)
    half = np.sort(rng.choice(n, n // 2, replace=False))
    small = [np.sort(rng.choice(n, 1500, replace=False)), np.sort(rng.choice(n, 700, replace=False))]
    og = origin_ids(n)
    with h.make_filter(og[half]) as rh, h.make_filter(og[small[0]]) as r0, h.make_filter(og[small[1]]) as r1:
        Q = data(np.float32, "DistL2", 8, d, 22)
        sel = np.array([-1, 0, -1, 0, 0, -1, 0, -1])
        got = h.search_exact_per_query(Q, 10, [None if g < 0 else rh for g in sel])
        for g, adm in ((-1, np.arange(n)), (0, half)):
            rows = rows_of(sel, g)
            same(take(got, rows), expected(po, h, X, Q[rows], 10, "DistL2", adm), f"split, group {g}")
        Q = data(np.float32, "DistL2", 400, d, 23)
        sel = np.arange(400) % 2
        got = h.search_exact_per_query(Q, 10, [(r0, r1)[g] for g in sel])
        for g in (0, 1):
            rows = rows_of(sel, g)
            same(take(got, rows), expected(po, h, X, Q[rows], 10, "DistL2", small[g]), f"unsplit, group {g}")


def test_degenerate_batches(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=5)
    with h.make_filter(origin_ids(N)[::3]) as rf:
        same(h.search_flat_per_query(Q, 10, 64, [rf] * len(Q)), h.search_flat(Q, 10, 64, filter=rf), "all one filter")
        same(h.search_flat_per_query(Q, 10, 64, [None] * len(Q)), h.search_flat(Q, 10, 64), "all -1")
        same(h.search_exact_per_query(Q, 10, [rf] * len(Q)), h.search_exact(Q, 10, filter=rf), "exact, all one filter")
        same(h.search_exact_per_query(Q, 10, [None] * len(Q)), h.search_exact(Q, 10), "exact, all -1")
    empty = h.search_flat_per_query(Q[:0], 10, 64, [])
    assert empty[4].shape == (0,)
    e = pkg.Hnsw(M, 100, 16, EFC, "DistL2")   # an empty index: every count 0
    with e.make_filter([1, 2]) as rf:
        for res in (e.search_flat_per_query(Q[:5, :8], 4, 16, [rf, None, rf, None, None]),
                    e.search_exact_per_query(Q[:5, :8], 4, [rf, None, rf, None, None])):
            assert np.all(res[4] == 0)


def test_many_filters(pkg, po):
    """200 distinct filters over 1 000 queries"""
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, nq=1000, seed=6)
    rng = np.random.default_rng(6)
    og = origin_ids(N)
    rfs = [h.make_filter(np.sort(rng.choice(og, int(rng.integers(1, N)), replace=False))) for _ in range(200)]
    sel = rng.integers(-1, 200, len(Q))
    filters = [None if g < 0 else rfs[g] for g in sel]
    same(h.search_flat_per_query(Q, 10, 64, filters),
         per_group(lambda q, rf: h.search_flat(q, 10, 64, filter=rf), Q, sel, rfs), "graph, 200 filters")
    same(h.search_exact_per_query(Q, 10, filters),
         per_group(lambda q, rf: h.search_exact(q, 10, filter=rf), Q, sel, rfs), "exact, 200 filters")
    for rf in rfs:
        rf.free()


def test_overflow_grows_and_reruns(pkg, po):
    """A filter admitting 3 of 20 000 points makes its searches expand the whole graph: on a fresh handle the first
    per-query batch overflows the visited tables and is re-run on grown ones.  Its answers equal the single calls'."""
    n, d = 20000, 24
    X = data(np.float32, "DistL2", n, d, 7)
    h = pkg.Hnsw(16, n, 16, 100, "DistL2")
    h.insert_flat(X, ids=origin_ids(n))
    Q = data(np.float32, "DistL2", 200, d, 107)
    og = origin_ids(n)
    with h.make_filter(og[[5, 9000, 19999]]) as three, h.make_filter(og[::2]) as half:
        sel = np.arange(len(Q)) % 3 - 1   # -1, 0, 1, -1, ...
        rfs = [three, half]
        got = h.search_flat_per_query(Q, 10, 64, [None if g < 0 else rfs[g] for g in sel])
        assert h.check_status() == 0
        same(got, per_group(lambda q, rf: h.search_flat(q, 10, 64, filter=rf), Q, sel, rfs), "overflow")
        assert np.all(got[4][sel == 0] <= 3)


def test_partitioned_handle_and_view(pkg, po):
    X = data(np.float32, "DistL2", N, 24, 8)
    Q = data(np.float32, "DistL2", 120, 24, 108)
    ids = origin_ids(N)
    h = pkg.Hnsw(M, N, 16, EFC, "DistL2")
    h.partition([0, 0])
    h.insert_flat(X, ids=ids)
    with h.make_filter(ids[1::3]) as a, h.make_filter(ids[:50]) as b:
        rfs = [a, b]
        sel = np.random.default_rng(8).integers(-1, 2, len(Q))
        filters = [None if g < 0 else rfs[g] for g in sel]
        got = h.search_flat_per_query(Q, 10, 64, filters)
        same(got, per_group(lambda q, rf: h.search_flat(q, 10, 64, filter=rf), Q, sel, rfs), "P=2 graph")
        assert np.all(got[2][got[2] != 0xFFFFFFFF] < N)   # global ranks
        same(h.search_exact_per_query(Q, 10, filters),
             per_group(lambda q, rf: h.search_exact(q, 10, filter=rf), Q, sel, rfs), "P=2 exact")
        v = h.partition_view(0)
        same(v.search_flat_per_query(Q, 10, 64, [None] * len(Q)), v.search_flat(Q, 10, 64), "view, -1")
        with pytest.raises(pkg.HnswError, match=r"filters\[0\]"):
            v.search_flat_per_query(Q[:2], 10, 64, [a, None])


def test_replicated_handle(pkg, po):
    if pkg.load_library().hnsw_b200_device_count() < 2:
        pytest.skip("needs two GPUs")
    X, _, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=9)
    Q = data(np.float32, "DistL2", 1000, 24, 109)   # >= 64 per device: sharded
    with h.make_filter(origin_ids(N)[::3]) as a, h.make_filter(origin_ids(N)[:300]) as b:
        sel = np.random.default_rng(9).integers(-1, 2, len(Q))
        filters = [None if g < 0 else (a, b)[g] for g in sel]
        one = h.search_flat_per_query(Q, 10, 64, filters)
        one_x = h.search_exact_per_query(Q, 10, filters)
        h.replicate([0, 1])
        same(h.search_flat_per_query(Q, 10, 64, filters), one, "two GPUs, graph")
        same(h.search_exact_per_query(Q, 10, filters), one_x, "two GPUs, exact")


def test_refusals_leave_the_handle_unchanged(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, nq=60, seed=10)
    E = pkg.HnswError
    L = pkg.load_library()
    allow = origin_ids(N)[::3]
    good = h.make_filter(allow)
    stale = h.make_filter(allow)
    freed = h.make_filter(allow)
    freed.free()
    other = pkg.Hnsw(M, N, 16, EFC, "DistL2")
    other.insert_flat(X, ids=origin_ids(N))
    foreign = other.make_filter(allow)
    mixed = [good if i % 2 else None for i in range(len(Q))]
    want = h.search_flat_per_query(Q, 10, 64, mixed)
    want_x = h.search_exact_per_query(Q, 10, mixed)

    def refused(bad, pos, why):
        filters = list(mixed)
        filters[pos] = bad
        for call in (lambda: h.search_flat_per_query(Q, 10, 64, filters), lambda: h.search_exact_per_query(Q, 10, filters)):
            with pytest.raises(E, match=rf"filters\[{pos}\] = {bad.id}: .*{why}"):
                call()
        same(h.search_flat_per_query(Q, 10, 64, mixed), want, "after a refused call")
        same(h.search_exact_per_query(Q, 10, mixed), want_x, "after a refused call, exact")
    refused(pkg.ResidentFilter(h, 10 ** 12), 0, "not a live filter")
    refused(freed, 7, "not a live filter")
    refused(foreign, 30, "not a live filter")
    refused(pkg.ResidentFilter(h, -5), 59, "not a live filter")
    fids = np.array([-1] * len(Q), np.int64)
    out = [np.empty((len(Q), 10), t) for t in (np.uint64, np.float32)] + [np.empty(len(Q), np.int32)]
    p = lambda a: a.ctypes.data_as(pkg.hnsw.C.c_void_p)   # noqa: E731
    assert L.hnsw_b200_search_flat_per_query(h._h, None, p(Q), len(Q), 24, 10, 64, p(out[0]), p(out[1]), None, None,
                                             p(out[2])) < 0
    assert "filters is NULL" in pkg.last_error()
    assert L.hnsw_b200_search_exact_per_query(h._h, None, p(Q), len(Q), 24, 10, p(out[0]), p(out[1]), None, None,
                                              p(out[2])) < 0
    assert L.hnsw_b200_search_flat_per_query(h._h, p(fids), p(Q), 0, 24, 10, 64, None, None, None, None, None) == 0
    # an insert makes `stale` (and `good`) stale: the first stale position is named
    h.insert_flat(data(np.float32, "DistL2", 10, 24, 77), ids=np.arange(10, dtype=np.uint64) + 10 ** 6)
    with pytest.raises(E, match=r"filters\[1\] = .*stale"):
        h.search_flat_per_query(Q, 10, 64, [None, stale] + [None] * (len(Q) - 2))
    fresh = h.make_filter(allow)
    mixed = [fresh if i % 2 else None for i in range(len(Q))]
    sel = np.where(np.arange(len(Q)) % 2, 0, -1)
    same(h.search_flat_per_query(Q, 10, 64, mixed),
         per_group(lambda q, rf: h.search_flat(q, 10, 64, filter=rf), Q, sel, [fresh]), "after an insert, with a new filter")
    for rf in (good, stale, fresh):
        rf.free()
    foreign.free()


def test_two_threads(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, nq=400, seed=11)
    with h.make_filter(origin_ids(N)[::3]) as a, h.make_filter(origin_ids(N)[:500]) as b:
        rng = np.random.default_rng(11)
        jobs = []
        for t in range(2):
            sel = rng.integers(-1, 2, len(Q))
            filters = [None if g < 0 else (a, b)[g] for g in sel]
            jobs.append((filters, h.search_flat_per_query(Q, 10, 64, filters), h.search_exact_per_query(Q, 10, filters)))
        got, errs = [[] for _ in jobs], []

        def run(t):
            try:
                for _ in range(5):
                    got[t].append((h.search_flat_per_query(Q, 10, 64, jobs[t][0]), h.search_exact_per_query(Q, 10, jobs[t][0])))
            except Exception as e:   # noqa: BLE001  (reported below, on the test's thread)
                errs.append(e)
        ths = [threading.Thread(target=run, args=(t,)) for t in range(2)]
        for th in ths:
            th.start()
        for th in ths:
            th.join()
        assert not errs, errs
        for t in range(2):
            for g, x in got[t]:
                same(g, jobs[t][1], f"thread {t}, graph")
                same(x, jobs[t][2], f"thread {t}, exact")

"""Point labels (include/hnsw_b200.h "Point labels"): Hnsw.set_labels / get_labels, and search_flat_labeled /
search_exact_labeled, one batch whose query i is restricted to the points labelled labels[i] (LABEL_NONE: every point).

Row i must equal, bit for bit, what the single-filter call returns with a resident filter that admits exactly the points
labelled labels[i] (the unfiltered call for LABEL_NONE): ids, distance bits, internal ids, PointIds and counts, and with
statistics on the counters equal the sum over those calls.  Labels follow inserts and relabelling at once."""
import tempfile
import threading

import numpy as np
import pytest

from test_gpu_exact import expected
from test_gpu_matrix import data, same
from test_gpu_per_query_filter import N, build, origin_ids, per_group, rows_of, stats_sum

pytestmark = pytest.mark.gpu

NONE = 0xFFFFFFFF


def point_labels(n, seed):
    """large labels (0: ~40 %, 1: ~30 %), tiny ones (7: one point, 8: three), the rest without a label"""
    rng = np.random.default_rng(seed)
    lab = rng.choice(np.array([0, 0, 0, 0, 1, 1, 1, 2, NONE, NONE], np.uint32), n)
    lab[lab == 7] = NONE
    lab[rng.choice(n, 4, replace=False)] = [7, 8, 8, 8]
    return lab


QLABELS = np.array([0, 1, 2, 7, 8, 99, NONE], np.uint32)   # 99: a label no point carries


def filters_for(h, lab, og):
    """one resident filter per query label (None for LABEL_NONE), admitting the points that carry it now"""
    return [None if L == NONE else h.make_filter(np.sort(og[lab == L])) for L in QLABELS]


def reference(h, Q, sel, rfs, call):
    """the single-filter call on each label's rows, in the batch's row order"""
    return per_group(lambda q, rf: call(q, rf), Q, np.where(QLABELS[sel] == NONE, -1, sel), rfs, None)


def free(rfs):
    for rf in rfs:
        if rf is not None:
            rf.free()


GRAPH_CASES = [(np.float32, "DistL2", 128), (np.float32, "DistL2", 100), (np.uint8, "DistHamming", 100),
               (np.uint16, "DistL1", 100), (np.int32, "DistL2", 24)]


@pytest.mark.parametrize("dtype,metric,d", GRAPH_CASES, ids=[f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}" for c in GRAPH_CASES])
def test_rows_equal_filter_calls(pkg, po, dtype, metric, d):
    X, Q, o, h = build(pkg, po, dtype, metric, d, seed=d + 1)
    og = origin_ids(N)
    lab = point_labels(N, d)
    h.set_labels(0, lab)
    assert np.array_equal(h.get_labels(0, N), lab)
    rfs = filters_for(h, lab, og)
    sel = np.random.default_rng(d).integers(0, len(QLABELS), len(Q))
    ql = QLABELS[sel]
    for tie in (0, 1):   # tie mode 1 changes the kernel of the LABEL_NONE rows only
        h.set_tie_mode(tie)
        for k, ef in ((1, 1), (10, 64), (40, 257)):
            what = f"tie={tie} k={k} ef={ef}"
            single = lambda q, rf: h.search_flat(q, k, ef, filter=rf)   # noqa: E731
            want = reference(h, Q, sel, rfs, single)
            same(h.search_flat_labeled(Q, k, ef, ql), want, what)
            h.enable_stats(True)
            h.get_stats()
            got = h.search_flat_labeled(Q, k, ef, ql)
            s_lab = h.get_stats()
            parts = []
            for g in np.unique(sel):
                single(Q[rows_of(sel, g)], rfs[g])
                parts.append(h.get_stats())
            h.enable_stats(False)
            same(got, want, what + " stats on")
            assert s_lab == stats_sum(parts), (what, s_lab, parts)
        for k in (1, 10):
            same(h.search_exact_labeled(Q, k, ql), reference(h, Q, sel, rfs, lambda q, rf: h.search_exact(q, k, filter=rf)),
                 f"tie={tie} exact k={k}")
    assert np.all(h.search_flat_labeled(Q, 10, 64, np.full(len(Q), 99, np.uint32))[4] == 0)
    free(rfs)


def test_labelled_rows_equal_the_oracle(pkg, po):
    """the oracle's filtered search with the predicate label == L"""
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=3)
    og = origin_ids(N)
    lab = point_labels(N, 3)
    h.set_labels(0, lab)
    for L in (0, 1, 8):
        got = h.search_flat_labeled(Q, 10, 64, np.full(len(Q), L, np.uint32))
        oo = o.search_batch(Q, 10, 64, filter_ids=np.sort(og[lab == L]))
        assert np.array_equal(got[4], oo[4]) and np.array_equal(got[2], oo[2]), L
        assert np.array_equal(got[1].view(np.uint32), oo[1].view(np.uint32)), L


def test_labels_follow_inserts_and_relabels(pkg, po):
    n0, n, d = 1500, 2000, 24
    X = data(np.float32, "DistL2", n, d, 4)
    og = origin_ids(n)
    h = pkg.Hnsw(8, n, 16, 48, "DistL2")
    h.insert_flat(X[:n0], ids=og[:n0])
    lab = np.arange(n0, dtype=np.uint32) % 3
    h.set_labels(0, lab)
    Q = data(np.float32, "DistL2", 200, d, 104)
    Q[:20] = X[n0:n0 + 20]   # new points: found once they are labelled
    ql = np.arange(len(Q), dtype=np.uint32) % 4
    ql[ql == 3] = NONE

    def check(labels, what):
        rfs = [h.make_filter(np.sort(og[: len(labels)][labels == L])) for L in range(3)]
        sel = np.where(ql == NONE, -1, ql.astype(np.int64))
        want = per_group(lambda q, rf: h.search_flat(q, 10, 64, filter=rf), Q, sel, rfs, 10)
        want_x = per_group(lambda q, rf: h.search_exact(q, 10, filter=rf), Q, sel, rfs, 10)
        got, got_x = h.search_flat_labeled(Q, 10, 64, ql), h.search_exact_labeled(Q, 10, ql)
        same(got, want, what)
        same(got_x, want_x, what + ", exact")
        free(rfs)
        return got, got_x

    check(lab, "before the insert")
    h.insert_flat(X[n0:], ids=og[n0:])   # the new points have no label: no refresh, and none of them is found
    full = np.concatenate([lab, np.full(n - n0, NONE, np.uint32)])
    assert np.array_equal(h.get_labels(0, n), full)
    got, got_x = check(full, "after the insert")
    lab_rows = ql != NONE
    for r in (got, got_x):
        it = r[2][lab_rows]
        assert np.all((it < n0) | (it == NONE))
    full[n0:] = np.arange(n0, n, dtype=np.uint32) % 3   # label the new points: now they are found
    h.set_labels(n0, full[n0:])
    got, got_x = check(full, "new points labelled")
    assert np.any(got_x[2][lab_rows] >= n0) and np.any(got[2][lab_rows] >= n0)
    rng = np.random.default_rng(4)   # relabel: move points between labels and clear some
    moved = rng.choice(n, 600, replace=False)
    full[moved[:400]] = (full[moved[:400]] + 1) % 3
    full[moved[400:]] = NONE
    h.set_labels(0, full)
    check(full, "relabelled")
    h.set_labels(100, np.full(50, NONE, np.uint32))   # LABEL_NONE clears
    full[100:150] = NONE
    check(full, "cleared")


def test_overflow_grows_and_reruns(pkg, po):
    """One label held by 3 of 20 000 points makes its searches expand the whole graph: on a fresh handle the first
    labelled batch overflows the visited tables and is re-run on grown ones."""
    n, d = 20000, 24
    X = data(np.float32, "DistL2", n, d, 7)
    og = origin_ids(n)
    h = pkg.Hnsw(16, n, 16, 100, "DistL2")
    h.insert_flat(X, ids=og)
    lab = np.full(n, 1, np.uint32)
    lab[::2] = 2
    lab[[5, 9000, 19999]] = 0
    h.set_labels(0, lab)
    Q = data(np.float32, "DistL2", 200, d, 107)
    ql = np.array([NONE, 0, 2], np.uint32)[np.arange(len(Q)) % 3]
    got = h.search_flat_labeled(Q, 10, 64, ql)
    assert h.check_status() == 0
    with h.make_filter(og[[5, 9000, 19999]]) as three, h.make_filter(np.sort(og[lab == 2])) as half:
        sel = np.arange(len(Q)) % 3 - 1
        same(got, per_group(lambda q, rf: h.search_flat(q, 10, 64, filter=rf), Q, sel, [three, half], 10), "overflow")
    assert np.all(got[4][ql == 0] <= 3)


@pytest.mark.parametrize("P", [2, 3])
def test_partitioned_handle_and_view(pkg, po, P):
    X = data(np.float32, "DistL2", N, 24, 8)
    Q = data(np.float32, "DistL2", 120, 24, 108)
    og = origin_ids(N)
    h = pkg.Hnsw(8, N, 16, 48, "DistL2")
    h.partition([0] * P)
    h.insert_flat(X, ids=og)
    lab = point_labels(N, P)
    h.set_labels(0, lab[:700])   # global ranks, in two calls that do not start on partition 0
    h.set_labels(700, lab[700:])
    assert np.array_equal(h.get_labels(0, N), lab) and np.array_equal(h.get_labels(3, 10), lab[3:13])
    rfs = filters_for(h, lab, og)
    sel = np.random.default_rng(P).integers(0, len(QLABELS), len(Q))
    ql = QLABELS[sel]
    got = h.search_flat_labeled(Q, 10, 64, ql)
    same(got, reference(h, Q, sel, rfs, lambda q, rf: h.search_flat(q, 10, 64, filter=rf)), f"P={P} graph")
    assert np.all(got[2][got[2] != NONE] < N)   # global ranks
    same(h.search_exact_labeled(Q, 10, ql), reference(h, Q, sel, rfs, lambda q, rf: h.search_exact(q, 10, filter=rf)),
         f"P={P} exact")
    free(rfs)
    v = h.partition_view(1)
    local = lab[1::P]
    assert np.array_equal(v.get_labels(0, len(local)), local)
    with pytest.raises(pkg.HnswError, match="read-only"):
        v.set_labels(0, local)
    vq = np.full(len(Q), 1, np.uint32)
    vq[::2] = NONE
    res = v.search_flat_labeled(Q, 10, 64, vq)
    same(tuple(x[::2] for x in res), v.search_flat(Q[::2], 10, 64), "view, LABEL_NONE rows")
    it = res[2][1::2]
    assert np.all(local[it[it != NONE]] == 1) and np.all(res[4][1::2] > 0)
    ex = v.search_exact_labeled(Q, 10, vq)
    rows = np.arange(1, len(Q), 2)
    same(tuple(x[rows] for x in ex), expected(po, v, X[1::P], Q[rows], 10, "DistL2", np.flatnonzero(local == 1)),
         "view, exact")


def test_replicated_handle(pkg, po):
    if pkg.load_library().hnsw_b200_device_count() < 2:
        pytest.skip("needs two GPUs")
    X, _, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=9)
    Q = data(np.float32, "DistL2", 1000, 24, 109)   # >= 64 per device: sharded
    h.set_labels(0, point_labels(N, 9))
    ql = QLABELS[np.random.default_rng(9).integers(0, len(QLABELS), len(Q))]
    one, one_x = h.search_flat_labeled(Q, 10, 64, ql), h.search_exact_labeled(Q, 10, ql)
    h.replicate([0, 1])
    same(h.search_flat_labeled(Q, 10, 64, ql), one, "two GPUs, graph")
    same(h.search_exact_labeled(Q, 10, ql), one_x, "two GPUs, exact")
    lab2 = point_labels(N, 10)   # the replica gets the new labels at its next labelled search
    h.set_labels(0, lab2)
    two = h.search_flat_labeled(Q, 10, 64, ql)
    h.replicate([0])
    same(two, h.search_flat_labeled(Q, 10, 64, ql), "relabelled, two GPUs against one")


def test_dump_reload_has_no_labels(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=12)
    h.set_labels(0, point_labels(N, 12))
    with tempfile.TemporaryDirectory() as tmp:
        used = h.file_dump(tmp, "lab")
        r = pkg.Hnsw.load(tmp, used, "DistL2")
    assert np.all(r.get_labels(0, N) == NONE)
    same(r.search_flat_labeled(Q, 10, 64, np.full(len(Q), NONE, np.uint32)), r.search_flat(Q, 10, 64), "reloaded")
    assert np.all(r.search_flat_labeled(Q, 10, 64, np.zeros(len(Q), np.uint32))[4] == 0)


def test_refusals_and_edges(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, nq=60, seed=10)
    E = pkg.HnswError
    L = pkg.load_library()
    lab = point_labels(N, 10)
    h.set_labels(0, lab)
    ql = QLABELS[np.arange(len(Q)) % len(QLABELS)]
    want = h.search_flat_labeled(Q, 10, 64, ql)
    out = [np.empty((len(Q), 10), t) for t in (np.uint64, np.float32)] + [np.empty(len(Q), np.int32)]
    p = lambda a: a.ctypes.data_as(pkg.hnsw.C.c_void_p)   # noqa: E731
    for first, cnt in ((N - 5, 6), (N + 1, 0)):
        with pytest.raises(E, match="out of range"):
            h.set_labels(first, np.zeros(cnt, np.uint32))
    assert L.hnsw_b200_set_labels(h._h, 2 ** 63, 2 ** 63, p(ql)) < 0   # first + n wraps around
    assert "out of range" in pkg.last_error()
    with pytest.raises(E, match="out of range"):
        h.get_labels(N - 1, 2)
    assert np.array_equal(h.get_labels(0, N), lab)   # nothing changed
    h.set_labels(N, np.zeros(0, np.uint32))
    assert L.hnsw_b200_search_flat_labeled(h._h, None, p(Q), len(Q), 24, 10, 64, p(out[0]), p(out[1]), None, None,
                                           p(out[2])) < 0
    assert "qlabels is NULL" in pkg.last_error()
    assert L.hnsw_b200_search_exact_labeled(h._h, None, p(Q), len(Q), 24, 10, p(out[0]), p(out[1]), None, None,
                                            p(out[2])) < 0
    assert L.hnsw_b200_set_labels(h._h, 0, 5, None) < 0
    assert L.hnsw_b200_search_flat_labeled(h._h, p(ql), p(Q), 0, 24, 10, 64, None, None, None, None, None) == 0
    assert h.search_flat_labeled(Q[:0], 10, 64, ql[:0])[4].shape == (0,)
    same(h.search_flat_labeled(Q, 10, 64, ql), want, "after the refused calls")
    for res in (h.search_flat_labeled(Q, 10, 64, np.full(len(Q), 12345, np.uint32)),
                h.search_exact_labeled(Q, 10, np.full(len(Q), 12345, np.uint32))):
        assert np.all(res[4] == 0) and np.all(res[2] == NONE)
    e = pkg.Hnsw(8, 100, 16, 48, "DistL2")   # an empty index: every count 0
    for res in (e.search_flat_labeled(Q[:5, :8], 4, 16, ql[:5]), e.search_exact_labeled(Q[:5, :8], 4, ql[:5])):
        assert np.all(res[4] == 0)


def test_many_distinct_labels(pkg, po):
    """100 000 queries with 100 000 distinct labels over 300 points, each labelled with its own rank: the labels below
    300 admit one point, the others none.  The reference is one per-query call with one single-point filter per label
    that some point carries and an empty filter for the rest."""
    n, d, nq = 300, 24, 100000
    X = data(np.float32, "DistL2", n, d, 13)
    og = origin_ids(n)
    h = pkg.Hnsw(8, n, 16, 48, "DistL2")
    h.insert_flat(X, ids=og)
    h.set_labels(0, np.arange(n, dtype=np.uint32))
    rng = np.random.default_rng(13)
    ql = rng.permutation(nq).astype(np.uint32)
    Q = data(np.float32, "DistL2", nq, d, 113)
    rfs = [h.make_filter(og[i:i + 1]) for i in range(n)]
    empty = h.make_filter([])
    filters = [rfs[L] if L < n else empty for L in ql]
    same(h.search_flat_labeled(Q, 5, 32, ql), h.search_flat_per_query(Q, 5, 32, filters), "graph, 100 000 labels")
    same(h.search_exact_labeled(Q, 5, ql), h.search_exact_per_query(Q, 5, filters), "exact, 100 000 labels")
    for rf in rfs + [empty]:
        rf.free()


def test_two_threads_search_while_a_third_sets_labels(pkg, po):
    """every answer is what one of the two label sets gives: set_labels takes the handle exclusively"""
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, nq=400, seed=11)
    sets = [point_labels(N, 11), point_labels(N, 12)]
    ql = QLABELS[np.random.default_rng(11).integers(0, len(QLABELS), len(Q))]
    want = []
    for lab in sets:
        h.set_labels(0, lab)
        want.append((h.search_flat_labeled(Q, 10, 64, ql), h.search_exact_labeled(Q, 10, ql)))
    got, errs, stop = [[], []], [], threading.Event()

    def search(t):
        try:
            for _ in range(6):
                got[t].append((h.search_flat_labeled(Q, 10, 64, ql), h.search_exact_labeled(Q, 10, ql)))
        except Exception as e:   # noqa: BLE001  (reported below, on the test's thread)
            errs.append(e)

    def relabel():
        i = 0
        while not stop.is_set():
            h.set_labels(0, sets[i % 2])
            i += 1

    ths = [threading.Thread(target=search, args=(t,)) for t in range(2)]
    writer = threading.Thread(target=relabel)
    writer.start()
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    stop.set()
    writer.join()
    assert not errs, errs
    for t in range(2):
        for g, x in got[t]:
            assert any(np.array_equal(g[2], w[0][2]) and np.array_equal(g[4], w[0][4]) for w in want), f"thread {t}"
            assert any(np.array_equal(x[2], w[1][2]) and np.array_equal(x[4], w[1][4]) for w in want), f"thread {t}"

"""Attribute ranges (include/hnsw_b200.h "Attribute ranges"): Hnsw.set_attributes, search_flat_ranges and
search_exact_ranges, one batch whose query i is restricted to the points whose int64 attribute lies in ranges[i], alone
or within the label set sets[i].

Row i must equal, bit for bit, what the single-filter call returns with a resident filter that admits exactly those
points (the unfiltered call for a full range and [LABEL_NONE], the label-set call for a full range and another set): ids,
distance bits, internal ids, PointIds and counts, and with statistics on the counters equal the sum over those calls."""
import tempfile

import numpy as np
import pytest

from answers import per_group, same, same_as_single_filter_calls
from exactref import expected, origin_ids
from graphs import data
from restrict import (FULL, GRAPH_CASES, I64_MAX, I64_MIN, NONE, ROWS, N, admitted, build, free, point_attrs,
                      point_labels, unrestricted)

pytestmark = pytest.mark.gpu

def filters_for(h, lab, attr, og, rows=ROWS):
    """one resident filter per (set, range) row (None for the unrestricted one)"""
    return [None if unrestricted(s) and tuple(r) == FULL else h.make_filter(np.sort(og[admitted(lab, attr, s, r)]))
            for s, r in rows]


def selector(sel, rows=ROWS):
    return np.array([-1 if unrestricted(rows[g][0]) and tuple(rows[g][1]) == FULL else g for g in sel], np.int64)


def args(sel, rows=ROWS):
    return np.array([rows[g][1] for g in sel], np.int64), [rows[g][0] for g in sel]


@pytest.mark.parametrize("dtype,metric,d", GRAPH_CASES, ids=[f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}" for c in GRAPH_CASES])
def test_rows_equal_filter_calls(pkg, po, dtype, metric, d):
    X, Q, o, h = build(pkg, po, dtype, metric, d, seed=d + 2)
    og = origin_ids(N)
    lab, attr = point_labels(N, d), point_attrs(N, d)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    assert np.array_equal(h.get_attributes(0, N), attr)
    rfs = filters_for(h, lab, attr, og)
    sel = np.random.default_rng(d).integers(0, len(ROWS), len(Q))
    rg, qs = args(sel)
    g = selector(sel)
    # tie mode 1 changes the kernel of the unrestricted rows only
    same_as_single_filter_calls(h, Q, g, rfs, lambda k, ef: h.search_flat_ranges(Q, k, ef, rg, qs),
                                lambda k: h.search_exact_ranges(Q, k, rg, qs))
    free(rfs)


def test_ranges_without_sets(pkg, po):
    """sets=None: every row's set is [LABEL_NONE]; the labels play no part"""
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=31)
    og = origin_ids(N)
    lab, attr = point_labels(N, 31), point_attrs(N, 31)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    rows = [([NONE], r) for _, r in ROWS]
    rfs = filters_for(h, lab, attr, og, rows)
    sel = np.arange(len(Q)) % len(rows)
    rg, _ = args(sel, rows)
    g = selector(sel, rows)
    same(h.search_flat_ranges(Q, 10, 64, rg), per_group(lambda q, rf: h.search_flat(q, 10, 64, filter=rf), Q, g, rfs),
         "graph")
    same(h.search_exact_ranges(Q, 10, [tuple(r) for r in rg]),
         per_group(lambda q, rf: h.search_exact(q, 10, filter=rf), Q, g, rfs), "exact, pairs")
    free(rfs)


def test_full_ranges_equal_label_set_and_unfiltered_rows(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=21)
    h.set_labels(0, point_labels(N, 21))
    h.set_attributes(0, point_attrs(N, 21))
    sets = [[0, 1], [2], [NONE], [], [8, 7]]
    qs = [sets[i % len(sets)] for i in range(len(Q))]
    full = np.tile(np.array(FULL, np.int64), (len(Q), 1))
    same(h.search_flat_ranges(Q, 10, 64, full, qs), h.search_flat_label_sets(Q, 10, 64, qs), "graph, label sets")
    same(h.search_exact_ranges(Q, 10, full, qs), h.search_exact_label_sets(Q, 10, qs), "exact, label sets")
    for tie in (0, 1):
        h.set_tie_mode(tie)
        same(h.search_flat_ranges(Q, 10, 64, full), h.search_flat(Q, 10, 64), f"graph, unfiltered, tie={tie}")
    same(h.search_exact_ranges(Q, 10, full), h.search_exact(Q, 10), "exact, unfiltered")


def test_rows_equal_the_oracle(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=3)
    og = origin_ids(N)
    lab, attr = point_labels(N, 3), point_attrs(N, 3)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    for s, r in (([NONE], (-300, 300)), ([0, 2], (0, 999)), ([1], (I64_MIN, -500))):
        got = h.search_flat_ranges(Q, 10, 64, [r] * len(Q), [s] * len(Q))
        oo = o.search_batch(Q, 10, 64, filter_ids=np.sort(og[admitted(lab, attr, s, r)]))
        assert np.array_equal(got[4], oo[4]) and np.array_equal(got[2], oo[2]), (s, r)
        assert np.array_equal(got[1].view(np.uint32), oo[1].view(np.uint32)), (s, r)


def test_every_row_its_own_window(pkg, po):
    """a different window per row, alone and within a label: as many runs as rows, on the graph and exactly"""
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, nq=240, seed=6)
    og = origin_ids(N)
    lab, attr = point_labels(N, 6), point_attrs(N, 6)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    lo = np.arange(len(Q), dtype=np.int64) * 7 - 900
    rows = [([NONE] if i % 2 else [i % 3], (int(lo[i]), int(lo[i]) + 150)) for i in range(len(Q))]
    rfs = filters_for(h, lab, attr, og, rows)
    sel = np.random.default_rng(6).permutation(len(Q))
    rg, qs = args(sel, rows)
    g = selector(sel, rows)
    assert np.all(g >= 0) and len(np.unique(g)) == len(Q)
    same(h.search_flat_ranges(Q, 10, 64, rg, qs), per_group(lambda q, rf: h.search_flat(q, 10, 64, filter=rf), Q, g, rfs),
         "graph")
    same(h.search_exact_ranges(Q, 10, rg, qs), per_group(lambda q, rf: h.search_exact(q, 10, filter=rf), Q, g, rfs),
         "exact")
    free(rfs)


def test_overflow_grows_and_reruns(pkg, po):
    """A range admitting 3 of 20 000 points makes its searches expand the whole graph: on a fresh handle the first batch
    overflows the visited tables and is re-run on grown ones."""
    n, d = 20000, 24
    X = data(np.float32, "DistL2", n, d, 7)
    og = origin_ids(n)
    h = pkg.Hnsw(16, n, 16, 100, "DistL2")
    h.insert_flat(X, ids=og)
    attr = np.arange(n, dtype=np.int64) % 1000
    attr[[5, 9000, 19999]] = 5000
    h.set_attributes(0, attr)
    Q = data(np.float32, "DistL2", 200, d, 107)
    rows = [FULL, (4000, 6000), (0, 499)]
    rg = np.array([rows[i % 3] for i in range(len(Q))], np.int64)
    h.enable_stats(True)
    h.get_stats()
    got = h.search_flat_ranges(Q, 10, 64, rg)
    first = h.get_stats()
    assert h.check_status() == 0
    same(h.search_flat_ranges(Q, 10, 64, rg), got, "the same batch on the grown tables")
    again = h.get_stats()
    h.enable_stats(False)
    assert first["evals"] > again["evals"] and first["queries"] > again["queries"], (first, again)
    with h.make_filter(og[[5, 9000, 19999]]) as three, h.make_filter(np.sort(og[attr < 500])) as half:
        sel = np.arange(len(Q)) % 3 - 1
        same(got, per_group(lambda q, rf: h.search_flat(q, 10, 64, filter=rf), Q, sel, [three, half]), "overflow")
    assert np.all(got[4][1::3] <= 3)


def test_attributes_follow_inserts_and_changes(pkg, po):
    """both exact orders (by value, and by label and value) and the graph rows follow inserts, new values and clearing"""
    n0, n, d = 1500, 2000, 24
    X = data(np.float32, "DistL2", n, d, 4)
    og = origin_ids(n)
    h = pkg.Hnsw(8, n, 16, 48, "DistL2")
    h.insert_flat(X[:n0], ids=og[:n0])
    lab = np.arange(n0, dtype=np.uint32) % 4
    attr = np.arange(n0, dtype=np.int64) % 100
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    Q = data(np.float32, "DistL2", 200, d, 104)
    Q[:20] = X[n0:n0 + 20]   # new points: found once they have attributes
    rows = [([NONE], (10, 60)), ([0, 1], (0, 49)), ([3], (20, 99)), ([NONE], FULL), ([2], FULL), ([1, 3], (I64_MIN, 30))]
    sel = np.arange(len(Q)) % len(rows)
    rg, qs = args(sel, rows)
    g = selector(sel, rows)

    def check(lab, attr, what):
        rfs = filters_for(h, lab, attr, og[: len(lab)], rows)
        want = per_group(lambda q, rf: h.search_flat(q, 10, 64, filter=rf), Q, g, rfs)
        want_x = per_group(lambda q, rf: h.search_exact(q, 10, filter=rf), Q, g, rfs)
        got, got_x = h.search_flat_ranges(Q, 10, 64, rg, qs), h.search_exact_ranges(Q, 10, rg, qs)
        same(got, want, what)
        same(got_x, want_x, what + ", exact")
        free(rfs)
        return got, got_x

    check(lab, attr, "before the insert")
    h.insert_flat(X[n0:], ids=og[n0:])
    lab = np.concatenate([lab, np.full(n - n0, NONE, np.uint32)])
    attr = np.concatenate([attr, np.full(n - n0, I64_MIN, np.int64)])
    assert np.array_equal(h.get_attributes(0, n), attr)
    got, got_x = check(lab, attr, "after the insert")
    ranged = np.isin(sel, [0, 1, 2, 5])
    for r in (got, got_x):
        it = r[2][ranged]
        assert np.all((it < n0) | (it == NONE))
    attr[n0:] = np.arange(n0, n, dtype=np.int64) % 100
    h.set_attributes(n0, attr[n0:])
    got, got_x = check(lab, attr, "new points with attributes")
    assert np.any(got_x[2][sel == 0] >= n0) and np.any(got[2][sel == 0] >= n0)
    lab[n0:] = np.arange(n0, n, dtype=np.uint32) % 4
    h.set_labels(n0, lab[n0:])
    check(lab, attr, "new points labelled")
    rng = np.random.default_rng(4)
    moved = rng.choice(n, 600, replace=False)
    attr[moved[:400]] = rng.integers(-50, 150, 400)
    attr[moved[400:]] = I64_MIN   # cleared
    h.set_attributes(0, attr)
    check(lab, attr, "new values and cleared ones")
    assert np.array_equal(h.get_attributes(0, n), attr)
    assert np.array_equal(h.get_labels(0, n), lab)   # attributes leave labels alone
    relabelled = rng.choice(n, 500, replace=False)   # points that have a label get another one: only the label-keyed
    lab[relabelled] = (lab[relabelled] + rng.integers(1, 4, 500)) % 4   # exact orders go stale
    h.set_labels(0, lab)
    check(lab, attr, "relabelled, attributes unchanged")
    assert np.array_equal(h.get_attributes(0, n), attr)   # labels leave attributes alone


@pytest.mark.parametrize("P", [2, 3])
def test_partitioned_handle_and_view(pkg, po, P):
    X = data(np.float32, "DistL2", N, 24, 8)
    Q = data(np.float32, "DistL2", 120, 24, 108)
    og = origin_ids(N)
    h = pkg.Hnsw(8, N, 16, 48, "DistL2")
    h.partition([0] * P)
    h.insert_flat(X, ids=og)
    lab, attr = point_labels(N, P), point_attrs(N, P)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    assert np.array_equal(h.get_attributes(0, N), attr)
    assert np.array_equal(h.get_attributes(5, 7), attr[5:12])
    rfs = filters_for(h, lab, attr, og)
    sel = np.random.default_rng(P).integers(0, len(ROWS), len(Q))
    rg, qs = args(sel)
    g = selector(sel)
    got = h.search_flat_ranges(Q, 10, 64, rg, qs)
    same(got, per_group(lambda q, rf: h.search_flat(q, 10, 64, filter=rf), Q, g, rfs), f"P={P} graph")
    assert np.all(got[2][got[2] != NONE] < N)   # global ranks
    same(h.search_exact_ranges(Q, 10, rg, qs), per_group(lambda q, rf: h.search_exact(q, 10, filter=rf), Q, g, rfs),
         f"P={P} exact")
    free(rfs)
    v = h.partition_view(1)
    local_lab, local_attr = lab[1::P], attr[1::P]
    assert np.array_equal(v.get_attributes(0, len(local_attr)), local_attr)
    with pytest.raises(pkg.HnswError):
        v.set_attributes(0, local_attr[:3])
    vr = np.array([FULL if i % 2 == 0 else (-200, 600) for i in range(len(Q))], np.int64)
    vs = [[NONE] if i % 2 == 0 else [2, 1] for i in range(len(Q))]
    res = v.search_flat_ranges(Q, 10, 64, vr, vs)
    same(tuple(x[::2] for x in res), v.search_flat(Q[::2], 10, 64), "view, unrestricted rows")
    adm = np.flatnonzero(admitted(local_lab, local_attr, [2, 1], (-200, 600)))
    it = res[2][1::2]
    assert np.all(np.isin(it[it != NONE], adm)) and np.all(res[4][1::2] > 0)
    ex = v.search_exact_ranges(Q, 10, vr, vs)
    rows = np.arange(1, len(Q), 2)
    same(tuple(x[rows] for x in ex), expected(po, v, X[1::P], Q[rows], 10, "DistL2", adm), "view, exact")


def test_replicated_handle(pkg, po):
    if pkg.load_library().hnsw_b200_device_count() < 2:
        pytest.skip("needs two GPUs")
    X, _, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=9)
    Q = data(np.float32, "DistL2", 1000, 24, 109)   # >= 64 per device: sharded
    h.set_labels(0, point_labels(N, 9))
    h.set_attributes(0, point_attrs(N, 9))
    rg, qs = args(np.random.default_rng(9).integers(0, len(ROWS), len(Q)))
    one, one_x = h.search_flat_ranges(Q, 10, 64, rg, qs), h.search_exact_ranges(Q, 10, rg, qs)
    h.replicate([0, 1])
    same(h.search_flat_ranges(Q, 10, 64, rg, qs), one, "two GPUs, graph")
    same(h.search_exact_ranges(Q, 10, rg, qs), one_x, "two GPUs, exact")
    h.set_attributes(0, point_attrs(N, 10))   # the replica gets the new attributes at its next search
    two, two_x = h.search_flat_ranges(Q, 10, 64, rg, qs), h.search_exact_ranges(Q, 10, rg, qs)
    h.replicate([0])
    same(two, h.search_flat_ranges(Q, 10, 64, rg, qs), "new values, two GPUs against one")
    same(two_x, h.search_exact_ranges(Q, 10, rg, qs), "new values, exact, two GPUs against one")


def test_dump_reload_has_no_attributes(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=12)
    h.set_attributes(0, point_attrs(N, 12))
    with tempfile.TemporaryDirectory() as tmp:
        used = h.file_dump(tmp, "attr")
        r = pkg.Hnsw.load(tmp, used, "DistL2")
    assert np.all(r.get_attributes(0, N) == pkg.ATTR_NONE)
    full = np.tile(np.array(pkg.RANGE_ALL, np.int64), (len(Q), 1))
    same(r.search_flat_ranges(Q, 10, 64, full), r.search_flat(Q, 10, 64), "reloaded")
    everything = np.tile(np.array([I64_MIN + 1, I64_MAX], np.int64), (len(Q), 1))
    for res in (r.search_flat_ranges(Q, 10, 64, everything), r.search_exact_ranges(Q, 10, everything)):
        assert np.all(res[4] == 0)


def test_refusals_and_edges(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, nq=60, seed=10)
    E = pkg.HnswError
    L = pkg.load_library()
    attr = point_attrs(N, 10)
    h.set_labels(0, point_labels(N, 10))
    h.set_attributes(0, attr)
    rg, qs = args(np.arange(len(Q)) % len(ROWS))
    want, want_x = h.search_flat_ranges(Q, 10, 64, rg, qs), h.search_exact_ranges(Q, 10, rg, qs)
    for first, cnt in ((N - 5, 6), (N + 1, 0)):
        with pytest.raises(E, match=r"attributes \[.*out of range"):
            h.set_attributes(first, np.zeros(cnt, np.int64))
    p = lambda a: a.ctypes.data_as(pkg.hnsw.C.c_void_p)   # noqa: E731
    assert L.hnsw_b200_set_attributes(h._h, 2 ** 63, 2 ** 63, p(attr)) < 0   # first + n wraps around
    assert "out of range" in pkg.last_error()
    with pytest.raises(E, match="out of range"):
        h.get_attributes(N - 1, 2)
    assert L.hnsw_b200_set_attributes(h._h, 0, 5, None) < 0
    assert "values is NULL" in pkg.last_error()
    assert np.array_equal(h.get_attributes(0, N), attr)   # nothing changed
    h.set_attributes(N, np.zeros(0, np.int64))
    with pytest.raises(ValueError, match="64-bit integers"):
        h.set_attributes(0, np.zeros(3, np.float64))
    with pytest.raises(ValueError, match=r"expected \(60, 2\)"):
        h.search_flat_ranges(Q, 10, 64, rg[:5])
    # the label-set checks, with their wording
    off = np.arange(len(Q) + 1, dtype=np.uint64)
    bad = off.copy()
    bad[8] = 10
    for call in (lambda s: h.search_flat_ranges(Q, 10, 64, rg, s), lambda s: h.search_exact_ranges(Q, 10, rg, s)):
        with pytest.raises(E, match=r"label set 8: qset_off\[9\] = 9 is below qset_off\[8\] = 10"):
            call((bad, np.zeros(len(Q) + 1, np.uint32)))
        mixed = [[1]] * len(Q)
        mixed[5] = [2, NONE, 2]
        with pytest.raises(E, match="label set 5 holds LABEL_NONE together with another label"):
            call(mixed)
    out = [np.empty((len(Q), 10), t) for t in (np.uint64, np.float32)] + [np.empty(len(Q), np.int32)]
    vals = np.zeros(len(Q), np.uint32)
    flat, exact = L.hnsw_b200_search_flat_ranges, L.hnsw_b200_search_exact_ranges
    assert flat(h._h, None, None, None, p(Q), len(Q), 24, 10, 64, p(out[0]), p(out[1]), None, None, p(out[2])) < 0
    assert "qrange is NULL" in pkg.last_error()
    assert exact(h._h, None, None, None, p(Q), len(Q), 24, 10, p(out[0]), p(out[1]), None, None, p(out[2])) < 0
    assert "qrange is NULL" in pkg.last_error()
    assert flat(h._h, p(rg), None, p(vals), p(Q), len(Q), 24, 10, 64, p(out[0]), p(out[1]), None, None, p(out[2])) < 0
    assert "qset_off is NULL" in pkg.last_error()
    assert exact(h._h, p(rg), p(off), None, p(Q), len(Q), 24, 10, p(out[0]), p(out[1]), None, None, p(out[2])) < 0
    assert "qset is NULL" in pkg.last_error()
    assert flat(None, None, None, None, p(Q), len(Q), 24, 10, 64, p(out[0]), p(out[1]), None, None, p(out[2])) < 0
    assert "NULL handle" in pkg.last_error()
    assert flat(h._h, None, None, None, p(Q), 0, 24, 10, 64, None, None, None, None, None) == 0
    assert exact(h._h, None, None, None, p(Q), 0, 24, 10, None, None, None, None, None) == 0
    assert h.search_flat_ranges(Q[:0], 10, 64, np.zeros((0, 2), np.int64))[4].shape == (0,)
    same(h.search_flat_ranges(Q, 10, 64, rg, qs), want, "after the refused calls")
    same(h.search_exact_ranges(Q, 10, rg, qs), want_x, "exact, after the refused calls")
    empty = np.tile(np.array([5, 4], np.int64), (len(Q), 1))
    for res in (h.search_flat_ranges(Q, 10, 64, empty), h.search_exact_ranges(Q, 10, empty),
                h.search_flat_ranges(Q, 10, 64, empty * 0 + [4242, 4242], [[12345]] * len(Q))):
        assert np.all(res[4] == 0) and np.all(res[2] == NONE)
    e = pkg.Hnsw(8, 100, 16, 48, "DistL2")   # an empty index: every count 0
    for res in (e.search_flat_ranges(Q[:5, :8], 4, 16, rg[:5], qs[:5]), e.search_exact_ranges(Q[:5, :8], 4, rg[:5])):
        assert np.all(res[4] == 0)

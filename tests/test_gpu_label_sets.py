"""Label sets (include/hnsw_b200.h "Label sets"): Hnsw.search_flat_label_sets / search_exact_label_sets, one batch whose
query i is restricted to the points whose label is in sets[i] ([LABEL_NONE]: every point; empty: none).

Row i must equal, bit for bit, what the single-filter call returns with a resident filter that admits exactly the points
whose label is in sets[i] (the unfiltered call for [LABEL_NONE]): ids, distance bits, internal ids, PointIds and counts,
and with statistics on the counters equal the sum over those calls.  A set of one label gives the labelled call's row."""
import numpy as np
import pytest

from answers import per_group, same, same_as_single_filter_calls
from exactref import expected, origin_ids
from graphs import data
from restrict import GRAPH_CASES, NONE, N, build, free, point_labels, unrestricted

pytestmark = pytest.mark.gpu

# point_labels carries 0 (~40 %), 1 (~30 %), 2, 7 (one point) and 8 (three points); 99 no point carries.  Sets out of
# order, with repeats, empty, and [NONE] with a repeat.
SETS = [[0, 1], [2, 7], [8, 2, 8], [7], [1, 99], [99], [], [NONE], [NONE, NONE], [2, 1, 0, 7, 8], [8, 7], [1, 0]]


def filters_for(h, lab, og, sets=SETS):
    """one resident filter per set (None for [LABEL_NONE]), admitting the points whose label is in it now"""
    return [None if unrestricted(s) else h.make_filter(np.sort(og[np.isin(lab, np.array(s, np.uint32))])) for s in sets]


def selector(sets, sel):
    """per_group's selector: -1 for the rows of an unrestricted set"""
    return np.array([-1 if unrestricted(sets[g]) else g for g in sel], np.int64)


def row_sets(sel, sets=SETS):
    return [sets[g] for g in sel]


@pytest.mark.parametrize("dtype,metric,d", GRAPH_CASES, ids=[f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}" for c in GRAPH_CASES])
def test_rows_equal_filter_calls(pkg, po, dtype, metric, d):
    X, Q, o, h = build(pkg, po, dtype, metric, d, seed=d + 1)
    og = origin_ids(N)
    lab = point_labels(N, d)
    h.set_labels(0, lab)
    rfs = filters_for(h, lab, og)
    sel = np.random.default_rng(d).integers(0, len(SETS), len(Q))
    qs, g = row_sets(sel), selector(SETS, sel)
    # tie mode 1 changes the kernel of the [LABEL_NONE] rows only
    same_as_single_filter_calls(h, Q, g, rfs, lambda k, ef: h.search_flat_label_sets(Q, k, ef, qs),
                                lambda k: h.search_exact_label_sets(Q, k, qs))
    free(rfs)


def test_one_label_sets_equal_labeled_calls(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=21)
    h.set_labels(0, point_labels(N, 21))
    ql = np.array([0, 1, 2, 7, 8, 99, NONE], np.uint32)[np.arange(len(Q)) % 7]
    qs = [[int(L)] for L in ql]
    same(h.search_flat_label_sets(Q, 10, 64, qs), h.search_flat_labeled(Q, 10, 64, ql), "graph")
    same(h.search_exact_label_sets(Q, 10, qs), h.search_exact_labeled(Q, 10, ql), "exact")
    # the (offsets, values) form, offsets not starting at 0, gives the same rows
    off = np.arange(len(Q) + 1, dtype=np.uint64) + 3
    vals = np.concatenate([np.zeros(3, np.uint32), ql, np.zeros(2, np.uint32)])
    same(h.search_flat_label_sets(Q, 10, 64, (off, vals)), h.search_flat_labeled(Q, 10, 64, ql), "offsets and values")


def test_rows_equal_the_oracle(pkg, po):
    """the oracle's filtered search with the union's origin ids"""
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=3)
    og = origin_ids(N)
    lab = point_labels(N, 3)
    h.set_labels(0, lab)
    for s in ([0, 2], [8, 7, 2], [1, 8]):
        got = h.search_flat_label_sets(Q, 10, 64, [s] * len(Q))
        oo = o.search_batch(Q, 10, 64, filter_ids=np.sort(og[np.isin(lab, s)]))
        assert np.array_equal(got[4], oo[4]) and np.array_equal(got[2], oo[2]), s
        assert np.array_equal(got[1].view(np.uint32), oo[1].view(np.uint32)), s


def test_overflow_grows_and_reruns(pkg, po):
    """A set admitting 3 of 20 000 points makes its searches expand the whole graph: on a fresh handle the first batch
    overflows the visited tables and is re-run on grown ones."""
    n, d = 20000, 24
    X = data(np.float32, "DistL2", n, d, 7)
    og = origin_ids(n)
    h = pkg.Hnsw(16, n, 16, 100, "DistL2")
    h.insert_flat(X, ids=og)
    lab = np.full(n, 1, np.uint32)
    lab[::2] = 2
    lab[[5, 9000]] = 0
    lab[19999] = 3
    h.set_labels(0, lab)
    Q = data(np.float32, "DistL2", 200, d, 107)
    sets = [[NONE], [3, 0, 44], [2]]
    qs = [sets[i % 3] for i in range(len(Q))]
    h.enable_stats(True)
    h.get_stats()
    got = h.search_flat_label_sets(Q, 10, 64, qs)
    first = h.get_stats()
    assert h.check_status() == 0
    same(h.search_flat_label_sets(Q, 10, 64, qs), got, "the same batch on the grown tables")
    again = h.get_stats()
    h.enable_stats(False)
    # the overflowing launches' work is counted besides the re-run's: the first call did more than the second
    assert first["evals"] > again["evals"] and first["queries"] > again["queries"], (first, again)
    with h.make_filter(og[[5, 9000, 19999]]) as three, h.make_filter(np.sort(og[lab == 2])) as half:
        sel = np.arange(len(Q)) % 3 - 1
        same(got, per_group(lambda q, rf: h.search_flat(q, 10, 64, filter=rf), Q, sel, [three, half]), "overflow")
    assert np.all(got[4][1::3] <= 3)


def test_sets_follow_inserts_and_relabels(pkg, po):
    n0, n, d = 1500, 2000, 24
    X = data(np.float32, "DistL2", n, d, 4)
    og = origin_ids(n)
    h = pkg.Hnsw(8, n, 16, 48, "DistL2")
    h.insert_flat(X[:n0], ids=og[:n0])
    lab = np.arange(n0, dtype=np.uint32) % 4
    h.set_labels(0, lab)
    Q = data(np.float32, "DistL2", 200, d, 104)
    Q[:20] = X[n0:n0 + 20]   # new points: found once they are labelled
    sets = [[0, 1], [2, 3], [3], [NONE], [1, 3, 0]]
    sel = np.arange(len(Q)) % len(sets)
    qs, g = row_sets(sel, sets), selector(sets, sel)

    def check(labels, what):
        rfs = filters_for(h, labels, og[: len(labels)], sets)
        want = per_group(lambda q, rf: h.search_flat(q, 10, 64, filter=rf), Q, g, rfs)
        want_x = per_group(lambda q, rf: h.search_exact(q, 10, filter=rf), Q, g, rfs)
        got, got_x = h.search_flat_label_sets(Q, 10, 64, qs), h.search_exact_label_sets(Q, 10, qs)
        same(got, want, what)
        same(got_x, want_x, what + ", exact")
        free(rfs)
        return got, got_x

    check(lab, "before the insert")
    h.insert_flat(X[n0:], ids=og[n0:])
    full = np.concatenate([lab, np.full(n - n0, NONE, np.uint32)])
    got, got_x = check(full, "after the insert")
    restricted = g >= 0
    for r in (got, got_x):
        it = r[2][restricted]
        assert np.all((it < n0) | (it == NONE))
    full[n0:] = np.arange(n0, n, dtype=np.uint32) % 4
    h.set_labels(n0, full[n0:])
    got, got_x = check(full, "new points labelled")
    assert np.any(got_x[2][restricted] >= n0) and np.any(got[2][restricted] >= n0)
    rng = np.random.default_rng(4)
    moved = rng.choice(n, 600, replace=False)
    full[moved[:400]] = (full[moved[:400]] + 1) % 4
    full[moved[400:]] = NONE
    h.set_labels(0, full)
    check(full, "relabelled")


@pytest.mark.parametrize("P", [2, 3])
def test_partitioned_handle_and_view(pkg, po, P):
    X = data(np.float32, "DistL2", N, 24, 8)
    Q = data(np.float32, "DistL2", 120, 24, 108)
    og = origin_ids(N)
    h = pkg.Hnsw(8, N, 16, 48, "DistL2")
    h.partition([0] * P)
    h.insert_flat(X, ids=og)
    lab = point_labels(N, P)
    h.set_labels(0, lab)
    rfs = filters_for(h, lab, og)
    sel = np.random.default_rng(P).integers(0, len(SETS), len(Q))
    qs, g = row_sets(sel), selector(SETS, sel)
    got = h.search_flat_label_sets(Q, 10, 64, qs)
    same(got, per_group(lambda q, rf: h.search_flat(q, 10, 64, filter=rf), Q, g, rfs), f"P={P} graph")
    assert np.all(got[2][got[2] != NONE] < N)   # global ranks
    same(h.search_exact_label_sets(Q, 10, qs), per_group(lambda q, rf: h.search_exact(q, 10, filter=rf), Q, g, rfs),
         f"P={P} exact")
    free(rfs)
    v = h.partition_view(1)
    local = lab[1::P]
    vs = [[NONE] if i % 2 == 0 else [2, 1] for i in range(len(Q))]
    res = v.search_flat_label_sets(Q, 10, 64, vs)
    same(tuple(x[::2] for x in res), v.search_flat(Q[::2], 10, 64), "view, [LABEL_NONE] rows")
    it = res[2][1::2]
    assert np.all(np.isin(local[it[it != NONE]], [1, 2])) and np.all(res[4][1::2] > 0)
    ex = v.search_exact_label_sets(Q, 10, vs)
    rows = np.arange(1, len(Q), 2)
    same(tuple(x[rows] for x in ex), expected(po, v, X[1::P], Q[rows], 10, "DistL2", np.flatnonzero(np.isin(local, [1, 2]))),
         "view, exact")


def test_replicated_handle(pkg, po):
    if pkg.load_library().hnsw_b200_device_count() < 2:
        pytest.skip("needs two GPUs")
    X, _, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=9)
    Q = data(np.float32, "DistL2", 1000, 24, 109)   # >= 64 per device: sharded
    h.set_labels(0, point_labels(N, 9))
    qs = row_sets(np.random.default_rng(9).integers(0, len(SETS), len(Q)))
    one, one_x = h.search_flat_label_sets(Q, 10, 64, qs), h.search_exact_label_sets(Q, 10, qs)
    h.replicate([0, 1])
    same(h.search_flat_label_sets(Q, 10, 64, qs), one, "two GPUs, graph")
    same(h.search_exact_label_sets(Q, 10, qs), one_x, "two GPUs, exact")
    h.set_labels(0, point_labels(N, 10))   # the replica gets the new labels at its next search
    two, two_x = h.search_flat_label_sets(Q, 10, 64, qs), h.search_exact_label_sets(Q, 10, qs)
    h.replicate([0])
    same(two, h.search_flat_label_sets(Q, 10, 64, qs), "relabelled, two GPUs against one")
    same(two_x, h.search_exact_label_sets(Q, 10, qs), "relabelled, exact, two GPUs against one")


def test_offsets_and_values_are_checked(pkg):
    """the (offsets, values) form is refused in Python when an offset lies outside values"""
    h = pkg.Hnsw(8, 100, 16, 48, "DistL2")
    Q = np.zeros((3, 8), np.float32)
    vals = np.arange(4, dtype=np.uint32)
    for off in ([0, 1, 2, 5], [-1, 0, 1, 2], [0.0, 1.0, 2.0, 3.0]):
        with pytest.raises(ValueError, match="offsets must be integers"):
            h.search_flat_label_sets(Q, 4, 16, (np.array(off), vals))
        with pytest.raises(ValueError, match="offsets must be integers"):
            h.search_exact_label_sets(Q, 4, (np.array(off), vals))
    with pytest.raises(ValueError, match="4 offsets for 2 queries"):
        h.search_flat_label_sets(Q[:2], 4, 16, (np.array([0, 1, 2, 3]), vals))


def test_refusals_and_edges(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 24, nq=60, seed=10)
    E = pkg.HnswError
    L = pkg.load_library()
    h.set_labels(0, point_labels(N, 10))
    qs = row_sets(np.arange(len(Q)) % len(SETS))
    want, want_x = h.search_flat_label_sets(Q, 10, 64, qs), h.search_exact_label_sets(Q, 10, qs)
    off = np.arange(len(Q) + 1, dtype=np.uint64)
    vals = np.zeros(len(Q), np.uint32)
    bad = off.copy()
    bad[8] = 10   # row 7 is [7, 10), row 8 is [10, 9)
    for call in (lambda s: h.search_flat_label_sets(Q, 10, 64, s), lambda s: h.search_exact_label_sets(Q, 10, s)):
        with pytest.raises(E, match=r"label set 8: qset_off\[9\] = 9 is below qset_off\[8\] = 10"):
            call((bad, np.zeros(len(Q) + 1, np.uint32)))
        mixed = [[1]] * len(Q)
        mixed[5] = [2, NONE, 2]
        mixed[9] = [NONE, 0]
        with pytest.raises(E, match="label set 5 holds LABEL_NONE together with another label"):
            call(mixed)
    out = [np.empty((len(Q), 10), t) for t in (np.uint64, np.float32)] + [np.empty(len(Q), np.int32)]
    p = lambda a: a.ctypes.data_as(pkg.hnsw.C.c_void_p)   # noqa: E731
    assert L.hnsw_b200_search_flat_label_sets(h._h, None, p(vals), p(Q), len(Q), 24, 10, 64, p(out[0]), p(out[1]), None,
                                              None, p(out[2])) < 0
    assert "qset_off is NULL" in pkg.last_error()
    assert L.hnsw_b200_search_exact_label_sets(h._h, p(off), None, p(Q), len(Q), 24, 10, p(out[0]), p(out[1]), None, None,
                                               p(out[2])) < 0
    assert "qset is NULL" in pkg.last_error()
    assert L.hnsw_b200_search_flat_label_sets(h._h, None, None, p(Q), 0, 24, 10, 64, None, None, None, None, None) == 0
    assert L.hnsw_b200_search_exact_label_sets(h._h, None, None, p(Q), 0, 24, 10, None, None, None, None, None) == 0
    assert h.search_flat_label_sets(Q[:0], 10, 64, [])[4].shape == (0,)
    same(h.search_flat_label_sets(Q, 10, 64, qs), want, "after the refused calls")
    same(h.search_exact_label_sets(Q, 10, qs), want_x, "exact, after the refused calls")
    for res in (h.search_flat_label_sets(Q, 10, 64, [[]] * len(Q)), h.search_exact_label_sets(Q, 10, [[]] * len(Q)),
                h.search_flat_label_sets(Q, 10, 64, [[12345, 99]] * len(Q))):
        assert np.all(res[4] == 0) and np.all(res[2] == NONE)
    e = pkg.Hnsw(8, 100, 16, 48, "DistL2")   # an empty index: every count 0
    for res in (e.search_flat_label_sets(Q[:5, :8], 4, 16, qs[:5]), e.search_exact_label_sets(Q[:5, :8], 4, qs[:5])):
        assert np.all(res[4] == 0)

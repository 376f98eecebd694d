"""Radius search (include/hnsw_b200.h "Radius search"): Hnsw.search_exact_radius / search_exact_radius_by_id /
radius_graph, every admitted point within each query's own distance, and how many there are.

Row i must equal the oracle's brute force over the admitted points (ORDER_GPU sums) cut after its last distance <= r_i,
on origin ids, distance bits, internal ids, PointIds and counts, and the search_exact* row of the same restriction cut
on the host.  Totals must equal the number of oracle distances <= r_i.  Radius mode runs inside exact_knn_kernel's
existing instantiations with the k-NN shape and shared memory, which the shape cases check launch by launch."""
import ctypes as C

import numpy as np
import pytest
import torch  # imported first, so that torch's own NCCL is the one the library binds at run time

from answers import same
from exactref import (EXACT_CASES, INVALID, SHAPE_CASES, d4_of, exact_shape, exact_slices, expected, filter_sets, handle,
                      origin_ids, points, shape_case_id, stored_queries, tile_points)
from graphs import case_id, data

pytestmark = pytest.mark.gpu

N, NQ = 1500, 40
NONE = 0xFFFFFFFF
I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
LEDGER = set()  # (pass, tq, rows, stages, S > 1) of every radius launch of the shape cases


def cut(rows, r):
    """search_exact rows cut after each row's last entry with distance <= r[i], padded as an exact call pads"""
    o, d, it, pid, c = (None if x is None else x.copy() for x in rows)
    for i in range(len(c)):
        n = int(np.sum(d[i, :c[i]] <= r[i]))
        o[i, n:], d[i, n:], c[i] = np.iinfo(np.uint64).max, np.inf, n
        if it is not None:
            it[i, n:] = INVALID
        if pid is not None:
            pid[i, n:] = -1
    return o, d, it, pid, c


def all_dists(po, X, Q, metric, adm):
    """[nq, len(adm)] oracle distances of every admitted point, ascending per row"""
    if len(adm) == 0:
        return np.zeros((len(Q), 0), np.float32)
    return po.bruteforce(X[adm], Q, len(adm), metric, po.ORDER_GPU)[1]


def radii(D):
    """one radius per query, cycling through 0, the exact 1st / 10th / 100th distance (bit-equal: the boundary point is
    in), the float just below the 10th (it is out), and +inf"""
    r = np.empty(len(D), np.float32)
    for i in range(len(D)):
        row = D[i]
        at = lambda j: row[min(j, len(row) - 1)] if len(row) else np.float32(1)
        kind = i % 6
        r[i] = [np.float32(0), at(0), at(9), at(99), np.nextafter(at(9), np.float32(0)), np.float32(np.inf)][kind]
    return r


def check_rows(got, want_rows, want_tot, what):
    same(got[:5], want_rows, what)
    assert np.array_equal(got[5], want_tot.astype(np.uint64)), f"{what}: totals"


def labelled(h, n, seed):
    """labels 0 .. 4 and attributes 0 .. 99 on every point; returns them"""
    rng = np.random.default_rng(seed)
    lab = rng.integers(0, 5, n).astype(np.uint32)
    attr = rng.integers(0, 100, n).astype(np.int64)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    return lab, attr


def restrictions(h, n, og, lab, attr, nq):
    """(name, keyword arguments of the radius and k-NN calls, admitted ids of row i, k-NN call) per restriction; the
    per-row ones alternate two restrictions over the rows, so that the rows are sorted and their radii travel with them"""
    every = np.arange(n)
    half = filter_sets(n, 7)["50%"]
    sets = [[1, 3] if i % 2 else [0] for i in range(nq)]
    ranges = [(10, 60) if i % 2 else (I64_MIN, I64_MAX) for i in range(nq)]
    rsets = [[2, 4] if i % 2 else [NONE] for i in range(nq)]
    set_adm = [np.flatnonzero(np.isin(lab, s)) for s in ([0], [1, 3])]
    rng_adm = [every, np.flatnonzero(np.isin(lab, [2, 4]) & (attr >= 10) & (attr <= 60))]
    rf = h.make_filter(og[half])
    return rf, [
        ("none", {}, [every, every], lambda Q, k: h.search_exact(Q, k)),
        ("filter", {"filter": rf}, [half, half], lambda Q, k: h.search_exact(Q, k, filter=rf)),
        ("label sets", {"sets": sets}, set_adm, lambda Q, k: h.search_exact_label_sets(Q, k, sets)),
        ("ranges+sets", {"ranges": ranges, "sets": rsets}, rng_adm,
         lambda Q, k: h.search_exact_ranges(Q, k, ranges, sets=rsets)),
    ]


def oracle(po, h, X, Q, k, metric, adms, r):
    """the oracle's rows (rows i of parity p over adms[p]) cut at r, and its totals"""
    nq = len(Q)
    rows = [np.empty((nq,) + s, t) for s, t in (((k,), np.uint64), ((k,), np.float32), ((k,), np.uint32),
                                                 ((k, 2), np.int32), ((), np.int32))]
    tot = np.zeros(nq, np.int64)
    for p in (0, 1):
        sel = np.arange(p, nq, 2)
        e = expected(po, h, X, Q[sel], k, metric, adms[p])
        for a, b in zip(rows, e):
            a[sel] = b
        tot[sel] = (all_dists(po, X, Q[sel], metric, adms[p]) <= r[sel, None]).sum(1)
    return cut(tuple(rows), r), tot


# ---------------------------------------------------------------- 1. oracle parity
@pytest.mark.parametrize("dtype,metric,d,ties", EXACT_CASES, ids=[case_id(c) for c in EXACT_CASES])
def test_radius_equals_oracle(pkg, po, dtype, metric, d, ties):
    X = data(dtype, metric, N, d, d + 3, ties)
    Q = data(dtype, metric, NQ, d, d + 103)
    Q[: NQ // 10] = X[: NQ // 10]
    h = handle(pkg, X, metric)
    og = origin_ids(N)
    lab, attr = labelled(h, N, d)
    rf, cases = restrictions(h, N, og, lab, attr, NQ)
    with rf:
        for name, kw, adms, knn in cases:
            D = all_dists(po, X, Q, metric, adms[0])
            r = radii(D)
            for k in (1, 10, 128, N + 2):
                want, tot = oracle(po, h, X, Q, k, metric, adms, r)
                got = h.search_exact_radius(Q, r, k, **kw)
                check_rows(got, want, tot, f"{name} k={k}")
                same(got[:5], cut(knn(Q, k), r), f"{name} k={k}: search_exact cut")
            kern = pkg.last_kernel()
            knn(Q, 10)
            assert pkg.last_kernel() == kern, f"{name}: the radius call ran {kern}, the k-NN call {pkg.last_kernel()}"
            # 6. knbn = 0: totals only, through NULL row arrays
            if name in ("none", "filter"):
                cnt = np.full(NQ, 7, np.int32)
                tot0 = np.zeros(NQ, np.uint64)
                assert pkg.load_library().hnsw_b200_search_exact_radius(
                    h._h, kw["filter"].id if kw else -1, None, None, None, Q.ctypes.data_as(C.c_void_p), NQ, d,
                    r.ctypes.data_as(C.c_void_p), 0, None, None, None, None, cnt.ctypes.data_as(C.c_void_p),
                    tot0.ctypes.data_as(C.c_void_p)) == 0, pkg.last_error()
                assert np.all(cnt == 0) and np.array_equal(tot0, got[5]), f"{name}: knbn = 0"
            z = h.search_exact_radius(Q, r, 0, **kw)
            assert np.all(z[4] == 0) and np.array_equal(z[5], got[5]), f"{name}: knbn = 0 (binding)"


# ---------------------------------------------------------------- 3. split launches
def test_split_launches(pkg, po):
    """4 queries over 60 000 points split the scan over many CTAs, whose counts add up in `totals`; the same 4 queries
    inside a 9 000-query batch must give the same rows and totals, and both the oracle's"""
    n, d = 60000, 24
    X = data(np.float32, "DistL2", n, d, 21)
    Q = data(np.float32, "DistL2", 9000, d, 22)
    h = handle(pkg, X, "DistL2")
    every = np.arange(n)
    D = all_dists(po, X, Q[:4], "DistL2", every)
    for j in (9, 99, 999):
        r4 = D[:, j].copy()
        r = np.concatenate([r4, np.full(len(Q) - 4, D[0, 9], np.float32)])
        for k in (10, 100):
            few = h.search_exact_radius(Q[:4], r4, k)
            want = cut(expected(po, h, X, Q[:4], k, "DistL2", every), r4)
            check_rows(few, want, (D <= r4[:, None]).sum(1), f"4 queries, radius at {j + 1}, k={k}")
            many = h.search_exact_radius(Q, r, k)
            same(tuple(x[:4] for x in many[:5]), few[:5], f"9000 queries, k={k}")
            assert np.array_equal(many[5][:4], few[5])


# ---------------------------------------------------------------- 4. instantiations and shapes
@pytest.mark.parametrize("dtype,metric,d,n,nq,k", SHAPE_CASES, ids=[shape_case_id(c) for c in SHAPE_CASES])
def test_shapes(pkg, po, dtype, metric, d, n, nq, k):
    """a radius launch has the k-NN launch's shape and shared memory (exactref's restatement of
    exact_layout / exact_shape / cost(S), which radius mode does not change) and runs its instantiation; its rows are
    the k-NN rows cut at a radius halfway down them"""
    X = points(dtype, metric, n, d, d + n)
    Q = stored_queries(X, dtype, metric, nq, d + n + 1)
    h = handle(pkg, X, metric)
    knn = h.search_exact(Q, k)
    kern, shape = pkg.last_kernel(), pkg.last_kernel_shape()
    r = knn[1][np.arange(nq), np.maximum(knn[4] // 2 - 1, 0)].copy()
    got = h.search_exact_radius(Q, r, k)
    assert pkg.last_kernel() == kern and pkg.last_kernel_shape() == shape, (pkg.last_kernel_shape(), shape)
    ps, tq, rows, stages, smem = exact_shape(d4_of(d, dtype), k, nq)
    assert shape[0] == smem
    S = exact_slices(tile_points([(nq, n)], tq), torch.cuda.get_device_properties(0).multi_processor_count * shape[2])
    LEDGER.add((ps, tq, rows, stages, S > 1))
    same(got[:5], cut(knn, r), "k-NN rows cut")
    D = all_dists(po, X, Q, metric, np.arange(n)) if n <= 6000 else None
    if D is not None:
        assert np.array_equal(got[5], (D <= r[:, None]).sum(1).astype(np.uint64))
    assert np.all(got[5] >= got[4])


def test_zz_every_shape_was_reached():
    if not LEDGER:
        pytest.skip("no shape case ran")
    assert {e[2] for e in LEDGER} >= {32, 16, 8, 4, 2, 1}, LEDGER
    assert {e[3] for e in LEDGER} >= {3, 2}, LEDGER
    assert {e[0] for e in LEDGER} >= {0, 1}, LEDGER
    assert {e[1] for e in LEDGER} >= {32, 16, 8, 4, 3, 2, 1}, LEDGER
    assert any(e[4] for e in LEDGER), LEDGER


# ---------------------------------------------------------------- 5. by stored point
@pytest.mark.parametrize("metric", ["DistL2", "DistDot"])
def test_by_id(pkg, po, metric):
    """rows equal the host-query call on get_vectors(qids); with exclude_self, search_exact_by_id's exclude_self row cut
    at r, and a total one less exactly when the point is admitted and within r; copies of a point stay"""
    X = data(np.float32, metric, N, 48, 61)
    X[N - 50:] = X[:50]   # points 0 .. 49 each have a copy
    h = handle(pkg, X, metric)
    og = origin_ids(N)
    lab, attr = labelled(h, N, 62)
    q = np.concatenate([np.arange(0, 60), np.random.default_rng(63).choice(N, 40, replace=False)]).astype(np.uint64)
    V = h.get_vectors(q)
    half = filter_sets(N, 64)["50%"]
    with h.make_filter(og[half]) as rf:
        for kw, adm in (({}, np.arange(N)), ({"filter": rf}, half),
                        ({"sets": [[1, 2]] * len(q)}, np.flatnonzero(np.isin(lab, [1, 2]))),
                        ({"ranges": [(20, 70)] * len(q)}, np.flatnonzero((attr >= 20) & (attr <= 70)))):
            D = all_dists(po, X, V, metric, adm)
            r = radii(D)
            full = h.search_exact_radius_by_id(q, r, N, **kw)   # every admitted point within r
            inside = np.array([np.any(full[2][i, :full[4][i]] == q[i]) for i in range(len(q))]).astype(np.uint64)
            for k in (1, 10, 128):
                got = h.search_exact_radius_by_id(q, r, k, **kw)
                same(got[:5], h.search_exact_radius(V, r, k, **kw)[:5], f"{kw.keys()} k={k}: host queries")
                assert np.array_equal(got[5], h.search_exact_radius(V, r, k, **kw)[5])
                ex = h.search_exact_radius_by_id(q, r, k, exclude_self=True, **kw)
                rows = h.search_exact_by_id(q, k, exclude_self=True, **kw)
                same(ex[:5], cut(rows, r), f"{kw.keys()} k={k}: exclude_self")
                assert np.array_equal(got[5] - ex[5], inside), f"{kw.keys()} k={k}: totals without the point itself"
    # copies stay: with r = 0 under L2, each of points 0 .. 49 finds its copy and only it
    if metric == "DistL2":
        got = h.search_exact_radius_by_id(np.arange(50, dtype=np.uint64), 0.0, 4, exclude_self=True)
        assert np.all(got[4] == 1) and np.array_equal(got[2][:, 0], np.arange(N - 50, N)) and np.all(got[5] == 1)


# ---------------------------------------------------------------- 7. refusals
def test_refusals(pkg, po):
    X = data(np.float32, "DistL2", N, 24, 71)
    Q = data(np.float32, "DistL2", 5, 24, 72)
    h = handle(pkg, X, "DistL2")
    L = pkg.load_library()
    vp = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    ids = np.full((5, 10), 7, np.uint64)
    dist = np.full((5, 10), 7, np.float32)
    cnt = np.full(5, 7, np.int32)
    tot = np.full(5, 7, np.uint64)

    def call(r, knbn=10, filter=-1, qset_off=None, qset=None):
        return L.hnsw_b200_search_exact_radius(h._h, filter, None, vp(qset_off), vp(qset), vp(Q), 5, 24, vp(r), knbn,
                                               vp(ids), vp(dist), None, None, vp(cnt), vp(tot))

    ok = np.ones(5, np.float32)
    for r, msg in ((np.array([1, 1, np.nan, 1, 1], np.float32), "radius[2]"),
                   (np.array([1, 1, 1, -0.5, 1], np.float32), "radius[3]"), (None, "radius is NULL")):
        assert call(r) < 0 and msg in pkg.last_error(), pkg.last_error()
    with h.make_filter(origin_ids(N)[:10]) as rf:
        off = np.arange(6, dtype=np.uint64)
        s = np.zeros(5, np.uint32)
        assert call(ok, filter=rf.id, qset_off=off, qset=s) < 0 and "cannot be combined" in pkg.last_error()
    assert call(ok, knbn=10 ** 6) < 0 and "too large" in pkg.last_error(), pkg.last_error()
    assert np.all(ids == 7) and np.all(dist == 7) and np.all(cnt == 7) and np.all(tot == 7), "a refusal wrote output"
    with pytest.raises(pkg.HnswError, match=r"qids\[1\]"):
        h.search_exact_radius_by_id([0, N], 1.0, 4)
    assert call(np.full(5, -0.0, np.float32)) == 0 and np.all(cnt == 0) and np.all(tot == 0)   # -0 is 0
    assert h.search_exact_radius(Q[:0], 1.0, 4)[5].size == 0


# ---------------------------------------------------------------- 8. partitions and replicas
@pytest.mark.parametrize("P", [2, 3])
def test_partitions(pkg, po, P):
    X = data(np.float32, "DistL2", N, 24, 81)
    Q = data(np.float32, "DistL2", NQ, 24, 82)
    ids = origin_ids(N)
    plain = pkg.Hnsw(8, N, 16, 48, "DistL2")
    plain.insert_flat(X, ids=ids)
    ph = pkg.Hnsw(8, N, 16, 48, "DistL2")
    ph.partition([0] * P)
    ph.insert_flat(X, ids=ids)
    r = radii(all_dists(po, X, Q, "DistL2", np.arange(N)))
    for k in (1, 10, 128):
        a = plain.search_exact_radius(Q, r, k, with_pid=False)
        b = ph.search_exact_radius(Q, r, k, with_pid=False)
        for x, y, what in zip(a, b, ("origin", "dist", "internal", "pid", "counts", "totals")):
            if x is not None:
                assert np.array_equal(x, y), (P, k, what)
        q = np.arange(0, N, 37, dtype=np.uint64)
        rq = np.full(q.size, r[2], np.float32)
        a = plain.search_exact_radius_by_id(q, rq, k, exclude_self=True, with_pid=False)
        b = ph.search_exact_radius_by_id(q, rq, k, exclude_self=True, with_pid=False)
        for x, y in zip(a, b):
            if x is not None:
                assert np.array_equal(x, y), (P, k, "by id")
    v = ph.partition_view(0)
    Xp = X[0::P]
    Dp = all_dists(po, Xp, Q, "DistL2", np.arange(len(Xp)))
    got = v.search_exact_radius(Q, r, 10)
    want = cut(expected(po, v, Xp, Q, 10, "DistL2", np.arange(len(Xp))), r)
    same(got[:5], want, "view")
    assert np.array_equal(got[5], (Dp <= r[:, None]).sum(1).astype(np.uint64))


def test_two_gpus_match_one(pkg, po):
    if pkg.load_library().hnsw_b200_device_count() < 2:
        pytest.skip("needs two GPUs")
    X = data(np.float32, "DistL2", 5000, 24, 91)
    Q = data(np.float32, "DistL2", 2000, 24, 92)
    h = handle(pkg, X, "DistL2")
    r = np.full(len(Q), np.median(all_dists(po, X, Q[:50], "DistL2", np.arange(5000))[:, 20]), np.float32)
    want = h.search_exact_radius(Q, r, 32)
    h.replicate([0, 1])
    got = h.search_exact_radius(Q, r, 32)
    for x, y in zip(want, got):
        assert np.array_equal(x, y)


# ---------------------------------------------------------------- 9. radius_graph
def test_radius_graph(pkg, po):
    """3 000 points in tight clusters, so that some points have more than 64 others within r and the re-run path runs;
    the CSR must equal the numpy epsilon-graph of the oracle's full distance matrix"""
    rng = np.random.default_rng(101)
    n, d = 3000, 16
    centres = rng.random((30, d), dtype=np.float32) * 10
    X = (centres[rng.integers(0, 30, n)] + rng.normal(0, 0.05, (n, d))).astype(np.float32)
    h = handle(pkg, X, "DistL2")
    ti, td = po.bruteforce(X, X, n, "DistL2", po.ORDER_GPU)
    r = np.float32(np.median(td[:, 80]))
    off, it, dd = h.radius_graph(r, knbn=64, batch=1000)
    assert off[-1] == len(it) == len(dd)
    big = 0
    for p in range(n):
        keep = (td[p] <= r) & (ti[p] != p)
        lo, hi = int(off[p]), int(off[p + 1])
        assert np.array_equal(it[lo:hi], ti[p][keep]), p
        assert np.array_equal(dd[lo:hi].view(np.uint32), td[p][keep].view(np.uint32)), p
        big += hi - lo > 64
    assert big > 0, "no point had more than 64 others within r"

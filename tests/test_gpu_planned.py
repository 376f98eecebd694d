"""Planned search (include/hnsw_b200.h "Planned search"): Hnsw.count_admitted, search_planned and search_planned_by_id.

count_admitted must equal numpy over the labels and attributes the test set.  Each planned row must take the path the
rule restated here in integers picks, and equal, bit for bit, the row of its defining call: search_flat_excluding or
search_exact_excluding with the same restriction and list (search_by_id or search_exact_by_id by stored point).  Rows
do not depend on the rest of their batch, so the defining rows are taken from one batch call of each.  The graphs are
small (M = 8, ef 1 to 32) so that one batch has rows on both sides of the rule; the labels form a geometric ladder of
sizes 1, 2, 4, ..., 2048, so that a set of ladder labels admits any count up to 4095."""
import ctypes as C
import math
import pathlib
import re

import numpy as np
import pytest
import torch  # imported first, so that torch's own NCCL is the one the library binds at run time

from answers import same
from graphs import data
from util import oracle_layers

pytestmark = pytest.mark.gpu

GAMMA = 23   # HNSW_B200_PLANNED_GAMMA, as the header documents it
N, M, EFC = 6000, 8, 64
NONE = 0xFFFFFFFF
ATTR_NONE = -(1 << 63)
RANGE_ALL = (-(1 << 63), (1 << 63) - 1)
GRID = [(1, 1), (10, 10), (10, 16), (32, 32)]
GRAPHS = [(np.float32, "DistL2", 48), (np.float32, "DistCosine", 100), (np.uint8, "DistHamming", 100)]
HEADER = pathlib.Path(__file__).resolve().parents[1] / "include" / "hnsw_b200.h"


def round128(x):
    return (x + 127) // 128 * 128


def exact_fits(row_bytes, k):
    """the exact scan holds k keys at this row size: its least shape (one query, a ring of two one-row stages) fits the
    220 KB shared-memory budget (kernels.h exact_layout)"""
    d4 = row_bytes // 16
    ring = d4 * 16
    queue = ring + 2 * d4 * 16
    qn = queue + k * 8 + 8 + 8 + 4
    bar = (qn + 4 + 15) & ~15
    return round128(bar + 16) <= 220 * 1024


def rule(c, n, kq, ef, row_bytes):
    """the planned rule: True for the exact scan"""
    return exact_fits(row_bytes, kq) and c * c <= GAMMA * n * max(ef, kq) * 2 * M


def row_bytes_of(dtype, d):
    return round128(d * np.dtype(dtype).itemsize)


def build(pkg, po, dtype, metric, d, seed):
    """an oracle graph (MODE_DET, ORDER_GPU, default ids: origin id = insertion rank) imported into the engine"""
    X = data(dtype, metric, N, d, seed)
    o = po.Oracle(M, N, 16, EFC, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X)
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, N, 16, EFC, metric, dtype=dtype)
    h.import_graph(X, og, lv, o.entry, oracle_layers(o))
    return X, h


def ladder(n, seed):
    """labels: label j (0..11) on 2^j points, label 12 on 1500, the rest none; attributes: the rank, none on every 50th"""
    rng = np.random.default_rng(seed)
    lab = np.full(n, NONE, np.uint32)
    at = 0
    perm = rng.permutation(n)
    for j, size in enumerate([1 << j for j in range(12)] + [1500]):
        lab[perm[at:at + size]] = j
        at += size
    attr = np.arange(n, dtype=np.int64)
    attr[::50] = ATTR_NONE
    return lab, attr


def bits_of(c):
    """the ladder labels whose sizes sum to c (< 4096)"""
    return [j for j in range(12) if (c >> j) & 1]


def restrictions(nq):
    sets = [[[NONE], [0], [3], [6], [8], [10], [11], [12], [], [12, 11], [12, 11, 10, 9], list(range(13)), [3, 7, 11],
             [11, 10, 9]][i % 14] for i in range(nq)]
    ranges = [[RANGE_ALL, (0, 0), (0, 10), (0, 100), (0, 1000), (0, 3000), (0, 5999), (100, 50), (-5, 2000)][i % 9]
              for i in range(nq)]
    return sets, ranges


def mask(lab, attr, s=None, r=None):
    m = np.ones(lab.size, bool)
    if s is not None and list(s) != [NONE]:
        m &= np.isin(lab, np.asarray(s, np.int64))
    if r is not None and tuple(r) != RANGE_ALL:
        m &= (attr >= r[0]) & (attr <= r[1]) & (attr != ATTR_NONE)
    return m


def counts_of(lab, attr, nq, sets=None, ranges=None, filt=None):
    if filt is not None:
        return np.full(nq, filt.size, np.uint64)
    return np.array([mask(lab, attr, None if sets is None else sets[i], None if ranges is None else ranges[i]).sum()
                     for i in range(nq)], np.uint64)


def lists_for(n, nq, seed):
    rng = np.random.default_rng(seed)
    return [[[], [int(rng.integers(n))], rng.choice(n, 30, replace=False).tolist(), rng.choice(n, n // 3).tolist()][i % 4]
            for i in range(nq)]


def pick(ex, exact_rows, graph_rows):
    """row i from exact_rows where ex[i], else from graph_rows"""
    out = []
    for g, x in zip(graph_rows, exact_rows if exact_rows is not None else graph_rows):
        if g is None:
            out.append(None)
            continue
        sel = ex.reshape((-1,) + (1,) * (g.ndim - 1))
        out.append(np.where(sel, x, g))
    return tuple(out)


def planned_want(h, Q, k, ef, lists, kw, counts, n, rb):
    """the defining rows and the rule's out_exact of search_planned(Q, k, ef, lists, **kw)"""
    ex = np.array([rule(int(c), n, k, ef, rb) for c in counts])
    L = lists if lists is not None else [[] for _ in range(len(Q))]
    g = h.search_flat_excluding(Q, k, ef, L, **kw)
    x = h.search_exact_excluding(Q, k, L, **kw) if ex.any() else None
    return pick(ex, x, g), ex.astype(np.int32)


def check_planned(h, Q, k, ef, lists, kw, counts, n, rb, what):
    want, ex = planned_want(h, Q, k, ef, lists, kw, counts, n, rb)
    got = h.search_planned(Q, k, ef, lists, **kw)
    same(got[:5], want, what)
    assert np.array_equal(got[5], ex), f"{what}: out_exact differs from the rule"
    return ex


@pytest.mark.parametrize("dtype,metric,d", GRAPHS, ids=[f"{np.dtype(c[0]).name}-{c[1]}" for c in GRAPHS])
def test_rows_and_routing(pkg, po, dtype, metric, d):
    X, h = build(pkg, po, dtype, metric, d, seed=d)
    lab, attr = ladder(N, d)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    nq = 56
    Q = data(dtype, metric, nq, d, d + 1)
    rb = row_bytes_of(dtype, d)
    sets, ranges = restrictions(nq)
    rng = np.random.default_rng(d)
    small, large = np.sort(rng.choice(N, 300, replace=False)), np.sort(rng.choice(N, 5000, replace=False))
    rfs = [h.make_filter(small.astype(np.uint64)), h.make_filter(large.astype(np.uint64))]
    lists = lists_for(N, nq, d + 2)
    cases = {
        "none": ({}, counts_of(lab, attr, nq)),
        "small filter": ({"filter": rfs[0]}, counts_of(lab, attr, nq, filt=small)),
        "large filter": ({"filter": rfs[1]}, counts_of(lab, attr, nq, filt=large)),
        "sets": ({"sets": sets}, counts_of(lab, attr, nq, sets=sets)),
        "ranges": ({"ranges": ranges}, counts_of(lab, attr, nq, ranges=ranges)),
        "sets and ranges": ({"sets": sets, "ranges": ranges}, counts_of(lab, attr, nq, sets, ranges)),
    }
    both = set()
    for name, (kw, counts) in cases.items():
        assert np.array_equal(h.count_admitted(n=nq, **kw), counts), f"{name}: count_admitted"
        for k, ef in GRID:
            for ls in (None, lists):
                ex = check_planned(h, Q, k, ef, ls, kw, counts, N, rb, f"{name} k={k} ef={ef} lists={ls is not None}")
                if 0 < ex.sum() < nq:
                    both.add(name)
    assert {"sets", "ranges", "sets and ranges"} <= both, f"no batch had rows on both sides: {both}"
    # by stored point, with and without exclude_self
    qids = rng.choice(N, nq, replace=False).astype(np.uint64)
    kw, counts = cases["sets and ranges"]
    for k, ef in ((1, 1), (10, 10), (10, 16)):
        for xs in (False, True):
            ex = np.array([rule(int(c), N, k + xs, ef, rb) for c in counts])
            g = h.search_by_id(qids, k, ef, exclude_self=xs, **kw)
            x = h.search_exact_by_id(qids, k, exclude_self=xs, **kw)
            got = h.search_planned_by_id(qids, k, ef, exclude_self=xs, **kw)
            same(got[:5], pick(ex, x, g), f"by id k={k} ef={ef} exclude_self={xs}")
            assert np.array_equal(got[5], ex), f"by id k={k} ef={ef} exclude_self={xs}: out_exact"
    # statistics: the graph rows' defining calls, the exact rows nothing
    h.enable_stats(True)
    for k, ef in ((10, 10), (1, 1)):
        ex = np.array([rule(int(c), N, k, ef, rb) for c in counts])
        assert 0 < ex.sum() < nq
        h.get_stats()
        h.search_planned(Q, k, ef, lists, **kw)
        got = h.get_stats()
        gr = np.flatnonzero(~ex)
        h.search_flat_excluding(Q[gr], k, ef, [lists[i] for i in gr], sets=[sets[i] for i in gr],
                                ranges=[ranges[i] for i in gr])
        assert got == h.get_stats(), f"stats k={k} ef={ef}"
    h.enable_stats(False)
    for rf in rfs:
        rf.free()


def test_rule_at_the_bound(pkg, po):
    dtype, metric, d = np.float32, "DistL2", 48
    X, h = build(pkg, po, dtype, metric, d, seed=5)
    lab, attr = ladder(N, 5)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    rb = row_bytes_of(dtype, d)
    k = ef = 5
    c0 = math.isqrt(GAMMA * N * ef * 2 * M)
    assert c0 + 1 < 4096
    sets = [bits_of(c0), bits_of(c0 + 1), bits_of(c0 - 1)] * 4
    counts = counts_of(lab, attr, len(sets), sets=sets)
    assert counts[:3].tolist() == [c0, c0 + 1, c0 - 1]
    assert np.array_equal(h.count_admitted(sets=sets), counts)
    Q = data(dtype, metric, len(sets), d, 6)
    ex = check_planned(h, Q, k, ef, None, {"sets": sets}, counts, N, rb, "at the bound")
    assert ex[:3].tolist() == [1, 0, 1], ex
    # with exclude_self, k' = 6 moves the bound
    c1 = math.isqrt(GAMMA * N * 6 * 2 * M)
    qs = [bits_of(c1), bits_of(c1 + 1)]
    got = h.search_planned_by_id(np.array([0, 1], np.uint64), k, ef, sets=qs, exclude_self=True)
    assert got[5].tolist() == [1, 0]


def test_counts(pkg, po):
    X, h = build(pkg, po, np.float32, "DistL2", 48, seed=9)
    lab, attr = ladder(N, 9)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    sets = [[NONE], [], [0], [12], [12, 3, 3, 12], list(range(13))]
    assert h.count_admitted(sets=sets).tolist() == [N, 0, 1, 1500, 1508, int((lab != NONE).sum())]
    ranges = [RANGE_ALL, (0, N), (10, 5), (0, 99), (-100, -1)]
    assert h.count_admitted(ranges=ranges).tolist() == [N, int((attr != ATTR_NONE).sum()), 0, 98, 0]
    nq = 28
    s, r = restrictions(nq)
    assert np.array_equal(h.count_admitted(sets=s, ranges=r), counts_of(lab, attr, nq, s, r))
    assert h.count_admitted(n=3).tolist() == [N] * 3
    adm = np.arange(0, N, 3, dtype=np.uint64)
    rf = h.make_filter(adm)
    assert h.count_admitted(filter=rf, n=2).tolist() == [adm.size] * 2
    # deleted points are counted
    h.delete_points(np.flatnonzero(lab == 12)[:100])
    assert h.count_admitted(sets=[[12]], ranges=[RANGE_ALL]).tolist() == [1500]
    assert h.count_admitted(filter=rf, n=1).tolist() == [adm.size]
    rf.free()


def test_deleted_points(pkg, po):
    dtype, metric, d = np.float32, "DistL2", 48
    X, h = build(pkg, po, dtype, metric, d, seed=11)
    lab, attr = ladder(N, 11)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    rng = np.random.default_rng(12)
    h.delete_points(np.concatenate([rng.choice(N, 600, replace=False), np.flatnonzero(lab <= 4)]))
    nq = 56
    Q = data(dtype, metric, nq, d, 13)
    sets, ranges = restrictions(nq)
    lists = lists_for(N, nq, 14)
    rb = row_bytes_of(dtype, d)
    for kw, counts in (({}, counts_of(lab, attr, nq)), ({"sets": sets, "ranges": ranges}, counts_of(lab, attr, nq, sets, ranges))):
        for k, ef in ((1, 1), (10, 10)):
            for ls in (None, lists):
                check_planned(h, Q, k, ef, ls, kw, counts, N, rb, f"deleted {list(kw)} k={k} ef={ef}")


def test_over_the_exact_limit(pkg):
    d, n = 18600, 400   # f32 rows of 74 496 bytes: the exact scan holds a few hundred keys
    rb = row_bytes_of(np.float32, d)
    limit = max(k for k in range(1, 2000) if exact_fits(rb, k))
    assert 16 < limit < 1000
    X = data(np.float32, "DistL2", n, d, 1)
    h = pkg.Hnsw(M, n, 16, EFC, "DistL2")
    h.insert_flat(X)
    Q = data(np.float32, "DistL2", 4, d, 2)
    sets = [[NONE]] * 4
    for k, want in ((limit, 1), (limit + 1, 0)):
        got = h.search_planned(Q, k, k, sets=sets)
        assert got[5].tolist() == [want] * 4, (k, got[5])
        ref = h.search_exact(Q, k) if want else h.search_flat(Q, k, k)
        same(got[:5], ref, f"k={k}")
    qids = np.arange(4, dtype=np.uint64)
    got = h.search_planned_by_id(qids, limit, limit, exclude_self=True)
    assert got[5].tolist() == [0] * 4
    same(got[:5], h.search_by_id(qids, limit, limit, exclude_self=True), "exclude_self over the limit")
    got = h.search_planned_by_id(qids, limit - 1, limit, exclude_self=True)
    assert got[5].tolist() == [1] * 4
    same(got[:5], h.search_exact_by_id(qids, limit - 1, exclude_self=True), "exclude_self at the limit")


def merge(views, P, k):
    """the partitioned rule: each row's answers of every view by (distance, partition, position), as global ranks"""
    nq = views[0][4].shape[0]
    o = np.full((nq, k), np.iinfo(np.uint64).max, np.uint64)
    dist = np.full((nq, k), np.inf, np.float32)
    it = np.full((nq, k), NONE, np.uint32)
    pid = np.full((nq, k, 2), -1, np.int32)
    cnt = np.zeros(nq, np.int32)
    for i in range(nq):
        e = [(float(v[1][i, j]), p, j) for p, v in enumerate(views) for j in range(v[4][i])]
        e.sort()
        for s, (_, p, j) in enumerate(e[:k]):
            v = views[p]
            o[i, s], dist[i, s], it[i, s], pid[i, s] = v[0][i, j], v[1][i, j], int(v[2][i, j]) * P + p, v[3][i, j]
        cnt[i] = min(k, len(e))
    return o, dist, it, pid, cnt


@pytest.mark.parametrize("P", [2, 3])
def test_partitions_and_views(pkg, P):
    d = 48
    X = data(np.float32, "DistL2", N, d, 31)
    h = pkg.Hnsw(M, N, 16, EFC, "DistL2")
    h.partition([0] * P)
    h.insert_flat(X)
    lab, attr = ladder(N, 32)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    nq = 56
    Q = data(np.float32, "DistL2", nq, d, 33)
    sets, ranges = restrictions(nq)
    rb = row_bytes_of(np.float32, d)
    kw = {"sets": sets, "ranges": ranges}
    total = np.zeros(nq, np.uint64)
    for k, ef in ((1, 1), (10, 10), (10, 16)):
        views, exs = [], np.zeros(nq, np.int32)
        for p in range(P):
            v = h.partition_view(p)
            nv = v.get_nb_point()
            vlab, vattr = v.get_labels(0, nv), v.get_attributes(0, nv)
            counts = counts_of(vlab, vattr, nq, sets, ranges)
            assert np.array_equal(v.count_admitted(**kw), counts), f"view {p}: count_admitted"
            if k == 1:
                total += counts
            exs += check_planned(v, Q, k, ef, None, kw, counts, nv, rb, f"P={P} view {p} k={k} ef={ef}")
            views.append(v.search_planned(Q, k, ef, **kw)[:5])
        got = h.search_planned(Q, k, ef, **kw)
        same(got[:5], merge(views, P, k), f"P={P} k={k} ef={ef}: the merge of the views")
        assert np.array_equal(got[5], exs), f"P={P} k={k} ef={ef}: out_exact is the views' sum"
    assert np.array_equal(h.count_admitted(**kw), total), "the handle's count is its views' sum"
    assert np.array_equal(total, counts_of(lab, attr, nq, sets, ranges))


def test_replicas(pkg, po):
    if torch.cuda.device_count() < 2:
        pytest.skip("replicas need two GPUs: not run")
    X, h = build(pkg, po, np.float32, "DistL2", 48, seed=21)
    lab, attr = ladder(N, 21)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    Q = data(np.float32, "DistL2", 400, 48, 22)
    sets, ranges = restrictions(400)
    lists = lists_for(N, 400, 23)
    want = h.search_planned(Q, 10, 10, lists, sets=sets, ranges=ranges)
    assert 0 < want[5].sum() < 400
    h.replicate([0, 1])
    got = h.search_planned(Q, 10, 10, lists, sets=sets, ranges=ranges)
    same(got[:5], want[:5], "replicated")
    assert np.array_equal(got[5], want[5])


def test_edges_and_refusals(pkg, po):
    e = pkg.Hnsw(M, 100, 16, EFC, "DistL2")
    Q = data(np.float32, "DistL2", 3, 24, 48)
    got = e.search_planned(Q, 5, 10)
    assert got[4].tolist() == [0, 0, 0] and got[5].tolist() == [1, 1, 1]
    assert e.count_admitted(n=2).tolist() == [0, 0]
    X = data(np.float32, "DistL2", 1000, 24, 47)
    h = pkg.Hnsw(M, 1000, 16, EFC, "DistL2")
    h.insert_flat(X)
    assert all(a.shape[0] == 0 for a in h.search_planned(Q[:0], 5, 10) if a is not None)
    L = h._L
    p = lambda a: a.ctypes.data_as(C.c_void_p)   # noqa: E731

    def call(off=None, ids=None, filter=-1, rg=None, so=None, sv=None, nq=3, handle=None, by_id=None, exact_out=True):
        """the raw C call on outputs filled with a sentinel; returns (rc, message, whether they stayed)"""
        ans = [np.full((3, 10), 7, np.uint64), np.full((3, 10), 7, np.float32), np.full((3, 10), 7, np.uint32),
               np.full((3, 10, 2), 7, np.int32), np.full(3, 7, np.int32), np.full(3, 7, np.int32)]
        hh = handle if handle is not None else h._h
        if by_id is None:
            rc = L.hnsw_b200_search_planned(hh, off, ids, filter, rg, so, sv, p(Q), nq, 24, 10, 16, *map(p, ans))
        else:
            rc = L.hnsw_b200_search_planned_by_id(hh, by_id, nq, 10, 16, 0, filter, rg, so, sv, *map(p, ans))
        return rc, pkg.last_error(), all(np.all(a == np.array(7).astype(a.dtype)) for a in ans)

    off = np.array([0, 1, 3, 3], np.uint64)
    ids = np.array([5, 9, 2], np.uint64)
    assert call(p(off), p(ids))[0] == 0
    assert call()[0] == 0
    rc, msg, kept = call(handle=C.c_void_p(0))
    assert rc != 0 and "NULL handle" in msg and kept
    assert call(nq=0)[0] == 0
    rc, msg, kept = call(None, p(ids))
    assert rc != 0 and "qx_off is NULL" in msg and kept
    rc, msg, kept = call(p(off), None)
    assert rc != 0 and "qx is NULL" in msg and kept
    rc, msg, kept = call(p(np.array([0, 2, 1, 3], np.uint64)), p(ids))
    assert rc != 0 and "excluded list 1: qx_off[2] = 1 is below qx_off[1] = 2" in msg and kept, msg
    rc, msg, kept = call(p(off), p(np.array([5, 9, 1004], np.uint64)))
    assert rc != 0 and "excluded list 1: qx[2] = 1004 is not below nb_point = 1000" in msg and kept, msg
    rf = h.make_filter(np.arange(0, 1000, 2, dtype=np.uint64))
    so, sv = np.array([0, 1, 2, 3], np.uint64), np.array([1, 2, 3], np.uint32)
    rc, msg, kept = call(filter=rf.id, so=p(so), sv=p(sv))
    assert rc != 0 and "cannot be combined" in msg and kept
    rc, msg, kept = call(so=p(np.array([0, 2, 1, 3], np.uint64)), sv=p(sv))
    assert rc != 0 and "label set 1" in msg and kept, msg
    rf.free()
    rc, msg, kept = call(filter=123456)
    assert rc != 0 and "filter 123456 is not a live filter" in msg and kept, msg
    rc = L.hnsw_b200_search_planned_by_id(h._h, None, 3, 10, 16, 0, -1, None, None, None,
                                           *map(p, h._answers(3, 10, True, True)), None)
    assert rc != 0 and "qids is NULL" in pkg.last_error()
    rc, msg, kept = call(by_id=p(np.array([0, 1, 1000], np.uint64)))
    assert rc != 0 and "qids[2] = 1000 is not below nb_point = 1000" in msg and kept, msg
    # count_admitted refuses as the calls do and leaves out_count untouched
    out = np.full(3, 7, np.uint64)
    assert L.hnsw_b200_count_admitted(h._h, 123456, None, None, None, 3, p(out)) != 0
    assert "filter 123456 is not a live filter" in pkg.last_error() and np.all(out == 7)
    assert L.hnsw_b200_count_admitted(h._h, -1, None, p(np.array([0, 2, 1, 3], np.uint64)), p(sv), 3, p(out)) != 0
    assert "label set 1" in pkg.last_error() and np.all(out == 7)
    assert L.hnsw_b200_count_admitted(None, -1, None, None, None, 3, p(out)) != 0 and np.all(out == 7)
    assert L.hnsw_b200_count_admitted(h._h, -1, None, None, None, 0, None) == 0
    # a stale filter: refused with the wording of the filtered calls
    h2 = pkg.Hnsw(M, 1004, 16, EFC, "DistL2")
    h2.insert_flat(X)
    rf2 = h2.make_filter(np.arange(1000, dtype=np.uint64))
    h2.insert_flat(X[:1])
    with pytest.raises(pkg.HnswError) as e1:
        h2.search_planned(Q, 10, 16, filter=rf2)
    with pytest.raises(pkg.HnswError) as e2:
        h2.search_flat(Q, 10, 16, filter=rf2)
    assert str(e1.value) == str(e2.value)
    with pytest.raises(pkg.HnswError) as e3:
        h2.count_admitted(filter=rf2, n=1)
    assert str(e3.value) == str(e2.value)
    rf2.free()


def test_gamma_is_the_header_value():
    m = re.search(r"#define HNSW_B200_PLANNED_GAMMA (\d+)", HEADER.read_text())
    assert m and int(m.group(1)) == GAMMA

"""Deleted points (include/hnsw_b200.h "Deleted points"): Hnsw.delete_points, restore_points, deleted, nb_deleted.

Unrestricted graph rows are checked bit for bit against the live-search reference (liveref.py, itself checked against
the oracle by test_liveref_cpu.py), counters included.  Restricted and exact rows must equal the same call under a
resident filter that admits exactly the row's points minus the deleted ones.  The graphs are oracle-built and imported
with default ids, so that an origin id (what a resident filter is made of) is the insertion rank (what delete takes)."""
import numpy as np
import pytest
import torch  # imported first, so that torch's own NCCL is the one the library binds at run time

from answers import device_answers, same, same_host_device
from graphs import data
from liveref import LiveRef
from restrict import deleted_set
from util import oracle_layers

pytestmark = pytest.mark.gpu

N, M, EFC, NQ = 1500, 8, 64, 24
GRID = [(1, 1), (10, 10), (10, 64), (64, 200)]
GRAPHS = [(np.float32, "DistL2", 48), (np.float32, "DistCosine", 100), (np.uint8, "DistHamming", 100)]
SETS = ["one", "entry", "top5", "tenth", "half", "all_but_one", "all"]


def build(pkg, po, dtype, metric, d, seed=3):
    X = data(dtype, metric, N, d, seed)
    o = po.Oracle(M, N, 16, EFC, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X)
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, N, 16, EFC, metric, dtype=dtype)
    h.import_graph(X, og, lv, o.entry, oracle_layers(o))
    Q = data(dtype, metric, NQ, d, seed + 100)
    return X, Q, o, h


def live_of(n, dead):
    keep = np.ones(n, bool)
    keep[dead] = False
    return keep


def no_deleted(got, dead, what):
    ids, cnt = got[2], got[4]
    for i in range(len(cnt)):
        assert not np.isin(ids[i, :cnt[i]], dead).any(), f"{what}: row {i} returns a deleted point"


@pytest.mark.parametrize("kind", SETS)
@pytest.mark.parametrize("dtype,metric,d", GRAPHS, ids=[g[1] for g in GRAPHS])
def test_live_rows_against_reference(pkg, po, dtype, metric, d, kind):
    X, Q, o, h = build(pkg, po, dtype, metric, d)
    ref = LiveRef(po, o, X, metric)
    dead = deleted_set(po, kind, X, Q, metric, o.entry)
    h.delete_points(dead)
    assert h.nb_deleted() == len(dead)
    assert np.array_equal(np.flatnonzero(h.deleted()), dead)
    admit = live_of(N, dead)
    q_dev = torch.from_numpy(Q).cuda()
    for k, ef in GRID:
        want, cw = ref.batch(Q, k, ef, admit, live=True)
        what = f"{metric} {kind} k={k} ef={ef}"
        h.enable_stats(True)
        h.get_stats()
        got = h.search_flat(Q, k, ef)
        cg = h.get_stats()
        h.enable_stats(False)
        assert "search_filter_kernel" in pkg.last_kernel(), (what, pkg.last_kernel())
        same(got, want, what)
        no_deleted(got, dead, what)
        if cg["queries"] == NQ:  # a launch re-run after a visited-table overflow counts its work twice
            for key in ("evals", "expansions", "adj_read"):
                assert cg[key] == cw[key], (what, key, cg, cw)
        t = h.submit_flat(Q, k, ef)
        same(h.wait_flat(t), want, what + " submit")
        if dtype == np.float32:
            rows = h.parallel_search([Q[i] for i in range(NQ)], k, ef)
            for i, r in enumerate(rows):
                assert [n.d_id for n in r] == list(want[0][i, :want[4][i]]), (what, "parallel_search", i)
            one = h.search(Q[0], k, ef)
            assert [n.d_id for n in one] == list(want[0][0, :want[4][0]]), (what, "search_neighbours")
        out = torch.empty((NQ, k, 16), dtype=torch.uint8, device="cuda")
        cnt = torch.empty((NQ,), dtype=torch.int32, device="cuda")
        h.search_device(q_dev.data_ptr(), NQ, k, ef, out.data_ptr(), cnt.data_ptr(), sync=True)
        same_host_device(want, device_answers(out, cnt), what + " device")


def twin(pkg, o, X, metric, dtype):
    """a handle on the same oracle graph with no point deleted: the reference rows do not go through the bitmap"""
    lv, rk, og = o.export_points()
    t = pkg.Hnsw(M, N, 16, EFC, metric, dtype=dtype)
    t.import_graph(X, og, lv, o.entry, oracle_layers(o))
    return t


def per_row_filters(t, adm, dead):
    """per row a resident filter of t over its admitted points minus the deleted ones, or None for an unrestricted row"""
    return [None if a is None else t.make_filter(np.setdiff1d(a, dead).astype(np.uint64)) for a in adm]


def free(rfs):
    for rf in rfs:
        if rf is not None:
            rf.free()


def by_filters(t, Q, rfs, k, ef=None, exact=False, qids=None, exclude_self=False, live=None):
    """row i of the single-filter call on t under rfs[i]; an unrestricted graph row (rfs[i] None) is live's own row"""
    parts = []
    for i, rf in enumerate(rfs):
        h = live if rf is None else t
        if qids is not None:
            q = qids[i:i + 1]
            parts.append(h.search_exact_by_id(q, k, filter=rf, exclude_self=exclude_self) if exact else
                         h.search_by_id(q, k, ef, filter=rf, exclude_self=exclude_self))
        else:
            q = Q[i:i + 1]
            parts.append(h.search_exact(q, k, filter=rf) if exact else h.search_flat(q, k, ef, filter=rf))
    return tuple(np.concatenate([p[j] for p in parts]) for j in range(5))


@pytest.mark.parametrize("dtype,metric,d", GRAPHS, ids=[g[1] for g in GRAPHS])
def test_restricted_and_exact_rows(pkg, po, dtype, metric, d):
    X, Q, o, h = build(pkg, po, dtype, metric, d)
    t = twin(pkg, o, X, metric, dtype)
    rng = np.random.default_rng(5)
    labels = rng.integers(0, 4, N).astype(np.uint32)
    attrs = rng.integers(0, 100, N).astype(np.int64)
    for x in (h, t):
        x.set_labels(0, labels)
        x.set_attributes(0, attrs)
    dead = deleted_set(po, "half", X, Q, metric, o.entry)
    h.delete_points(dead)
    assert t.nb_deleted() == 0
    qlab = (np.arange(NQ) % 4).astype(np.uint32)
    ranges = [(10 * (i % 5), 10 * (i % 5) + 60) for i in range(NQ)]
    allow = np.sort(rng.choice(N, N // 3, replace=False))
    excl = [rng.choice(N, 30, replace=False) for _ in range(NQ)]
    k, ef = 10, 64
    rf_allow = h.make_filter(allow.astype(np.uint64))
    sets = [[int(qlab[i]), int((qlab[i] + 1) % 4)] for i in range(NQ)]
    cases = {
        "filter_t": ([allow] * NQ, lambda ex: (h.search_exact(Q, k, filter=rf_allow) if ex else
                                               h.search_flat(Q, k, ef, filter=allow))),
        "resident": ([allow] * NQ, lambda ex: (h.search_exact(Q, k, filter=rf_allow) if ex else
                                               h.search_flat(Q, k, ef, filter=rf_allow))),
        "per_query": ([allow if i % 2 else None for i in range(NQ)],
                      lambda ex: (h.search_exact_per_query if ex else
                                  lambda *a: h.search_flat_per_query(a[0], a[1], ef, a[2]))(
                          Q, k, [rf_allow if i % 2 else None for i in range(NQ)])),
        "labeled": ([np.flatnonzero(labels == qlab[i]) for i in range(NQ)],
                    lambda ex: h.search_exact_labeled(Q, k, qlab) if ex else h.search_flat_labeled(Q, k, ef, qlab)),
        "label_sets": ([np.flatnonzero(np.isin(labels, sets[i])) for i in range(NQ)],
                       lambda ex: (h.search_exact_label_sets(Q, k, sets) if ex else
                                   h.search_flat_label_sets(Q, k, ef, sets))),
        "ranges": ([np.flatnonzero((attrs >= lo) & (attrs <= hi)) for lo, hi in ranges],
                   lambda ex: h.search_exact_ranges(Q, k, ranges) if ex else h.search_flat_ranges(Q, k, ef, ranges)),
        "excluding": ([np.setdiff1d(np.arange(N), e) for e in excl],
                      lambda ex: (h.search_exact_excluding(Q, k, excl) if ex else
                                  h.search_flat_excluding(Q, k, ef, excl))),
    }
    for name, (adm, call) in cases.items():
        for exact in (False, True):
            # an unrestricted exact row scans the live points; an unrestricted graph row is a live row of h
            rfs = per_row_filters(t, [np.arange(N) if a is None and exact else a for a in adm], dead)
            got = call(exact)
            same(got, by_filters(t, Q, rfs, k, ef, exact, live=h), f"{metric} {name} exact={exact}")
            no_deleted(got, dead, f"{metric} {name} exact={exact}")
            free(rfs)
    # traversal counters of restricted rows, statistics on: those of the reference calls, when nothing was re-run
    rfs = per_row_filters(t, [allow] * NQ, dead)
    for x in (h, t):
        x.enable_stats(True)
        x.get_stats()
    h.search_flat(Q, k, ef, filter=rf_allow)
    cg = h.get_stats()
    by_filters(t, Q, rfs, k, ef)
    cw = t.get_stats()
    for x in (h, t):
        x.enable_stats(False)
    if cg["queries"] == NQ and cw["queries"] == NQ:  # a launch re-run after a visited-table overflow counts twice
        for key in ("evals", "expansions", "adj_read"):
            assert cg[key] == cw[key], (metric, "restricted counters", key, cg, cw)
    free(rfs)
    # by stored point, deleted query ids included, with and without exclude_self, under a resident filter and without
    qids = np.concatenate([dead[:NQ // 2], np.setdiff1d(np.arange(N), dead)[:NQ // 2]]).astype(np.uint64)
    for ex_self in (False, True):
        rfs = per_row_filters(t, [allow] * NQ, dead)
        for exact in (False, True):
            got = (h.search_exact_by_id(qids, k, filter=rf_allow, exclude_self=ex_self) if exact else
                   h.search_by_id(qids, k, ef, filter=rf_allow, exclude_self=ex_self))
            same(got, by_filters(t, None, rfs, k, ef, exact, qids, ex_self), f"{metric} by_id self={ex_self} {exact}")
        free(rfs)
        # without a restriction: exact rows are the resident-filter rows over the live points
        rfs = per_row_filters(t, [np.arange(N)] * NQ, dead)
        got = h.search_exact_by_id(qids, k, exclude_self=ex_self)
        same(got, by_filters(t, None, rfs, k, ef, True, qids, ex_self), f"{metric} exact by_id self={ex_self}")
        free(rfs)
    # without a restriction, graph rows by stored point are live rows: the reference's on the stored vectors
    ref = LiveRef(po, o, X, metric)
    want, _ = ref.batch(X[qids.astype(np.int64)], k, ef, live_of(N, dead), live=True)
    same(h.search_by_id(qids, k, ef), want, f"{metric} live by_id")
    assert "search_filter_kernel" in pkg.last_kernel()
    # unrestricted exact rows, the device-resident twins, and float64 brute force over the live points
    live_rf = t.make_filter(np.setdiff1d(np.arange(N), dead).astype(np.uint64))
    want = t.search_exact(Q, k, filter=live_rf)
    same(h.search_exact(Q, k), want, f"{metric} exact")
    q_dev = torch.from_numpy(Q).cuda()
    out = torch.empty((NQ, k, 16), dtype=torch.uint8, device="cuda")
    cnt = torch.empty((NQ,), dtype=torch.int32, device="cuda")
    h.search_exact_device(q_dev.data_ptr(), NQ, k, out.data_ptr(), cnt.data_ptr(), sync=True)
    same_host_device(want, device_answers(out, cnt), f"{metric} exact device")
    rfs = per_row_filters(t, [allow] * NQ, dead)
    wf = by_filters(t, Q, rfs, k, ef)
    h.search_device(q_dev.data_ptr(), NQ, k, ef, out.data_ptr(), cnt.data_ptr(), sync=True, filter=rf_allow)
    same_host_device(wf, device_answers(out, cnt), f"{metric} device filtered")
    free(rfs)
    if dtype == np.float32:
        live = np.setdiff1d(np.arange(N), dead)
        Xd = X[live].astype(np.float64)
        for i in range(NQ):
            if metric == "DistL2":
                dd = np.sqrt(((Xd - Q[i].astype(np.float64)) ** 2).sum(1))
            else:
                qn = Q[i].astype(np.float64)
                dd = 1 - Xd @ qn / (np.linalg.norm(Xd, axis=1) * np.linalg.norm(qn))
            best = live[np.argsort(dd, kind="stable")[:k]]
            assert len(set(best) & set(want[2][i].tolist())) >= k - 1, (metric, i)
    # radius rows and totals, by vector and by stored point
    radius = np.full(NQ, float(np.median(want[1][:, -1])), np.float32)
    got = h.search_exact_radius(Q, radius, k)
    ref_r = t.search_exact_radius(Q, radius, k, filter=live_rf)
    same(got[:5], ref_r[:5], f"{metric} radius")
    assert np.array_equal(got[5], ref_r[5]), f"{metric} radius totals"
    got = h.search_exact_radius_by_id(qids, radius, k)
    ref_r = t.search_exact_radius_by_id(qids, radius, k, filter=live_rf)
    same(got[:5], ref_r[:5], f"{metric} radius by id")
    assert np.array_equal(got[5], ref_r[5]), f"{metric} radius by id totals"
    live_rf.free()
    rf_allow.free()


def test_restore_gives_back_every_answer(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 48)
    k, ef = 10, 64
    before = {"flat": h.search_flat(Q, k, ef), "exact": h.search_exact(Q, k)}
    kinds = {}
    h.search_flat(Q, k, ef)
    kinds["lean"] = pkg.last_kernel()
    h.set_tie_mode(1)
    before["std"] = h.search_flat(Q, k, ef)
    kinds["std"] = pkg.last_kernel()
    h.set_tie_mode(0)
    before["generic"] = h.search_flat(Q, k, 300)
    kinds["generic"] = pkg.last_kernel()
    dead = deleted_set(po, "tenth", X, Q, "DistL2", o.entry)
    h.delete_points(dead)
    h.delete_points(dead)  # a repeat does nothing
    assert h.nb_deleted() == len(dead)
    h.search_flat(Q, k, ef)
    assert "search_filter_kernel" in pkg.last_kernel()
    h.restore_points(dead)
    h.restore_points(dead[:3])  # restoring a live point does nothing
    assert h.nb_deleted() == 0 and not h.deleted().any()
    same(h.search_flat(Q, k, ef), before["flat"], "flat after restore")
    assert pkg.last_kernel() == kinds["lean"]
    same(h.search_exact(Q, k), before["exact"], "exact after restore")
    h.set_tie_mode(1)
    same(h.search_flat(Q, k, ef), before["std"], "std after restore")
    assert pkg.last_kernel() == kinds["std"]
    h.set_tie_mode(0)
    same(h.search_flat(Q, k, 300), before["generic"], "generic after restore")
    assert pkg.last_kernel() == kinds["generic"]


def test_inserts_after_delete(pkg, po):
    d = 48
    X = data(np.float32, "DistL2", N + 300, d, 9)
    o = po.Oracle(M, N + 300, 16, EFC, "DistL2", d, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X[:N])
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, N + 300, 16, EFC, "DistL2")
    h.import_graph(X[:N], og, lv, o.entry, oracle_layers(o))
    Q = data(np.float32, "DistL2", NQ, d, 10)
    before = np.setdiff1d(np.arange(N), [5, 7])
    rf = h.make_filter(before.astype(np.uint64))
    dead = deleted_set(po, "tenth", X[:N], Q, "DistL2", o.entry)
    h.delete_points(dead)
    # the resident filter made before the delete is not stale: its rows are its rows minus the deleted points
    rows = h.search_flat(Q, 10, 64, filter=rf)
    no_deleted(rows, dead, "old filter")
    rf2 = h.make_filter(np.setdiff1d(before, dead).astype(np.uint64))
    same(rows, h.search_flat(Q, 10, 64, filter=rf2), "old filter rows")
    rf.free()
    rf2.free()
    plain = pkg.Hnsw(M, N + 300, 16, EFC, "DistL2")
    plain.import_graph(X[:N], og, lv, o.entry, oracle_layers(o))
    levels = o.draw_levels(300)
    h.insert_flat(X[N:], levels=levels)
    plain.insert_flat(X[N:], levels=levels)
    for layer in range(16):
        a, b = h.export_layer(layer), plain.export_layer(layer)
        for x, y in zip(a, b):
            assert np.array_equal(x, y), f"layer {layer} differs from the graph built without deletions"
    got = h.deleted()
    assert len(got) == N + 300 and np.array_equal(np.flatnonzero(got), dead)
    ex = h.search_exact(X[N:N + 50], 1)
    assert np.array_equal(ex[2][:, 0], np.arange(N, N + 50)), "a new point is live"


@pytest.mark.parametrize("P", [2, 3])
def test_partitioned(pkg, po, P):
    d = 48
    X = data(np.float32, "DistL2", N, d, 12)
    Q = data(np.float32, "DistL2", NQ, d, 13)
    h = pkg.Hnsw(M, N, 16, EFC, "DistL2")
    h.partition([0] * P)
    h.insert_flat(X)
    dead = deleted_set(po, "tenth", X, Q, "DistL2", 0)
    h.delete_points(dead)
    assert h.nb_deleted() == len(dead)
    assert np.array_equal(np.flatnonzero(h.deleted()), dead)
    k, ef = 10, 64
    got = h.search_flat(Q, k, ef)
    no_deleted(got, dead, f"P={P}")
    # exact rows: an unpartitioned handle of the same points, none deleted, under a filter of the live points
    t = pkg.Hnsw(M, N, 16, EFC, "DistL2")
    t.insert_flat(X)
    with t.make_filter(np.setdiff1d(np.arange(N), dead).astype(np.uint64)) as live_rf:
        want = t.search_exact(Q, k, filter=live_rf)
        ge = h.search_exact(Q, k)
        assert np.array_equal(ge[4], want[4]) and np.array_equal(ge[2], want[2]), f"P={P} exact ids"
        assert np.array_equal(ge[1].view(np.uint32), want[1].view(np.uint32)), f"P={P} exact distances"
    # the merge: each row is the partitions' live rows merged by (distance, partition, position), with global ranks
    views = [h.partition_view(p) for p in range(P)]
    rows = [v.search_flat(Q, k, ef) for v in views]
    for i in range(NQ):
        cand = sorted((rows[p][1][i, j], p, j) for p in range(P) for j in range(rows[p][4][i]))[:k]
        assert got[4][i] == len(cand), (P, i, "count")
        for j, (dj, p, pos) in enumerate(cand):
            assert got[2][i, j] == rows[p][2][i, pos] * P + p, (P, i, j, "merged id")
            assert got[1][i, j].view(np.uint32) == rows[p][1][i, pos].view(np.uint32), (P, i, j, "merged distance")
    for p in range(P):
        v = h.partition_view(p)
        local = dead[dead % P == p] // P
        assert np.array_equal(np.flatnonzero(v.deleted()), local)
        assert v.nb_deleted() == len(local)
        r = v.search_flat(Q, k, ef)
        no_deleted(r, local, f"view {p}")
        with pytest.raises(pkg.HnswError):
            v.delete_points([0])
        with pytest.raises(pkg.HnswError):
            v.restore_points([0])
        assert v.nb_deleted() == len(local)
    h.restore_points(dead)
    assert h.nb_deleted() == 0


def test_replicas(pkg, po):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    d = 48
    X = data(np.float32, "DistL2", N, d, 14)
    Q = data(np.float32, "DistL2", 512, d, 15)
    h = pkg.Hnsw(M, N + 100, 16, EFC, "DistL2")
    h.insert_flat(X)
    one = pkg.Hnsw(M, N + 100, 16, EFC, "DistL2")
    lv, rk, og, entry = h.export_points()
    one.import_graph(X, og, lv, entry, [h.export_layer(l) for l in range(16)])
    h.replicate([0, 1])
    dead = deleted_set(po, "tenth", X, Q, "DistL2", entry)
    h.delete_points(dead)
    one.delete_points(dead)
    same(h.search_flat(Q, 10, 64), one.search_flat(Q, 10, 64), "sharded after delete")
    extra = data(np.float32, "DistL2", 100, d, 16)
    lv2 = np.zeros(100, np.int32)
    h.insert_flat(extra, levels=lv2)
    one.insert_flat(extra, levels=lv2)
    same(h.search_flat(Q, 10, 64), one.search_flat(Q, 10, 64), "sharded after insert")


def test_refusals(pkg, po):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 48)
    h.delete_points([3])
    L = pkg.load_library()
    assert L.hnsw_b200_delete_points(None, None, 0) != 0
    assert L.hnsw_b200_restore_points(None, None, 0) != 0
    assert L.hnsw_b200_get_nb_deleted(None) == -1
    assert L.hnsw_b200_delete_points(h._h, None, 2) != 0
    assert "ranks is NULL" in pkg.last_error()
    with pytest.raises(pkg.HnswError, match=r"ranks\[1\] = 1500 is not below nb_point = 1500"):
        h.delete_points([4, N, 5])
    with pytest.raises(pkg.HnswError):
        h.restore_points([N + 7])
    with pytest.raises(pkg.HnswError):
        h.deleted(N - 1, 2)
    assert L.hnsw_b200_delete_points(h._h, None, 0) == 0
    assert np.array_equal(np.flatnonzero(h.deleted()), [3]) and h.nb_deleted() == 1


def test_dump_keeps_every_point(pkg, po, tmp_path):
    X, Q, o, h = build(pkg, po, np.float32, "DistL2", 48)
    h.file_dump(tmp_path, "plain")
    h.delete_points(np.arange(0, N, 3))
    h.file_dump(tmp_path, "deleted")
    for name in ("plain", "deleted"):
        assert (tmp_path / f"{name}.hnsw.data").stat().st_size > 0
    a = (tmp_path / "plain.hnsw.graph").read_bytes(), (tmp_path / "plain.hnsw.data").read_bytes()
    b = (tmp_path / "deleted.hnsw.graph").read_bytes(), (tmp_path / "deleted.hnsw.data").read_bytes()
    assert a == b, "a dump after a delete differs from the dump without deletions"
    r = pkg.Hnsw.load(str(tmp_path), "deleted", "DistL2")
    assert r.get_nb_point() == N and r.nb_deleted() == 0
    same(r.search_flat(Q, 10, 64), pkg.Hnsw.load(str(tmp_path), "plain", "DistL2").search_flat(Q, 10, 64), "reload")

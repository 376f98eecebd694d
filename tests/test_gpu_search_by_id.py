"""Search by stored point (include/hnsw_b200.h "Search by stored point"): Hnsw.get_vectors, get_point_data,
search_by_id, search_exact_by_id, search_device_by_id and knn_graph.

Row i of a by-id call must equal, bit for bit, the host-query call on get_vectors(qids[i]) (ids, distance bits, internal
ids, PointIds, counts, and with statistics on the traversal counters), served by the same kernel instantiation.  With
exclude_self it must equal that call with knbn + 1, without the point's own entry (or without the last entry when the
row does not hold the point), cut to knbn; that rule is computed here in numpy."""
import numpy as np
import pytest
import torch  # device buffers; imported first, so that torch's own NCCL is the one the library binds at run time

from answers import same
from exactref import expected, origin_ids
from graphs import data
from restrict import minus_self
from util import oracle_layers

pytestmark = pytest.mark.gpu

N, M, EFC = 1200, 8, 64
NONE = 0xFFFFFFFF


def build(pkg, po, dtype, metric, d, seed, ties=False, n=N):
    """an oracle graph (MODE_DET, ORDER_GPU) imported into the engine; ties: every vector stored 4 times"""
    X = data(dtype, metric, n, d, seed, ties)
    o = po.Oracle(M, n, 16, EFC, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X, ids=origin_ids(n))
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, n + 16, 16, EFC, metric, dtype=dtype)
    h.import_graph(X, og, lv, o.entry, oracle_layers(o))
    return X, o, h


def some_ids(n, seed, count=80):
    """distinct ranks in random order, then a few repeated, then the first and the last point"""
    rng = np.random.default_rng(seed)
    q = rng.choice(n, count, replace=False)
    return np.concatenate([q, q[:5], [0, n - 1]]).astype(np.uint64)


F32_CASES = [(np.float32, m, d) for m in ("DistL1", "DistL2", "DistDot", "DistCosine") for d in (24, 48, 100, 150)]
INT_CASES = [(np.uint8, "DistL2", 128), (np.uint8, "DistL2", 512), (np.uint16, "DistL2", 64), (np.uint16, "DistL2", 256),
             (np.uint32, "DistL1", 24), (np.int32, "DistL2", 24)]
CASES = F32_CASES + INT_CASES


@pytest.mark.parametrize("dtype,metric,d", CASES, ids=[f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}" for c in CASES])
def test_rows_equal_host_queries(pkg, po, dtype, metric, d):
    X, o, h = build(pkg, po, dtype, metric, d, seed=d + 3)
    qids = some_ids(N, d)
    V = h.get_vectors(qids)
    assert np.array_equal(V, X[qids.astype(np.int64)])
    k = 10
    for tie, efs in ((0, (k, 64, 65, 129)), (1, (64,))):   # tie mode 1: the std-tie kernel
        h.set_tie_mode(tie)
        for ef in efs:
            for stats in (False, True):
                h.enable_stats(stats)
                h.get_stats(reset=True)
                want = h.search_flat(V, k, ef)
                kw, sw = pkg.last_kernel(), h.get_stats()
                got = h.search_by_id(qids, k, ef)
                kg, sg = pkg.last_kernel(), h.get_stats()
                same(got, want, f"tie {tie} ef {ef} stats {stats}")
                assert kg == kw, (kg, kw)
                if stats:
                    assert sg == sw and sg["evals"] > 0, (sg, sw)
    h.set_tie_mode(0)
    h.enable_stats(False)
    same(h.search_by_id(qids, k, 64), o.search_batch(X[qids.astype(np.int64)], k, 64), "oracle")
    # exact: the host-query call and the oracle's brute force
    want = h.search_exact(V, k)
    kw = pkg.last_kernel()
    got = h.search_exact_by_id(qids, k)
    assert pkg.last_kernel() == kw
    same(got, want, "exact")
    same(got, expected(po, h, X, X[qids.astype(np.int64)], k, metric, np.arange(N)), "exact vs oracle")


def test_restrictions(pkg, po):
    X, o, h = build(pkg, po, np.float32, "DistL2", 48, seed=11)
    qids = some_ids(N, 5)
    V = h.get_vectors(qids)
    rng = np.random.default_rng(2)
    lab = rng.integers(0, 6, N).astype(np.uint32)
    lab[rng.random(N) < 0.1] = NONE
    attr = rng.integers(-500, 500, N).astype(np.int64)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    rf = h.make_filter(np.sort(origin_ids(N)[::3]))
    nq = len(qids)
    sets = [[NONE] if i % 5 == 0 else [int(i % 6), int((i * 7) % 6)] for i in range(nq)]
    ranges = np.array([(-(1 << 63), (1 << 63) - 1) if i % 4 == 0 else (-200 + i, 200 + 3 * i) for i in range(nq)], np.int64)
    for k, ef in ((10, 64), (10, 200)):
        same(h.search_by_id(qids, k, ef, filter=rf), h.search_flat(V, k, ef, filter=rf), "resident filter")
        same(h.search_by_id(qids, k, ef, sets=sets), h.search_flat_label_sets(V, k, ef, sets), "label sets")
        same(h.search_by_id(qids, k, ef, ranges=ranges), h.search_flat_ranges(V, k, ef, ranges), "ranges")
        same(h.search_by_id(qids, k, ef, ranges=ranges, sets=sets), h.search_flat_ranges(V, k, ef, ranges, sets=sets),
             "ranges within sets")
    same(h.search_exact_by_id(qids, 10, filter=rf), h.search_exact(V, 10, filter=rf), "exact resident filter")
    same(h.search_exact_by_id(qids, 10, sets=sets), h.search_exact_label_sets(V, 10, sets), "exact label sets")
    same(h.search_exact_by_id(qids, 10, ranges=ranges), h.search_exact_ranges(V, 10, ranges), "exact ranges")
    same(h.search_exact_by_id(qids, 10, ranges=ranges, sets=sets), h.search_exact_ranges(V, 10, ranges, sets=sets),
         "exact ranges within sets")
    rf.free()


def check_exclude_self(h, qids, k, ef, **kw):
    V = h.get_vectors(qids)
    want = minus_self(h.search_flat_ranges(V, k + 1, ef, kw["ranges"]) if "ranges" in kw
                      else h.search_flat(V, k + 1, ef, filter=kw.get("filter")), qids, k)
    same(h.search_by_id(qids, k, ef, exclude_self=True, **kw), want, f"exclude_self graph {kw}")
    want = minus_self(h.search_exact_ranges(V, k + 1, kw["ranges"]) if "ranges" in kw
                      else h.search_exact(V, k + 1, filter=kw.get("filter")), qids, k)
    same(h.search_exact_by_id(qids, k, exclude_self=True, **kw), want, f"exclude_self exact {kw}")


@pytest.mark.parametrize("metric", ["DistL2", "DistDot"])
def test_exclude_self(pkg, po, metric):
    # every vector stored 4 times: the three copies stay, the point goes
    X, o, h = build(pkg, po, np.float32, metric, 24, seed=17, ties=True)
    qids = some_ids(N, 9)
    for k, ef in ((10, 10), (10, 64), (3, 3), (40, 129)):
        check_exclude_self(h, qids, k, ef)
    got = h.search_by_id(qids, 10, 64, exclude_self=True)
    if metric == "DistL2":
        assert not np.any(got[2] == qids[:, None].astype(np.uint32)), "a point is in its own row"
    # a restriction that excludes the point: its row is the first k of the k + 1 row
    attr = np.arange(N, dtype=np.int64)
    h.set_attributes(0, attr)
    ranges = np.array([(int(q) + 1, int(q) + 400) for q in qids], np.int64)
    check_exclude_self(h, qids, 10, 64, ranges=ranges)
    rf = h.make_filter(np.sort(origin_ids(N)[1::2]))
    check_exclude_self(h, qids, 10, 64, filter=rf)
    rf.free()


def test_device_variant(pkg, po):
    X, o, h = build(pkg, po, np.float32, "DistL2", 100, seed=23)
    qids = some_ids(N, 4)
    nq, k, ef = len(qids), 10, 64
    d_q = torch.from_numpy(qids.view(np.int64)).cuda()
    for exact in (False, True):
        for excl in (False, True):
            want = (h.search_exact_by_id(qids, k, exclude_self=excl) if exact
                    else h.search_by_id(qids, k, ef, exclude_self=excl))
            for sync in (True, False):
                out = torch.full((nq, k * 2), -1, dtype=torch.int64, device="cuda")   # Neighbour_api: 16 bytes a slot
                cnt = torch.full((nq,), -7, dtype=torch.int32, device="cuda")
                h.search_device_by_id(d_q.data_ptr(), nq, k, ef, out.data_ptr(), cnt.data_ptr(), exclude_self=excl,
                                      exact=exact, sync=sync)
                if not sync:
                    h.stream_wait_last(torch.cuda.current_stream().cuda_stream)
                    assert h.check_status() == 0
                torch.cuda.synchronize()
                a = out.cpu().numpy().view(np.uint64).reshape(nq, k, 2)
                assert np.array_equal(cnt.cpu().numpy(), want[4]), (exact, excl, sync)
                assert np.array_equal(a[:, :, 0], want[0])
                dist = (a[:, :, 1] & 0xFFFFFFFF).astype(np.uint32)
                internal = (a[:, :, 1] >> 32).astype(np.uint32)
                assert np.array_equal(dist, want[1].view(np.uint32))
                assert np.array_equal(internal, want[2])
    bad = torch.tensor([3, N], dtype=torch.int64, device="cuda")
    out = torch.empty((2, k * 2), dtype=torch.int64, device="cuda")
    cnt = torch.empty((2,), dtype=torch.int32, device="cuda")
    with pytest.raises(pkg.HnswError, match=r"qids\[1\] = 1200"):
        h.search_device_by_id(bad.data_ptr(), 2, k, ef, out.data_ptr(), cnt.data_ptr())


@pytest.mark.parametrize("P", [2, 3])
def test_partitions(pkg, po, P):
    n, d = 1500, 48
    X = data(np.float32, "DistL2", n, d, 31)
    h = pkg.Hnsw(M, n, 16, EFC, "DistL2")
    h.partition([0] * P)
    h.insert_flat(X, ids=origin_ids(n))
    qids = some_ids(n, P)
    V = h.get_vectors(qids)
    assert np.array_equal(V, X[qids.astype(np.int64)])
    same(h.search_by_id(qids, 10, 64), h.search_flat(V, 10, 64), "partitioned")
    same(h.search_exact_by_id(qids, 10), h.search_exact(V, 10), "partitioned exact")
    for k, ef in ((10, 64), (5, 5)):
        same(h.search_by_id(qids, k, ef, exclude_self=True), minus_self(h.search_flat(V, k + 1, ef), qids, k),
             "partitioned exclude_self")
        same(h.search_exact_by_id(qids, k, exclude_self=True), minus_self(h.search_exact(V, k + 1), qids, k),
             "partitioned exact exclude_self")
    h.set_labels(0, (np.arange(n) % 4).astype(np.uint32))
    sets = [[int(i % 4)] for i in range(len(qids))]
    same(h.search_by_id(qids, 10, 64, sets=sets), h.search_flat_label_sets(V, 10, 64, sets), "partitioned sets")
    same(h.search_by_id(qids, 10, 64, sets=sets, exclude_self=True),
         minus_self(h.search_flat_label_sets(V, 11, 64, sets), qids, 10), "partitioned sets exclude_self")
    d_q = torch.zeros(1, dtype=torch.int64, device="cuda")
    out = torch.empty((1, 20), dtype=torch.int64, device="cuda")
    cnt = torch.empty(1, dtype=torch.int32, device="cuda")
    with pytest.raises(pkg.HnswError, match="partitioned"):
        h.search_device_by_id(d_q.data_ptr(), 1, 10, 64, out.data_ptr(), cnt.data_ptr())
    # a partition view: its own local ids
    v = h.partition_view(1)
    nv = v.get_nb_point()
    lq = some_ids(nv, 8, count=40)
    assert np.array_equal(v.get_vectors(lq), X[1::P][lq.astype(np.int64)])
    Vl = v.get_vectors(lq)
    same(v.search_by_id(lq, 10, 64), v.search_flat(Vl, 10, 64), "view")
    same(v.search_by_id(lq, 10, 64, exclude_self=True), minus_self(v.search_flat(Vl, 11, 64), lq, 10), "view exclude_self")


def test_get_vectors_and_point_data(pkg, po):
    X, o, h = build(pkg, po, np.uint16, "DistL2", 64, seed=41)
    E = h.export_vectors()
    r = np.array([5, 6, 7, 0, N - 1, 5], np.uint64)
    assert np.array_equal(h.get_vectors(r), E[r.astype(np.int64)])
    assert h.get_vectors([]).shape == (0, 64)
    lv, rk, _, _ = h.export_points()
    for i in (0, 17, 640, N - 1):
        assert np.array_equal(h.get_point_data((int(lv[i]), int(rk[i]))), E[i])
    top = int(lv.max())
    assert h.get_point_data((0, int((lv == 0).sum()))) is None
    assert h.get_point_data((top + 1, 0)) is None
    assert h.get_point_data((0, -1)) is None
    with pytest.raises(pkg.HnswError, match=r"ranks\[1\] = 1200"):
        h.get_vectors([1, N])


def test_knn_graph(pkg, po):
    X, o, h = build(pkg, po, np.float32, "DistCosine", 48, seed=43)
    k = 8
    ids, ds = h.knn_graph(k, ef=32, batch=500)
    qa = np.arange(N, dtype=np.uint64)
    for s in range(0, N, 500):
        _, d, it, _, _ = h.search_by_id(qa[s:s + 500], k, 32, exclude_self=True)
        assert np.array_equal(ids[s:s + 500], it) and np.array_equal(ds[s:s + 500].view(np.uint32), d.view(np.uint32))
    eids, eds = h.knn_graph(k, exact=True, batch=700)
    want = minus_self(expected(po, h, X, X, k + 1, "DistCosine", np.arange(N)), qa, k)
    assert np.array_equal(eids, want[2]) and np.array_equal(eds.view(np.uint32), want[1].view(np.uint32))
    recall = np.mean([len(set(ids[i]) & set(eids[i])) / k for i in range(N)])
    assert recall > 0.9, recall


def test_refusals(pkg, po):
    X, o, h = build(pkg, po, np.float32, "DistL2", 24, seed=47)
    L = h._L
    ans = h._answers(3, 10, True, True)
    with pytest.raises(pkg.HnswError, match=r"qids\[2\] = 1200 is not below nb_point = 1200"):
        h.search_by_id([0, 1, N], 10, 64)
    with pytest.raises(pkg.HnswError, match=r"qids\[0\]"):
        h.search_exact_by_id([N + 5], 10)
    import ctypes as C
    p = [a.ctypes.data_as(C.c_void_p) for a in ans]
    assert L.hnsw_b200_search_flat_by_id(h._h, None, 3, 10, 64, 0, -1, None, None, None, *p) != 0
    assert "qids is NULL" in pkg.last_error()
    assert L.hnsw_b200_search_flat_by_id(h._h, None, 0, 10, 64, 0, -1, None, None, None, *p) == 0   # nq == 0
    assert L.hnsw_b200_search_flat_by_id(None, None, 3, 10, 64, 0, -1, None, None, None, *p) != 0
    assert "NULL handle" in pkg.last_error()
    rf = h.make_filter(np.sort(origin_ids(N)[::2]))
    with pytest.raises(pkg.HnswError, match="cannot be combined"):
        h.search_by_id([0, 1], 10, 64, filter=rf, sets=[[1], [2]])
    with pytest.raises(pkg.HnswError, match="cannot be combined"):
        h.search_exact_by_id([0, 1], 10, filter=rf, ranges=[(0, 1), (0, 1)])
    h.insert_flat(X[:1], ids=np.array([99999], np.uint64))   # the filter goes stale
    with pytest.raises(pkg.HnswError):
        h.search_by_id([0, 1], 10, 64, filter=rf)
    msg = pkg.last_error()
    with pytest.raises(pkg.HnswError) as e:
        h.search_flat(X[:2], 10, 64, filter=rf)
    assert str(e.value) == msg
    rf.free()

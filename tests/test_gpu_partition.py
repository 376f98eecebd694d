"""Partitioned index (include/hnsw_b200.h "Partitioned index"): points split over P partitions, every query searched on
every partition, the P answer lists merged.

Most cases place several partitions on device 0, so they run on one GPU; the two-GPU case skips below two devices.
Every partition must build the graph the oracle builds from its share of the points (X[p::P]), and a partitioned search
must equal the oracle answers of the P partitions merged by the rule (distance, partition, position), bit for bit."""
import threading

import numpy as np
import pytest

from test_gpu_matrix import assert_same_graph, data, same
from util import recall_ids

pytestmark = pytest.mark.gpu

N, NQ, M = 2000, 60, 8
INV = 0xFFFFFFFF


def origin_ids(n):
    return (np.arange(n, dtype=np.uint64) * 7 + 3)   # distinct from every rank, so a mix-up shows


def oracle_parts(po, X, ids, levels, P, metric, efc, dtype):
    out = []
    for p in range(P):
        o = po.Oracle(M, max(1, len(X[p::P])), 16, efc, metric, X.shape[1], dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
        o.insert_batch(X[p::P], ids=ids[p::P], levels=levels[p::P])
        out.append(o)
    return out


def build(pkg, po, dtype, metric, d, efc, P, devices=None, serial=True, seed=1, n=N):
    X = data(dtype, metric, n, d, seed)
    levels = po.Oracle(M, n, 16, efc, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU).draw_levels(n)
    ids = origin_ids(n)
    h = pkg.Hnsw(M, n, 16, efc, metric, dtype=dtype)
    if serial:
        h.set_insert_batching(1 << 30, 1)   # set before partition(): copied to every partition
    h.partition(devices if devices is not None else [0] * P)
    h.insert_flat(X, ids=ids, levels=levels)
    assert h.get_nb_point() == n and h.partition_count() == P
    return X, ids, levels, h


def merged(answers, k):
    """the P answer lists of (origin, dist, internal, pid, counts) merged by (distance, partition, position)"""
    P = len(answers)
    nq = answers[0][0].shape[0]
    o = np.full((nq, k), np.iinfo(np.uint64).max, np.uint64)
    d = np.full((nq, k), np.inf, np.float32)
    it = np.full((nq, k), INV, np.uint32)
    pid = np.full((nq, k, 2), -1, np.int32)
    cnt = np.zeros(nq, np.int32)
    for q in range(nq):
        ent = sorted(((float(a[1][q, j]), p, j) for p, a in enumerate(answers) for j in range(a[4][q])),
                     key=lambda e: e[:3])[:k]
        cnt[q] = len(ent)
        for s, (_, p, j) in enumerate(ent):
            a = answers[p]
            o[q, s], d[q, s], pid[q, s] = a[0][q, j], a[1][q, j], a[3][q, j]
            it[q, s] = int(a[2][q, j]) * P + p
    return o, d, it, pid, cnt


def queries(X, dtype, metric, seed):
    Q = data(dtype, metric, NQ, X.shape[1], seed + 100)
    Q[: NQ // 10] = X[: NQ // 10]   # stored points: distance-0 answers
    return Q


def check_graphs(h, oracles):
    for p, o in enumerate(oracles):
        assert_same_graph(h.partition_view(p), o, len(o))


GRAPH_CASES = [(np.float32, "DistL2", 24), (np.float32, "DistCosine", 24), (np.uint8, "DistHamming", 100)]


@pytest.mark.parametrize("efc", [48, 200])
@pytest.mark.parametrize("P", [1, 2, 3, 4])
@pytest.mark.parametrize("dtype,metric,d", GRAPH_CASES, ids=[f"{np.dtype(c[0]).name}-{c[1]}" for c in GRAPH_CASES])
def test_partition_graphs_and_search_parity(pkg, po, dtype, metric, d, P, efc):
    X, ids, levels, h = build(pkg, po, dtype, metric, d, efc, P, seed=d + P)
    oracles = oracle_parts(po, X, ids, levels, P, metric, efc, dtype)
    check_graphs(h, oracles)
    Q = queries(X, dtype, metric, d + P)
    for k in (1, 10, 40):
        for ef in sorted({k, 64, 129}):
            for stats in (False, True):
                for o in oracles:
                    o.counters()
                h.enable_stats(stats)
                h.get_stats()
                got = h.search_flat(Q, k, ef)
                want = merged([o.search_batch(Q, k, ef) for o in oracles], k)
                same(got, want, f"P={P} k={k} ef={ef} stats={stats}")
                if stats:
                    cg = h.get_stats()
                    co = [o.counters() for o in oracles]
                    for key in ("evals", "expansions", "adj_read"):
                        assert cg[key] == sum(c[key] for c in co), (k, ef, key)
                    assert cg["queries"] == P * NQ   # a query counts once per partition
    h.enable_stats(False)
    # filter mode 1 (sorted origin ids) and mode 2 (a callback, called on this thread only, once per stored point)
    allow = ids[1::3]
    for k, ef in ((5, 5), (10, 64)):
        want = merged([o.search_batch(Q, k, ef, filter_ids=allow) for o in oracles], k)
        same(h.search_flat(Q, k, ef, filter=allow), want, f"filter ids k={k} ef={ef}")
        calls, threads = [], set()
        allowed = set(allow.tolist())

        def fn(i):
            calls.append(i)
            threads.add(threading.get_ident())
            return i in allowed
        same(h.search_flat(Q, k, ef, filter=fn), want, f"filter fn k={k} ef={ef}")
        assert len(calls) == N and sorted(calls) == sorted(ids.tolist())
        assert threads == {threading.get_ident()}
    # tie mode 1 on the tie-heavy metric, against the oracle's literal std heaps
    if metric == "DistHamming":
        h.set_tie_mode(1)
        for o in oracles:
            o.set_mode(po.MODE_STD)
        for k, ef in ((10, 32), (40, 129)):
            same(h.search_flat(Q, k, ef), merged([o.search_batch(Q, k, ef) for o in oracles], k), f"std-tie k={k}")


def test_one_partition_is_the_unpartitioned_index(pkg, po):
    """P = 1 with the default (batched) insert and levels drawn by the handle: every answer bit-identical"""
    X = data(np.float32, "DistL2", N, 24, 5)
    Q = queries(X, np.float32, "DistL2", 5)
    hs = []
    for part in (False, True):
        h = pkg.Hnsw(M, N, 16, 64, "DistL2")
        h.set_level_seed(11)
        if part:
            h.partition([0])
        h.insert_flat(X[:1200])
        h.parallel_insert([(X[i], i) for i in range(1200, N)])
        hs.append(h)
    plain, part = hs
    view = part.partition_view(0)
    lv, rk, og, e = plain.export_points()
    vlv, vrk, vog, ve = view.export_points()
    assert e == ve and np.array_equal(lv, vlv) and np.array_equal(rk, vrk) and np.array_equal(og, vog)
    for layer in range(int(lv.max()) + 1):
        for a, b in zip(plain.export_layer(layer), view.export_layer(layer)):
            assert np.array_equal(a, b)
    for k, ef in ((1, 1), (10, 64), (40, 129)):
        same(part.search_flat(Q, k, ef), plain.search_flat(Q, k, ef), f"search_flat k={k}")
        a, b = plain.parallel_search(list(Q), k, ef), part.parallel_search(list(Q), k, ef)
        assert [[(n.d_id, n.distance) for n in r] for r in a] == [[(n.d_id, n.distance) for n in r] for r in b]
    for x, y in zip(plain.bruteforce(Q, 10), part.bruteforce(Q, 10)):
        assert np.array_equal(x, y)


def test_reference_entry_points_on_a_partitioned_handle(pkg, po):
    P, n = 3, 600
    X = data(np.float32, "DistL2", n, 24, 9)
    Q = queries(X, np.float32, "DistL2", 9)
    ids = origin_ids(n)
    hs = []
    for mixed in (False, True):
        h = pkg.Hnsw(M, n, 16, 64, "DistL2")
        h.set_insert_batching(1 << 30, 1)
        h.partition([0] * P)
        if mixed:   # insert_f32 one by one, parallel_insert_f32, then insert_flat: one global insertion order
            for i in range(0, 7):
                h.insert((X[i], int(ids[i])))
            h.parallel_insert([(X[i], int(ids[i])) for i in range(7, 300)])
            h.insert_flat(X[300:], ids=ids[300:])
        else:
            h.insert_flat(X, ids=ids)
        hs.append(h)
    a, b = hs
    for p in range(P):
        va, vb = a.partition_view(p), b.partition_view(p)
        for x, y in zip(va.export_points(), vb.export_points()):
            assert np.array_equal(x, y)
        for x, y in zip(va.export_layer(0), vb.export_layer(0)):
            assert np.array_equal(x, y)
    for k, ef in ((1, 16), (10, 64)):
        o, d, _, _, c = b.search_flat(Q, k, ef)
        par = b.parallel_search(list(Q), k, ef)
        for q in range(NQ):
            assert len(par[q]) == c[q]
            assert [(nb.d_id, nb.distance) for nb in par[q]] == list(zip(o[q, :c[q]].tolist(), d[q, :c[q]].tolist()))
            one = b.search(Q[q], k, ef)
            assert [(nb.d_id, nb.distance) for nb in one] == [(nb.d_id, nb.distance) for nb in par[q]]


def test_bruteforce_and_recall(pkg, po):
    # ground truth: bruteforce on a partitioned handle is exact kNN over all points, with global insertion ranks
    X, ids, levels, h = build(pkg, po, np.float32, "DistL2", 24, 48, 3, serial=False)
    Q = queries(X, np.float32, "DistL2", 3)
    bi, bd = h.bruteforce(Q, 10)
    d64 = np.sqrt(((Q[:, None, :].astype(np.float64) - X[None, :, :]) ** 2).sum(-1))   # DistL2 is the Euclidean norm
    assert np.array_equal(bi, np.argsort(d64, axis=1, kind="stable")[:, :10].astype(np.uint32))
    assert np.allclose(bd, np.sort(d64, axis=1)[:, :10], rtol=1e-4, atol=1e-5)
    ti, td = po.bruteforce(X, Q, 10, "DistL2", po.ORDER_GPU)
    assert np.array_equal(bi, ti) and np.array_equal(bd.view(np.uint32), td.view(np.uint32))
    # recall on 50 000 clustered points, four partitions on one device, against the unpartitioned index
    n, d = 50000, 64
    X = pkg.datagen.clustered(n, d, 21)
    Q = pkg.datagen.clustered(1000, d, 22)
    rec = {}
    for P in (1, 4):
        h = pkg.Hnsw(16, n, 16, 100, "DistL2")
        if P > 1:
            h.partition([0] * P)
        h.insert_flat(X)
        ti, _ = h.bruteforce(Q, 10)
        _, _, it, _, c = h.search_flat(Q, 10, 64)
        rec[P] = recall_ids(it, c, ti)
    print(f"recall@10 at ef=64: unpartitioned {rec[1]:.4f}, 4 partitions {rec[4]:.4f}")
    assert rec[4] >= rec[1] - 0.01, rec


def answers(h, Q):
    return h.search_flat(Q, 10, 64)


def test_refusals_leave_the_handle_unchanged(pkg, po, tmp_path):
    P = 2
    X, ids, levels, h = build(pkg, po, np.float32, "DistL2", 24, 48, P, n=800)
    Q = queries(X, np.float32, "DistL2", 4)
    want = answers(h, Q)
    exports = [[h.partition_view(p).export_layer(l) for l in range(2)] for p in range(P)]

    def unchanged():
        assert h.get_nb_point() == 800
        same(answers(h, Q), want, "after a refused call")
        for p in range(P):
            for l in range(2):
                for x, y in zip(h.partition_view(p).export_layer(l), exports[p][l]):
                    assert np.array_equal(x, y)

    E = pkg.HnswError
    refused = [
        lambda: h.replicate([0]),
        lambda: h.nccl_init(1, 0, np.zeros(128, np.uint8)),
        lambda: h.nccl_broadcast_index(0),
        lambda: h.submit_flat(Q, 10, 64),
        lambda: h.search_device(0, 0, 10, 64, 0, 0),   # an empty batch: an ordinary handle would return at once
        lambda: h.dist_batch(Q, np.zeros((NQ, 4), np.uint32)),
        lambda: h.file_dump(str(tmp_path), "part"),
        lambda: h.export_points(),
        lambda: h.export_vectors(),
        lambda: h.export_layer(0),
        lambda: h.flat_neighborhood(),
        lambda: h.import_graph(X[:4], ids[:4], np.zeros(4, np.uint8), 0, []),
        lambda: h.blob_header(),
        lambda: h._chk(min(h._L.hnsw_b200_blob_count(h._h), 0)),   # -1: refused
        lambda: h.blob_alloc(np.zeros(16, np.uint64)),
        lambda: h.blob_commit(),
        lambda: h.partition([0, 0]),
        lambda: h.insert_flat(np.zeros((3, 25), np.float32)),   # wrong dimension: checked before any partition changes
    ]
    for call in refused:
        with pytest.raises(E):
            call()
        unchanged()
    assert h.file_dump_cwd("part") == -1
    # a view answers read-only calls and refuses the rest
    v = h.partition_view(1)
    assert v.get_nb_point() == 400 and v.partition_count() == 1
    assert v.file_dump(str(tmp_path), "p1") == "p1"
    v.flat_neighborhood()
    v.search_flat(Q, 10, 64)
    for call in (lambda: v.insert_flat(X[:2]), lambda: v.insert((X[0], 1)), lambda: v.set_extend_candidates(False),
                 lambda: v.set_keeping_pruned(True), lambda: v.set_tie_mode(1), lambda: v.set_searching_mode(True),
                 lambda: v.enable_stats(True), lambda: v.set_insert_batching(4, 4), lambda: v.modify_level_scale(0.5),
                 lambda: v.set_level_seed(3), lambda: v.partition([0]), lambda: v.replicate([0]),
                 lambda: v.blob_alloc(np.zeros(16, np.uint64)), lambda: v.blob_commit(),
                 lambda: v.import_graph(X[:4], ids[:4], np.zeros(4, np.uint8), 0, [])):
        with pytest.raises(E):
            call()
        unchanged()
    pkg.load_library().hnsw_b200_drop(v._h)   # dropping a view is refused, not a double free
    unchanged()
    # partition() itself: refused on a non-empty or NCCL-initialised handle
    plain = pkg.Hnsw(M, 100, 16, 48, "DistL2")
    plain.insert_flat(X[:10])
    with pytest.raises(E):
        plain.partition([0, 0])
    fresh = pkg.Hnsw(M, 100, 16, 48, "DistL2")
    fresh.nccl_init(1, 0, pkg.Hnsw.nccl_unique_id())
    with pytest.raises(E):
        fresh.partition([0, 0])
    # a shared-memory check failure leaves every partition empty
    wide = pkg.Hnsw(M, 100, 16, 48, "DistL2")
    wide.partition([0, 0])
    with pytest.raises(E):
        wide.insert_flat(np.zeros((4, 30000), np.float32))
    assert wide.get_nb_point() == 0 and all(wide.partition_view(p).get_nb_point() == 0 for p in range(2))


def test_searches_from_several_threads(pkg, po):
    X, ids, levels, h = build(pkg, po, np.float32, "DistL2", 24, 48, 3, serial=False)
    Q = queries(X, np.float32, "DistL2", 7)
    want = {k: h.search_flat(Q, k, 64) for k in (1, 10, 40)}
    errs = []

    def run(t):
        try:
            for i in range(6):
                k = (1, 10, 40)[(t + i) % 3]
                same(h.search_flat(Q, k, 64), want[k], f"thread {t} k={k}")
        except Exception as e:   # noqa: BLE001  (reported below, on the test's thread)
            errs.append(e)
    th = [threading.Thread(target=run, args=(t,)) for t in range(4)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errs, errs


@pytest.mark.parametrize("serial", [True, False])
def test_two_gpus_match_one(pkg, po, serial):
    if pkg.load_library().hnsw_b200_device_count() < 2:
        pytest.skip("needs two GPUs")
    res = []
    for devs in ([0, 0], [0, 1]):
        X, ids, levels, h = build(pkg, po, np.float32, "DistL2", 24, 48, 2, devices=devs, serial=serial)
        Q = queries(X, np.float32, "DistL2", 8)
        res.append((h, [h.partition_view(p).export_layer(0) for p in range(2)], h.search_flat(Q, 10, 64)))
    for a, b in zip(res[0][1], res[1][1]):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)
    same(res[1][2], res[0][2], "[0, 1] vs [0, 0]")

"""Full-size checks at BASELINE.json configs[1] (1 000 000 x 128 f32 L2, M=16, ef_c=200, 10 000 queries, ef=64): the
searches are checked through size-independent properties (sortedness, idempotence, self-retrieval, permutation
invariance, agreement with the exact brute-force kernel) plus an oracle spot-check of a query sample on the SAME graph
(exported from the GPU, imported into the oracle).  The graph itself is compared with the oracle's batch-synchronous
build of the same points and levels in tests/test_gpu_batched_insert.py::test_c2_full_size_equals_batched_oracle."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def c2(pkg):
    n, d = 1000000, 128
    X = pkg.datagen.clustered(n, d, 1)
    h = pkg.Hnsw(16, n, 16, 200, "DistL2")
    h.insert_flat(X)
    Q = pkg.datagen.clustered(10000, d, 2)
    return X, Q, h


def test_fullsize_properties(pkg, c2):
    X, Q, h = c2
    assert h.get_nb_point() == len(X)
    o, d, it, pid, cnt = h.search_flat(Q, 10, 64)
    assert np.all(cnt == 10)
    assert np.all(np.diff(d, axis=1) >= 0)                                  # ascending (hnsw.rs:1544)
    assert np.all(it < len(X)) and np.all(o == it)                          # default origin id == insertion rank
    assert all(len(set(row.tolist())) == 10 for row in it[:2000])           # no duplicate neighbour
    o2, d2, it2, _, cnt2 = h.search_flat(Q, 10, 64)                         # idempotent
    assert np.array_equal(it, it2) and np.array_equal(d.view(np.uint32), d2.view(np.uint32))
    perm = np.random.default_rng(0).permutation(len(Q))                     # answers follow the input order
    o3, d3, it3, _, _ = h.search_flat(Q[perm], 10, 64)
    assert np.array_equal(it3, it[perm]) and np.array_equal(d3, d[perm])
    # returned distances are the true distances to the returned points (f64 check, 1e-5 relative)
    for i in (0, 17, 9999):
        ref = np.sqrt(((X[it[i]].astype(np.float64) - Q[i].astype(np.float64)) ** 2).sum(1))
        assert np.allclose(d[i], ref, rtol=1e-5)
    # k / ef monotonicity: the top-5 of (k=5) equals the first 5 of (k=10) at the same ef
    o5, d5, it5, _, _ = h.search_flat(Q[:500], 5, 64)
    assert np.array_equal(it5, it[:500, :5])
    # self retrieval: stored points find themselves at distance 0 (tests/equality.rs logs this rate)
    s = h.search_flat(X[:2000], 1, 64)
    found = s[2][:, 0] == np.arange(2000)
    print("self-retrieval rate at 1M, ef=64:", found.mean())
    # (not 1.0 by design: the reference files back-links under the new point's level, hnsw.rs:1257, which leaves a few
    # per cent of points hard to reach at layer 0 -- SURVEY.md finding 3; the oracle shows the same on small indexes)
    assert found.mean() > 0.85 and np.all(s[1][found, 0] == 0.0)


def test_fullsize_recall_and_oracle_spotcheck(pkg, po, c2):
    X, Q, h = c2
    o, d, it, pid, cnt = h.search_flat(Q[:1000], 10, 64)
    bi, bd = h.bruteforce(Q[:1000], 10)                                     # exact, K5 kernel
    rec = np.mean([len(set(it[i].tolist()) & set(bi[i].tolist())) / 10 for i in range(1000)])
    ball = np.mean([(d[i] <= bd[i, 9]).sum() / 10 for i in range(1000)])    # the reference's recall definition
    assert rec > 0.8 and ball >= rec
    # brute force itself against numpy on a few queries
    for i in (0, 500):
        dd = np.sqrt(((X.astype(np.float32) - Q[i]) ** 2).sum(1))
        assert set(np.argsort(dd, kind="stable")[:10].tolist()) == set(bi[i].tolist())
    # oracle on the same graph (MODE_DET + GPU summation order): identical answers for a query sample
    lv, rk, og, entry = h.export_points()
    orc = po.Oracle(16, len(X), 16, 200, "DistL2", 128, mode=po.MODE_DET, order=po.ORDER_GPU)
    orc.import_graph(X, og, lv, entry, {l: h.export_layer(l) for l in range(int(lv.max()) + 1)})
    oo, od, oi, _, oc = orc.search_batch(Q[:300], 10, 64, nthreads=8)
    assert np.array_equal(oi, it[:300]) and np.array_equal(od.view(np.uint32), d[:300].view(np.uint32))


def _oracle_on_gpu_graph(po, h, X, M, efc, metric, d):
    """the GPU-built graph, imported into the oracle (MODE_DET + the kernels' summation order)"""
    lv, rk, og, entry = h.export_points()
    orc = po.Oracle(M, len(X), 16, efc, metric, d, mode=po.MODE_DET, order=po.ORDER_GPU)
    orc.import_graph(X, og, lv, entry, {l: h.export_layer(l) for l in range(int(lv.max()) + 1)})
    return orc


def test_c4_mnist_shape_full_size_all_queries_equal_oracle(pkg, po):
    """BASELINE.json configs[3] at full size: 60 000 x 784 f32 L2, M=32, ef=200, all 10 000 queries.  The oracle searches
    the SAME graph: ids, distance bits and the traversal counters must be equal."""
    import os
    n, d, M, efc, k, ef = 60000, 784, 32, 400, 10, 200
    X = pkg.datagen.uniform(n, d, 1)
    h = pkg.Hnsw(M, n, 16, efc, "DistL2")
    h.insert_flat(X)
    Q = pkg.datagen.uniform(10000, d, 2)
    h.enable_stats(True)
    h.get_stats()
    go, gd, gi, _, gc = h.search_flat(Q, k, ef)
    cg = h.get_stats()
    orc = _oracle_on_gpu_graph(po, h, X, M, efc, "DistL2", d)
    orc.counters()
    oo, od, oi, _, oc = orc.search_batch(Q, k, ef, nthreads=os.cpu_count() or 8)
    co = orc.counters()
    assert np.array_equal(gc, oc) and np.array_equal(gi, oi)
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))
    for key in ("evals", "expansions", "adj_read"):
        assert cg[key] == co[key], (key, cg, co)
    bi, bd = h.bruteforce(Q[:500], k)
    rec = np.mean([len(set(gi[i].tolist()) & set(bi[i].tolist())) / k for i in range(500)])
    print("C4 recall@10 at ef=200:", rec)
    assert rec > 0.5   # iid uniform 784-d is adversarial for any graph index (SURVEY 8d); the parity above is the test


@pytest.mark.parametrize("metric", ["DistDot", "DistCosine"])
def test_c3_glove_shape_full_size_oracle_spotcheck(pkg, po, metric):
    """BASELINE.json configs[2] at full size: 1 183 514 x 25 unit vectors, M=24, ef=128, with the metric the config names
    (DistCosine) and the one the reference's example actually runs on normalised data (DistDot)."""
    n, d, M, efc, k, ef = 1183514, 25, 24, 200, 10, 128
    X = pkg.datagen.unit(n, d, 1)
    h = pkg.Hnsw(M, n, 16, efc, metric)
    h.insert_flat(X)
    Q = pkg.datagen.unit(10000, d, 2)
    go, gd, gi, _, gc = h.search_flat(Q, k, ef)
    assert np.all(gc == k) and np.all(np.diff(gd, axis=1) >= 0) and np.all(gd >= 0)
    go2, gd2, gi2, _, _ = h.search_flat(Q, k, ef)
    assert np.array_equal(gi, gi2) and np.array_equal(gd.view(np.uint32), gd2.view(np.uint32))
    bi, bd = h.bruteforce(Q[:1000], k)
    rec = np.mean([len(set(gi[i].tolist()) & set(bi[i].tolist())) / k for i in range(1000)])
    print(f"C3 {metric} recall@10 at ef=128:", rec)
    assert rec > 0.8
    orc = _oracle_on_gpu_graph(po, h, X, M, efc, metric, d)
    oo, od, oi, _, oc = orc.search_batch(Q[:300], k, ef, nthreads=8)
    assert np.array_equal(oi, gi[:300]) and np.array_equal(od.view(np.uint32), gd[:300].view(np.uint32))

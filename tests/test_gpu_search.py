"""GPU parity, search path: libhnsw_b200.so (through the C ABI) vs the CPU oracle on the SAME graph.

The oracle runs in MODE_DET with ORDER_GPU distances, i.e. the total order (dist, id) and the
summation order the kernels implement, so ids AND distances must be bit-identical, and the
traversal counters (distance evaluations, expansions, adjacency ids read) must be equal.
MODE_STD / ORDER_REF (the literal reference behaviour) is compared with the tolerances
BASELINE.json names: recall@k within 1e-3, distances within 1e-5 relative.
"""
import numpy as np
import pytest

from util import gpu_layers, oracle_layers, recall_ids

pytestmark = pytest.mark.gpu


def build_pair(pkg, po, n, d, M, efc, metric, kind="uniform", max_layer=16, seed=1):
    X = pkg.datagen.make(kind, n, d, seed)
    o = po.Oracle(M, n, max_layer, efc, metric, d, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X)
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, n, max_layer, efc, metric)
    h.import_graph(X, og, lv, o.entry, oracle_layers(o))
    return X, o, h


CASES = [
    # n, d, M, ef_c, metric, data kind, k, ef
    (10000, 25, 16, 200, "DistL2", "uniform", 10, 24),     # BASELINE.json configs[0] (random.rs shape)
    (4000, 128, 16, 100, "DistL2", "clustered", 10, 64),   # SIFT shape, small
    (3000, 25, 24, 100, "DistDot", "unit", 10, 128),       # GloVe shape (angular = DistDot on unit vectors)
    (3000, 25, 24, 100, "DistCosine", "clustered", 10, 64),
    (1500, 784, 32, 100, "DistL2", "uniform", 10, 200),    # MNIST shape: wide rows, generic-d kernel
    (2000, 10, 32, 128, "DistL1", "uniform", 16, 1024),    # tests/equality.rs shape: k=16, ef=1024
    (2000, 70, 8, 60, "DistL2", "uniform", 5, 5),          # d_pad=96 (generic path), ef == k
    (3000, 32, 16, 100, "DistL2", "clustered", 10, 200),   # 128-byte rows, ef 129-256: generic kernel, 256-slot queue
]


@pytest.mark.parametrize("n,d,M,efc,metric,kind,k,ef", CASES)
def test_search_matches_det_oracle_bit_exact(pkg, po, n, d, M, efc, metric, kind, k, ef):
    X, o, h = build_pair(pkg, po, n, d, M, efc, metric, kind)
    Q = pkg.datagen.make(kind, 500, d, 2)
    o.counters()
    oo, od, oi, opid, oc = o.search_batch(Q, k, ef)
    cnt_o = o.counters()
    h.enable_stats(True)
    go, gd, gi, gpid, gc = h.search_flat(Q, k, ef)
    cnt_g = h.get_stats()
    assert np.array_equal(gc, oc)
    assert np.array_equal(gi, oi), "internal ids differ from the MODE_DET oracle"
    assert np.array_equal(go, oo)
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32)), "distances are not bit-identical"
    assert np.array_equal(gpid, opid)
    for key in ("evals", "expansions", "adj_read"):
        assert cnt_g[key] == cnt_o[key], (key, cnt_g, cnt_o)


def test_std_reference_mode_within_tolerance(pkg, po):
    """literal reference behaviour (Rust-std heaps, AVX2-shaped sums) vs GPU: recall 1e-3, distance 1e-5 rel."""
    n, d, M, efc, k, ef = 10000, 25, 16, 200, 10, 24
    X, o, h = build_pair(pkg, po, n, d, M, efc, "DistL2")
    Q = pkg.datagen.uniform(1000, d, 2)
    o.set_mode(po.MODE_STD)
    o.set_order(po.ORDER_REF)
    oo, od, oi, _, oc = o.search_batch(Q, k, ef)
    go, gd, gi, _, gc = h.search_flat(Q, k, ef)
    ti, td = po.bruteforce(X, Q, k, "DistL2")
    r_o, r_g = recall_ids(oi, oc, ti), recall_ids(gi, gc, ti)
    assert abs(r_o - r_g) <= 1e-3, (r_o, r_g)
    same = (oi == gi)
    assert same.mean() > 0.999
    rel = np.abs(od[same] - gd[same]) / np.maximum(np.abs(od[same]), 1e-30)
    assert rel.max() <= 1e-5


def test_c_abi_reference_entry_points(pkg, po):
    """search_neighbours_f32 / parallel_search_neighbours_f32 (row pointers, leaked-answer structs): answers in
    input order (hnsw.rs:1622-1633) and equal to the flat call."""
    X, o, h = build_pair(pkg, po, 3000, 16, 12, 64, "DistL2")
    Q = pkg.datagen.uniform(100, 16, 5)
    go, gd, gi, _, gc = h.search_flat(Q, 7, 32)
    par = h.parallel_search([q for q in Q], 7, 32)
    assert len(par) == len(Q)
    for i, nb in enumerate(par):
        assert [x.d_id for x in nb] == go[i, :gc[i]].tolist()
        assert np.array_equal(np.array([x.distance for x in nb], np.float32), gd[i, :gc[i]])
    one = h.search(Q[3], 7, 32)
    assert [x.d_id for x in one] == go[3, :gc[3]].tolist()


def test_self_query_distance_zero_and_small_index(pkg, po):
    """reference asserts: a stored point queried with itself comes back at distance 0
    (hnsw.rs:1871-1879, hnswio.rs:1639-1640); k larger than the index returns what exists."""
    X, o, h = build_pair(pkg, po, 300, 12, 8, 40, "DistL1")
    go, gd, gi, _, gc = h.search_flat(X[:50], 3, 40)
    assert np.all(gd[:, 0] == 0.0)
    assert np.array_equal(go[:, 0], np.arange(50, dtype=np.uint64))
    X2, o2, h2 = build_pair(pkg, po, 5, 4, 8, 40, "DistL2")
    go, gd, gi, _, gc = h2.search_flat(X2[:2], 10, 16)
    oo, od, oi, _, oc = o2.search_batch(X2[:2], 10, 16)
    assert np.array_equal(gc, oc) and gc.max() <= 5
    assert np.array_equal(gi, oi)


def test_empty_index_and_errors(pkg):
    h = pkg.Hnsw(16, 100, 16, 50, "DistL2")
    o, d, it, pid, cnt = h.search_flat(np.zeros((3, 8), np.float32), 4, 16)
    assert np.all(cnt == 0)  # hnsw.rs:1498-1500
    with pytest.raises(pkg.HnswError):
        pkg.Hnsw(16, 100, 16, 50, "DistNope")
    L = pkg.load_library()
    assert not L.init_hnsw_ptrdist_f32(16, 50, None)


def test_dist_batch_and_bruteforce_kernels(pkg, po):
    X, o, h = build_pair(pkg, po, 2000, 128, 8, 40, "DistL2", "clustered")
    Q = pkg.datagen.clustered(64, 128, 9)
    cand = np.random.default_rng(3).integers(0, 2000, (64, 50)).astype(np.uint32)
    got = h.dist_batch(Q, cand)
    for i in (0, 7, 63):
        for j in (0, 13, 49):
            ref = po.dist(Q[i], X[cand[i, j]], "DistL2", po.ORDER_GPU)
            assert got[i, j] == np.float32(ref)
            ref2 = po.dist(Q[i], X[cand[i, j]], "DistL2", po.ORDER_REF)
            assert abs(got[i, j] - ref2) <= 1e-5 * abs(ref2)
    bi, bd = h.bruteforce(Q, 10)
    ti, td = po.bruteforce(X, Q, 10, "DistL2", po.ORDER_GPU)
    assert np.array_equal(bi, ti)
    assert np.array_equal(bd.view(np.uint32), td.view(np.uint32))


def test_filtered_search_matches_oracle(pkg, po):
    """search_filter with a FilterT (sorted id list and predicate forms, filter.rs:7-24) vs the oracle's
    restatement of the filter branches (hnsw.rs:981-1001, 1037-1050, 1549-1563): identical ids/distances;
    plus the reference's own assertions (tests/filtertest.rs:141,211,258,263-269)."""
    X, o, h = build_pair(pkg, po, 3000, 16, 8, 100, "DistL2")
    Q = pkg.datagen.uniform(60, 16, 8)
    allow = np.arange(0, 3000, 3)
    oo, od, oi, opid, oc = o.search_batch(Q, 10, 64, filter_ids=allow)
    go, gd, gi, gpid, gc = h.search_flat(Q, 10, 64, filter=allow)
    assert np.array_equal(gc, oc) and np.array_equal(gi, oi)
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))
    assert np.all(go[gc[:, None] > np.arange(10)[None, :]] % 3 == 0)
    # predicate form == sorted-list form
    g2 = h.search_flat(Q, 10, 64, filter=lambda i: i % 3 == 0)
    assert np.array_equal(g2[2], gi) and np.array_equal(g2[4], gc)
    # always-false filter => 0 hits; single-admit filter => <= 1 hit, and it is the admitted id
    z = h.search_flat(Q, 10, 64, filter=lambda i: False)
    assert np.all(z[4] == 0)
    one = h.search_flat(Q, 10, 4, filter=[1234])
    oone = o.search_batch(Q, 10, 4, filter_ids=[1234])
    assert np.all(one[4] <= 1) and np.array_equal(one[4], oone[4]) and np.array_equal(one[2], oone[2])
    # ef == 1 with a restrictive filter (the case where the reference's W can run empty)
    e1 = h.search_flat(Q, 1, 1, filter=allow)
    o1 = o.search_batch(Q, 1, 1, filter_ids=allow)
    assert np.array_equal(e1[4], o1[4]) and np.array_equal(e1[2], o1[2])
    # through the mirrored single-query API
    res = h.search_filter(Q[0], 10, 64, filter=allow.tolist())
    assert [r.d_id for r in res] == go[0, :gc[0]].tolist()


INT_CASES = [
    # dtype, metric, d, value range
    (np.uint8, "DistHamming", 48, 4),
    (np.uint16, "DistHamming", 40, 3),
    (np.uint32, "DistHamming", 24, 3),
    (np.int32, "DistHamming", 24, 3),
    (np.uint8, "DistJaccard", 64, 16),
    (np.uint16, "DistJaccard", 33, 1000),
    (np.uint32, "DistJaccard", 20, 100000),
    (np.uint8, "DistL2", 100, 256),
    (np.uint16, "DistL1", 30, 5000),
    (np.int32, "DistL2", 17, 2000),
]


@pytest.mark.parametrize("dtype,metric,d,vrange", INT_CASES)
def test_integer_types_match_det_oracle(pkg, po, dtype, metric, d, vrange):
    """SURVEY §8 f1: integer element types with Hamming / Jaccard / L1 / L2 (libext.rs:779-1116).  Ties are the norm
    here: the engine orders them by (distance, id) exactly like the oracle's MODE_DET => identical neighbour ids,
    bit-identical distances; build with one insert in flight => identical graph."""
    n, M, efc, k, ef = 1500, 8, 48, 10, 32
    rng = np.random.default_rng(5)
    lo = -vrange if dtype == np.int32 and metric != "DistHamming" else 0
    X = rng.integers(lo, vrange, (n, d)).astype(dtype)
    Q = rng.integers(lo, vrange, (200, d)).astype(dtype)
    o = po.Oracle(M, n, 16, efc, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    levels = o.draw_levels(n)
    o.insert_batch(X, levels=levels)
    h = pkg.Hnsw(M, n, 16, efc, metric, dtype=dtype)
    h.set_insert_batching(1 << 30, 1)
    h.insert_flat(X, levels=levels)
    goff, gids, gds = h.export_layer(0)
    ooff, oids, ods = o.export_layer(0)
    assert np.array_equal(goff, ooff) and np.array_equal(gids, oids), "graph differs"
    assert np.array_equal(gds.view(np.uint32), ods.view(np.uint32))
    oo, od, oi, opid, oc = o.search_batch(Q, k, ef)
    go, gd, gi, gpid, gc = h.search_flat(Q, k, ef)
    assert np.array_equal(gc, oc) and np.array_equal(gi, oi)
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))
    # brute force kernel == oracle brute force (ties by id)
    bi, bd = h.bruteforce(Q[:20], k)
    ti, td = po.bruteforce(X, Q[:20], k, metric, po.ORDER_GPU)
    assert np.array_equal(bi, ti) and np.array_equal(bd.view(np.uint32), td.view(np.uint32))
    # typed reference entry points
    par = h.parallel_search([q for q in Q[:5]], k, ef)
    for i in range(5):
        assert [x.d_id for x in par[i]] == go[i, :gc[i]].tolist()


def test_integer_det_vs_std_tie_report(pkg, po):
    """MODE_STD (Rust-std heap tie behaviour) vs MODE_DET on Hamming data: same distance multiset at the k-th
    boundary for almost every query; the ids may differ only inside equal-distance groups."""
    n, d = 2000, 32
    rng = np.random.default_rng(9)
    X = rng.integers(0, 3, (n, d)).astype(np.uint8)
    Q = rng.integers(0, 3, (200, d)).astype(np.uint8)
    o = po.Oracle(8, n, 16, 64, "DistHamming", d, dtype=np.uint8, mode=po.MODE_DET)
    o.insert_batch(X)
    a = o.search_batch(Q, 10, 64)
    o.set_mode(po.MODE_STD)
    b = o.search_batch(Q, 10, 64)
    same_d = np.mean(np.all(a[1] == b[1], axis=1))
    print("fraction of queries with identical distance lists under std vs det tie rules:", same_d)
    assert same_d > 0.8


PROB_METRICS = ["DistHellinger", "DistJeffreys", "DistJensenShannon"]


@pytest.mark.parametrize("metric", PROB_METRICS)
def test_probability_metrics_match_reference_order_oracle(pkg, po, metric):
    """Hellinger / Jeffreys / Jensen-Shannon (init_hnsw_f32 accepts them, libext.rs:468-520): the device uses logf / sqrtf
    and the kernels' summation order, the literal-reference oracle std::log and AVX2-shaped sums, so the bar is the
    tolerance BASELINE.json states (1e-5 relative, recall within 1e-3), not bit equality."""
    n, d, M, efc, k, ef = 3000, 32, 12, 80, 10, 48
    rng = np.random.default_rng(5)
    X = rng.random((n, d), dtype=np.float32) + np.float32(1e-3)
    X /= X.sum(1, keepdims=True)                      # discrete probability vectors, strictly positive
    Q = rng.random((300, d), dtype=np.float32) + np.float32(1e-3)
    Q /= Q.sum(1, keepdims=True)
    o = po.Oracle(M, n, 16, efc, metric, d, mode=po.MODE_STD, order=po.ORDER_REF)
    o.insert_batch(X)
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, n, 16, efc, metric)
    h.import_graph(X, og, lv, o.entry, oracle_layers(o))
    # the distance kernel alone: every value within 1e-5 relative (absolute 1e-7 near zero) of the reference-order sum
    cand = rng.integers(0, n, (300, 40)).astype(np.uint32)
    got = h.dist_batch(Q, cand)
    for i in range(0, 300, 7):
        want = np.array([po.dist(Q[i], X[j], metric, po.ORDER_REF) for j in cand[i]], np.float32)
        assert np.allclose(got[i], want, rtol=1e-5, atol=1e-7), (metric, i)
    # the search on the same graph: recall within 1e-3 of the oracle's, distances of shared answers within 1e-5
    oo, od, oi, _, oc = o.search_batch(Q, k, ef)
    go, gd, gi, _, gc = h.search_flat(Q, k, ef)
    ti, td = po.bruteforce(X, Q, k, metric)
    assert abs(recall_ids(oi, oc, ti) - recall_ids(gi, gc, ti)) <= 1e-3
    same = oi == gi
    assert same.mean() > 0.99
    assert np.allclose(gd[same], od[same], rtol=1e-5, atol=1e-7)


STD_TIE_CASES = [c for c in INT_CASES if c[1] in ("DistHamming", "DistJaccard")] + [(np.uint16, "DistL1", 30, 6)]


@pytest.mark.parametrize("dtype,metric,d,vrange", STD_TIE_CASES)
def test_integer_types_match_std_oracle_in_tie_mode(pkg, po, dtype, metric, d, vrange):
    """BASELINE.json: "identical neighbour-id sets for integer Hamming/Jaccard".  With hnsw_b200_set_tie_mode(h, 1) the GPU
    replays the reference's std BinaryHeaps (search_std.cu), so on the SAME graph its answers must equal the literal-reference
    oracle (MODE_STD: distance-only Ord, std sift rules): ids, distances, counts and the traversal counters."""
    n, M, efc, k, ef = 1500, 8, 48, 10, 32
    rng = np.random.default_rng(5)
    X = rng.integers(0, vrange, (n, d)).astype(dtype)
    Q = rng.integers(0, vrange, (300, d)).astype(dtype)
    o = po.Oracle(M, n, 16, efc, metric, d, dtype=dtype, mode=po.MODE_STD, order=po.ORDER_GPU)
    o.insert_batch(X)                                   # the literal reference build (serial)
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, n, 16, efc, metric, dtype=dtype)
    h.import_graph(X, og, lv, o.entry, oracle_layers(o))
    o.counters()
    oo, od, oi, opid, oc = o.search_batch(Q, k, ef)
    co = o.counters()
    det = h.search_flat(Q, k, ef)                       # default tie mode, for the report below
    h.set_tie_mode(1)
    h.enable_stats(True)
    h.get_stats()
    go, gd, gi, gpid, gc = h.search_flat(Q, k, ef)
    cg = h.get_stats()
    assert np.array_equal(gc, oc)
    assert np.array_equal(gi, oi), "ids differ from the literal-reference oracle"
    assert np.array_equal(go, oo) and np.array_equal(gpid, opid)
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))
    for key in ("evals", "expansions", "adj_read"):
        assert cg[key] == co[key], (key, cg, co)
    # the reference's typed entry point takes the same path
    par = h.parallel_search([q for q in Q[:5]], k, ef)
    for i in range(5):
        assert [x.d_id for x in par[i]] == oo[i, :oc[i]].tolist()
    # and the default mode differs only by tie resolution: same distance at every rank for nearly every query
    same_d = np.mean(np.all(det[1] == gd, axis=1))
    same_ids = np.mean(np.all(det[2] == gi, axis=1))
    print(f"{metric} {np.dtype(dtype).name}: default tie mode returns the same distance list for {same_d:.2%} of the queries, "
          f"the same id list for {same_ids:.2%}")
    h.set_tie_mode(0)
    back = h.search_flat(Q, k, ef)
    assert np.array_equal(back[2], det[2])


def test_tie_mode_std_equals_default_without_ties(pkg, po):
    """on data without equal distances both tie modes are the reference: identical answers"""
    X, o, h = build_pair(pkg, po, 4000, 24, 12, 64, "DistL2", "clustered")
    Q = pkg.datagen.clustered(300, 24, 3)
    a = h.search_flat(Q, 10, 48)
    h.set_tie_mode(1)
    b = h.search_flat(Q, 10, 48)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_filtered_search_on_tie_heavy_metric_matches_oracle(pkg, po):
    """ADVICE r1: the filtered stop / retain rule compares distances only (hnsw.rs:981).  With Hamming data, where a popped
    candidate often TIES with W's farthest, a (distance, id) comparison would run the retain pass where the reference does
    not; kernel and oracle must agree on ids, distances and counts with both filter forms, also at small ef."""
    n, d = 2000, 32
    rng = np.random.default_rng(11)
    X = rng.integers(0, 3, (n, d)).astype(np.uint8)
    Q = rng.integers(0, 3, (120, d)).astype(np.uint8)
    o = po.Oracle(8, n, 16, 64, "DistHamming", d, dtype=np.uint8, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X)
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(8, n, 16, 64, "DistHamming", dtype=np.uint8)
    h.import_graph(X, og, lv, o.entry, oracle_layers(o))
    for allow, k, ef in ((np.arange(0, n, 3), 10, 32), (np.arange(5, n, 17), 5, 8), (np.arange(0, n, 2), 10, 10)):
        oo, od, oi, _, oc = o.search_batch(Q, k, ef, filter_ids=allow)
        go, gd, gi, _, gc = h.search_flat(Q, k, ef, filter=allow)
        assert np.array_equal(gc, oc), (k, ef)
        assert np.array_equal(gi, oi), (k, ef)
        assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))

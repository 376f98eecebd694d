"""GPU edge cases: long neighbour lists (2M > 32: multi-chunk expansion), ef_construction above the chunked-queue
limit (generic queue in the insert kernel), capacity growth across many insert calls, tiny / odd shapes, host
threads sharing one index, error paths.  All checked against the oracle."""
import threading

import numpy as np
import pytest

from util import csr_lists

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,efc,d,metric", [(40, 120, 16, "DistL2"), (32, 400, 10, "DistL1"), (129, 300, 8, "DistL2")])
def test_long_lists_and_big_ef_construction(pkg, po, M, efc, d, metric):
    """tests/serpar.rs shape (M=32, ef_c=400) and lists longer than one 32-lane chunk (2M = 80, 258)."""
    n = 1200
    X = pkg.datagen.uniform(n, d, 31)
    o = po.Oracle(M, n, 16, efc, metric, d, mode=po.MODE_DET, order=po.ORDER_GPU)
    levels = o.draw_levels(n)
    o.insert_batch(X, levels=levels)
    h = pkg.Hnsw(M, n, 16, efc, metric)
    h.set_insert_batching(1 << 30, 1)
    h.insert_flat(X, levels=levels)
    goff, gids, gds = h.export_layer(0)
    ooff, oids, ods = o.export_layer(0)
    assert np.array_equal(goff, ooff) and np.array_equal(gids, oids)
    assert np.array_equal(gds.view(np.uint32), ods.view(np.uint32))
    Q = pkg.datagen.uniform(100, d, 32)
    for k, ef in ((10, 48), (20, 300)):
        a, b = o.search_batch(Q, k, ef), h.search_flat(Q, k, ef)
        assert np.array_equal(a[2], b[2]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


def test_incremental_inserts_and_capacity_growth(pkg, po):
    """max_elements is only a hint (hnsw.rs:452-461): 5000 points into an index created for 16, in uneven calls mixing
    insert_f32, parallel_insert_f32 and the flat call; graph == oracle serial build."""
    n, d, M, efc = 5000, 12, 8, 40
    X = pkg.datagen.uniform(n, d, 41)
    o = po.Oracle(M, 16, 16, efc, "DistL2", d, mode=po.MODE_DET, order=po.ORDER_GPU)
    levels = o.draw_levels(n)
    o.insert_batch(X, levels=levels)
    h = pkg.Hnsw(M, 16, 16, efc, "DistL2")
    h.set_insert_batching(1 << 30, 1)
    pos = 0
    for sz in (1, 1, 3, 50, 700, 1, 2000, 2244):
        h.insert_flat(X[pos:pos + sz], ids=np.arange(pos, pos + sz), levels=levels[pos:pos + sz])
        pos += sz
    assert pos == n and h.get_nb_point() == n
    goff, gids, _ = h.export_layer(0)
    ooff, oids, _ = o.export_layer(0)
    assert np.array_equal(goff, ooff) and np.array_equal(gids, oids)
    for layer in (1, 2):
        gl = csr_lists(*h.export_layer(layer)[:2])
        ol = csr_lists(*o.export_layer(layer)[:2])
        lv = o.export_points()[0]
        assert all(gl[p] == ol[p] for p in range(n) if lv[p] >= layer)


def test_tiny_and_odd_shapes(pkg, po):
    # one point, k larger than the index
    h = pkg.Hnsw(4, 10, 16, 8, "DistL2")
    h.insert((np.array([1.0, 2.0, 3.0], np.float32), 9))
    r = h.search(np.array([1.0, 2.0, 3.0], np.float32), 5, 3)
    assert len(r) == 1 and r[0].d_id == 9 and r[0].distance == 0.0
    # u8 vectors of 3 bytes (row tail handled byte-wise), d = 1
    for dt, d in ((np.uint8, 3), (np.float32, 1), (np.uint16, 5)):
        rng = np.random.default_rng(1)
        X = rng.integers(0, 50, (300, d)).astype(dt)
        metric = "DistL1"
        o = po.Oracle(6, 300, 16, 20, metric, d, dtype=dt, mode=po.MODE_DET, order=po.ORDER_GPU)
        lv = o.draw_levels(300)
        o.insert_batch(X, levels=lv)
        g = pkg.Hnsw(6, 300, 16, 20, metric, dtype=dt)
        g.set_insert_batching(1 << 30, 1)
        g.insert_flat(X, levels=lv)
        a, b = o.search_batch(X[:40], 4, 16), g.search_flat(X[:40], 4, 16)
        assert np.array_equal(a[2], b[2]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))


def test_many_host_threads_one_index(pkg, po):
    """search* take &self and may be called from many host threads (hnsw.rs:830-833)"""
    X = pkg.datagen.uniform(3000, 16, 51)
    h = pkg.Hnsw(12, 3000, 16, 64, "DistL2")
    h.insert_flat(X)
    Q = pkg.datagen.uniform(64, 16, 52)
    want = h.search_flat(Q, 5, 32)
    out, errs = {}, []

    def work(t):
        try:
            for _ in range(5):
                out[t] = h.search_flat(Q, 5, 32)
        except Exception as e:  # pragma: no cover
            errs.append(e)
    th = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs
    for t in range(8):
        assert np.array_equal(out[t][0], want[0]) and np.array_equal(out[t][1], want[1])


def test_error_paths_are_loud(pkg):
    h = pkg.Hnsw(8, 100, 16, 20, "DistL2")
    h.insert((np.zeros(6, np.float32), 0))
    with pytest.raises(pkg.HnswError):          # dimension mismatch is refused (the flat store needs one dimension)
        h.insert((np.zeros(7, np.float32), 1))
    with pytest.raises(pkg.HnswError):
        h.search_flat(np.zeros((2, 9), np.float32), 3, 8)
    with pytest.raises(pkg.HnswError):          # Jaccard is not defined for i32 upstream either (libext.rs:779-810)
        pkg.Hnsw(8, 10, 16, 20, "DistJaccard", dtype=np.int32)
    with pytest.raises(pkg.HnswError):
        pkg.Hnsw(1, 10, 16, 20, "DistL2")      # ln(1) = 0 breaks the level law
    with pytest.raises(pkg.HnswError):
        h.modify_level_scale(0.5)               # only before the first insert (hnsw.rs:881-888)


def test_single_point_at_any_level(pkg):
    """hnsw.rs:1871-1879 test_sparse_search: one inserted point is found whatever level it drew (distance 0),
    and its PointId carries that level."""
    for lvl in (0, 3, 15):
        h = pkg.Hnsw(16, 10, 16, 50, "DistL1")
        v = np.arange(8, dtype=np.float32)
        h.insert_flat(v[None, :], ids=[77], levels=[lvl])
        o, d, it, pid, cnt = h.search_flat(v[None, :], 3, 10)
        assert cnt[0] == 1 and o[0, 0] == 77 and d[0, 0] == 0.0 and tuple(pid[0, 0]) == (lvl, 0)
        assert h.get_max_level_observed() == lvl


def test_level_law_and_scale(pkg):
    """LayerGenerator law (hnsw.rs:363-374) as drawn by the engine: P(level >= 1) = 1/M, and M^-2 after
    modify_level_scale(0.5) (hnsw.rs:876-905)."""
    n, M = 60000, 16
    X = pkg.datagen.uniform(n, 4, 61)
    for scale, want in ((None, 1.0 / M), (0.5, 1.0 / M ** 2)):
        h = pkg.Hnsw(M, n, 16, 16, "DistL2")
        if scale:
            h.modify_level_scale(scale)
        h.insert_flat(X)
        lv = h.export_points()[0]
        p = (lv >= 1).mean()
        assert abs(p - want) < 4 * np.sqrt(want / n) + 1e-4, (scale, p, want)


def test_row_pointer_entry_points_for_u8(pkg, po):
    """insert_u8 / parallel_insert_u8 / parallel_search_neighbours_u8 (libext.rs:1052-1116)"""
    rng = np.random.default_rng(7)
    X = rng.integers(0, 6, (400, 24)).astype(np.uint8)
    h = pkg.Hnsw(8, 400, 16, 32, "DistHamming", dtype=np.uint8)
    h.insert((X[0], 500))
    h.parallel_insert([(X[i], 500 + i) for i in range(1, 400)])
    assert h.get_nb_point() == 400
    par = h.parallel_search([X[3], X[399]], 2, 32)
    assert par[0][0].d_id == 503 and par[0][0].distance == 0.0 and par[1][0].d_id == 899


def test_failed_insert_leaves_a_consistent_index(pkg):
    """An insert call that cannot run (here: ef_construction far beyond the insert kernel's shared memory) is refused
    BEFORE it changes anything: the point count, the dump and later searches see only the points that are linked."""
    h = pkg.Hnsw(16, 1000, 16, 40, "DistL2")
    X = pkg.datagen.uniform(300, 16, 1)
    h.insert_flat(X)
    before = h.search_flat(X[:20], 3, 16)
    bad = pkg.Hnsw(16, 1000, 16, 200000, "DistL2")      # ef_construction = 200 000: 1.6 MB of queue per warp
    with pytest.raises(pkg.HnswError):
        bad.insert_flat(X[:50])
    assert bad.get_nb_point() == 0                       # nothing of the refused call is counted
    o, d, it, _, c = bad.search_flat(X[:4], 2, 8)
    assert np.all(c == 0)
    # 128-byte rows and a small ef, but no entry point: the generic kernel with a row length read at run time answers
    bad32 = pkg.Hnsw(16, 1000, 16, 200000, "DistL2")
    X32 = pkg.datagen.uniform(50, 32, 1)
    with pytest.raises(pkg.HnswError):
        bad32.insert_flat(X32)
    o, d, it, _, c = bad32.search_flat(X32[:4], 2, 8)
    assert np.all(c == 0)
    # the healthy handle is unaffected, and a refused dimension mismatch changes nothing either
    with pytest.raises(pkg.HnswError):
        h.insert_flat(pkg.datagen.uniform(5, 17, 2))
    assert h.get_nb_point() == 300
    for a, b in zip(before, h.search_flat(X[:20], 3, 16)):
        assert np.array_equal(a, b)


def test_corrupt_dump_header_returns_null(pkg, tmp_path):
    """nb_point / dimension in a damaged header must not size allocations (the reference returns an error, hnswio.rs)"""
    h = pkg.Hnsw(8, 100, 16, 40, "DistL2")
    h.insert_flat(pkg.datagen.uniform(60, 8, 1))
    base = h.file_dump(tmp_path, "hdr")
    g = tmp_path / (base + ".hnsw.graph")
    raw = bytearray(g.read_bytes())
    # Description: magic u32, version... nb_point is a u64 field; flip the high bytes of every 8-byte word that holds 60
    hit = 0
    for off in range(0, min(len(raw), 200) - 8):
        if int.from_bytes(raw[off:off + 8], "little") == 60:
            raw[off + 5] = 0x7F
            hit += 1
    assert hit >= 1
    g.write_bytes(bytes(raw))
    with pytest.raises(pkg.HnswError):
        pkg.Hnsw.load(tmp_path, base, "DistL2")


def test_submit_wait_pipelines_batches(pkg, po):
    """hnsw_b200_search_flat_submit / _wait: same answers as the one-call form, several tickets outstanding, and a call
    that changes the index waits for the outstanding tickets instead of racing them"""
    X = pkg.datagen.clustered(5000, 32, 1)
    h = pkg.Hnsw(12, 6000, 16, 80, "DistL2")
    h.insert_flat(X)
    Qs = [pkg.datagen.clustered(700 + 13 * i, 32, 10 + i) for i in range(6)]
    want = [h.search_flat(q, 7, 40) for q in Qs]
    tickets = [h.submit_flat(q, 7, 40) for q in Qs[:4]]            # four in flight (the per-handle maximum)
    got = [h.wait_flat(t) for t in tickets]
    got += [h.wait_flat(h.submit_flat(q, 7, 40)) for q in Qs[4:]]
    for w, g in zip(want, got):
        for a, b in zip(w, g):
            assert np.array_equal(a, b)
    # a writer waits for outstanding tickets: insert from another thread while a ticket is open
    t = h.submit_flat(Qs[0], 7, 40)
    done = []
    th = threading.Thread(target=lambda: (h.insert_flat(pkg.datagen.clustered(200, 32, 99), ids=np.arange(5000, 5200, dtype=np.uint64)),
                                          done.append(1)))
    th.start()
    res = h.wait_flat(t)
    th.join(timeout=60)
    assert done == [1] and h.get_nb_point() == 5200
    for a, b in zip(want[0], res):
        assert np.array_equal(a, b)                               # the ticket saw the index as it was at submit time


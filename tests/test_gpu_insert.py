"""GPU parity, insert path (insert_f32 / parallel_insert_f32 / hnsw_b200_insert_flat).

1. With one insert in flight (batch size 1) the GPU build is a deterministic serial build and must
   produce EXACTLY the graph of the oracle's serial MODE_DET build from the same levels: same
   neighbour ids, bit-equal link distances, same entry point (the reference's check_graph_equality,
   /root/reference/src/hnsw.rs:1686-1753).
2. With many inserts in flight (the production setting) recall@10 of searches on the GPU-built graph
   stays within 0.01 of the graph of the oracle's threaded build, which races inserts like the
   reference's nondeterministic parallel_insert (hnsw.rs:1222-1223).  That is a check of quality; the
   batched build itself is compared bit for bit with the oracle's batch-synchronous build in
   tests/test_gpu_batched_insert.py.
"""
import numpy as np
import pytest

from util import csr_lists, recall_ids

pytestmark = pytest.mark.gpu


def test_serial_gpu_build_equals_oracle_graph(pkg, po):
    n, d, M, efc = 1500, 20, 8, 60
    X = pkg.datagen.uniform(n, d, 11)
    o = po.Oracle(M, n, 16, efc, "DistL2", d, mode=po.MODE_DET, order=po.ORDER_GPU)
    levels = o.draw_levels(n)
    o.insert_batch(X, levels=levels)
    h = pkg.Hnsw(M, n, 16, efc, "DistL2")
    h.set_insert_batching(1 << 30, 1)
    h.insert_flat(X, levels=levels)
    lv, rk, og, entry = h.export_points()
    olv, ork, oog = o.export_points()
    assert entry == o.entry
    assert np.array_equal(lv, olv) and np.array_equal(rk, ork) and np.array_equal(og, oog)
    for layer in range(0, int(olv.max()) + 1):
        goff, gids, gds = h.export_layer(layer)
        ooff, oids, ods = o.export_layer(layer)
        gl, ol = csr_lists(goff, gids), csr_lists(ooff, oids)
        for p in range(n):
            # the oracle also keeps lists no search can reach (above a point's present level); the
            # engine does not materialise them (DESIGN.md): compare where the engine has a list
            if layer > 0 and not gl[p] and olv[p] < layer:
                continue
            assert gl[p] == ol[p], (layer, p, gl[p], ol[p])
        if layer == 0:
            assert np.array_equal(gds.view(np.uint32), ods.view(np.uint32))


@pytest.mark.parametrize("n,d,M,efc,metric,kind", [
    (20000, 25, 16, 200, "DistL2", "uniform"),
    (20000, 128, 16, 200, "DistL2", "clustered"),
])
def test_batched_gpu_build_recall_matches_oracle_build(pkg, po, n, d, M, efc, metric, kind):
    X = pkg.datagen.make(kind, n, d, 1)
    Q = pkg.datagen.make(kind, 500, d, 2)
    ti, td = po.bruteforce(X, Q, 10, metric)
    o = po.Oracle(M, n, 16, efc, metric, d, mode=po.MODE_DET, order=po.ORDER_GPU)
    levels = o.draw_levels(n)
    o.insert_batch(X, levels=levels, nthreads=8)
    oo, od, oi, _, oc = o.search_batch(Q, 10, 64)
    h = pkg.Hnsw(M, n, 16, efc, metric)
    h.insert_flat(X, levels=levels)
    assert h.get_nb_point() == n
    go, gd, gi, _, gc = h.search_flat(Q, 10, 64)
    r_o, r_g = recall_ids(oi, oc, ti), recall_ids(gi, gc, ti)
    print("recall oracle-built", r_o, "gpu-built", r_g)
    assert r_g >= r_o - 0.01
    # every stored point must be findable by its own vector most of the time (tests/equality.rs logs this)
    so, sd, si, _, sc = h.search_flat(X[:500], 1, 64)
    assert (si[:, 0] == np.arange(500)).mean() > 0.97


def test_reference_entry_points_insert_then_search(pkg, po):
    """insert_f32 one by one, then parallel_insert_f32 with row pointers, then search."""
    d = 16
    X = pkg.datagen.uniform(600, d, 4)
    h = pkg.Hnsw(12, 1000, 16, 48, "DistL2")
    for i in range(40):
        h.insert((X[i], 1000 + i))
    h.parallel_insert([(X[i], 1000 + i) for i in range(40, 600)])
    assert h.get_nb_point() == 600
    res = h.search(X[123], 3, 32)
    assert res[0].d_id == 1123 and res[0].distance == 0.0
    par = h.parallel_search([X[5], X[599]], 2, 32)
    assert par[0][0].d_id == 1005 and par[1][0].d_id == 1599


@pytest.mark.parametrize("extend,keep_pruned", [(True, False), (False, True), (True, True)])
def test_serial_gpu_build_options_equal_oracle(pkg, po, extend, keep_pruned):
    """set_extend_candidates / set_keeping_pruned (hnsw.rs:845-870): serial GPU build == oracle graph."""
    n, d, M, efc = 1200, 12, 6, 40
    X = pkg.datagen.uniform(n, d, 21)
    o = po.Oracle(M, n, 16, efc, "DistL2", d, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.set_extend_candidates(extend)
    o.set_keeping_pruned(keep_pruned)
    levels = o.draw_levels(n)
    o.insert_batch(X, levels=levels)
    h = pkg.Hnsw(M, n, 16, efc, "DistL2")
    h.set_extend_candidates(extend)
    h.set_keeping_pruned(keep_pruned)
    h.set_insert_batching(1 << 30, 1)
    h.insert_flat(X, levels=levels)
    goff, gids, gds = h.export_layer(0)
    ooff, oids, ods = o.export_layer(0)
    assert np.array_equal(goff, ooff) and np.array_equal(gids, oids)
    assert np.array_equal(gds.view(np.uint32), ods.view(np.uint32))
    with pytest.raises(pkg.HnswError):
        pkg.Hnsw(32, 100, 16, 48, "DistL2").set_extend_candidates(True)   # ef_c <= 2M: refused, not ignored

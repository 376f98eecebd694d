"""GPU tests of link mode 1 (hnsw_b200_set_link_mode): every back-link of an insert filed in the layer it was made in,
instead of under the new point's level as the reference does (hnsw.rs:1257).

1. Serial builds (one insert in flight) equal the oracle's mode-1 MODE_DET / ORDER_GPU build bit for bit, on every
   row-chunk form, several element types and metrics, the 128-slot and generic insert queues and with
   extend_candidates + keep_pruned; lean, generic, filtered and std-tie searches on them equal the oracle's.
2. A build that switches mode half-way equals the oracle doing the same.
3. Production (batched) builds: recall within 0.01 of the oracle's serial mode-1 build and at least the GPU mode-0
   build's, and at most a tenth of mode 0's upper-level points without a layer-0 in-link.
The oracle's mode-1 builds are tests/linkgraph.py's insert_link_mode1 (the oracle itself restates only the reference's
rule).
4. Settings: default, refusals, partitions; dump and reload.
"""
import numpy as np
import pytest

from answers import same
from linkgraph import insert_link_mode1, without_layer0_inlink
from util import csr_lists, recall_ids

pytestmark = pytest.mark.gpu

N, M = 1000, 8


def numpy_data(dtype, metric, n, d, seed):
    """rows from numpy's generator (f32 in [0, 1)), not datagen's as graphs.data draws them"""
    rng = np.random.default_rng(seed)
    dt = np.dtype(dtype)
    if dt == np.float32:
        return rng.random((n, d), dtype=np.float32)
    hi = {"DistHamming": 3}.get(metric, {np.dtype(np.uint8): 256, np.dtype(np.uint16): 5000}.get(dt, 2000))
    lo = -hi if dt == np.int32 and metric != "DistHamming" else 0
    return rng.integers(lo, hi, (n, d)).astype(dt)


def promoting_levels(po, n, seed):
    """drawn levels, capped so that the entry point is promoted at points 3, 40, 200 and 600 (the last by two layers)"""
    lv = po.Oracle(M, n, 16, 48, "DistL2", 4, seed=seed).draw_levels(n)
    i = np.arange(n)
    lv = np.minimum(lv, np.select([i < 3, i < 40, i < 200, i < 600], [0, 1, 2, 3], 5))
    for p, l in ((3, 1), (40, 2), (200, 3), (600, 5)):
        lv[p] = l
    return lv.astype(np.int32)


def oracle(po, dtype, metric, d, efc, n=N, extend=False, keep_pruned=False):
    o = po.Oracle(M, n, 16, efc, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.set_extend_candidates(extend)
    o.set_keeping_pruned(keep_pruned)
    return o


def engine(pkg, dtype, metric, d, efc, n=N, extend=False, keep_pruned=False):
    h = pkg.Hnsw(M, n, 16, efc, metric, dtype=dtype)
    h.set_extend_candidates(extend)
    h.set_keeping_pruned(keep_pruned)
    h.set_insert_batching(1 << 30, 1)   # one insert in flight: a deterministic serial build
    return h


def assert_same_lists(h, o):
    """graphs.assert_same_graph's rule, with the link distances of the upper layers compared too"""
    lv, rk, og, entry = h.export_points()
    olv, ork, oog = o.export_points()
    assert entry == o.entry
    assert np.array_equal(lv, olv) and np.array_equal(rk, ork) and np.array_equal(og, oog)
    for layer in range(0, int(olv.max()) + 1):
        goff, gids, gds = h.export_layer(layer)
        ooff, oids, ods = o.export_layer(layer)
        gl, ol = csr_lists(goff, gids), csr_lists(ooff, oids)
        gd, od = csr_lists(goff, gds.view(np.uint32)), csr_lists(ooff, ods.view(np.uint32))
        for p in range(len(lv)):
            if layer > 0 and not gl[p] and olv[p] < layer:   # a list no search can reach, which the engine does not store
                continue
            assert gl[p] == ol[p], (layer, p, gl[p], ol[p])
            assert gd[p] == od[p], ("link distances", layer, p)


def same_with_counters(h, o, Q, k, ef, what, filt=None):
    o.counters()
    want = o.search_batch(Q, k, ef, filter_ids=filt)
    co = o.counters()
    h.enable_stats(filt is None)
    h.get_stats()
    same(h.search_flat(Q, k, ef, filter=filt), want, what)
    cg = h.get_stats()
    h.enable_stats(False)
    if filt is None:
        for key in ("evals", "expansions", "adj_read"):
            assert cg[key] == co[key], (what, key, cg, co)


SERIAL_CASES = [
    (np.float32, "DistL2", 24, 200, False), (np.float32, "DistL2", 48, 200, False),
    (np.float32, "DistL2", 100, 200, False), (np.float32, "DistL2", 150, 200, False),
    (np.float32, "DistCosine", 100, 200, False), (np.uint8, "DistHamming", 100, 48, False),
    (np.uint16, "DistL1", 200, 48, False), (np.int32, "DistL2", 24, 48, False),
    (np.float32, "DistL2", 24, 48, False), (np.float32, "DistL2", 48, 300, False),
    (np.float32, "DistL2", 48, 200, True),
]


@pytest.mark.parametrize("dtype,metric,d,efc,options", SERIAL_CASES,
                         ids=[f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}-efc{c[3]}" + ("-ext-kp" if c[4] else "")
                              for c in SERIAL_CASES])
def test_serial_mode1_build_and_search_equal_oracle(pkg, po, dtype, metric, d, efc, options):
    X = numpy_data(dtype, metric, N, d, d + efc)
    levels = promoting_levels(po, N, d)
    o = oracle(po, dtype, metric, d, efc, extend=options, keep_pruned=options)
    insert_link_mode1(o, X, levels)
    h = engine(pkg, dtype, metric, d, efc, extend=options, keep_pruned=options)
    h.set_link_mode(1)
    h.insert_flat(X, levels=levels)
    assert h.get_link_mode() == 1
    assert_same_lists(h, o)
    Q = numpy_data(dtype, metric, 100, d, d + 1)
    Q[:10] = X[:10]
    same_with_counters(h, o, Q, 10, 64, "lean")
    same_with_counters(h, o, Q, 10, 129, "generic")
    same_with_counters(h, o, Q, 10, 24, "filtered", filt=np.arange(1, N, 3))
    o.set_mode(po.MODE_STD)
    h.set_tie_mode(1)
    same_with_counters(h, o, Q, 10, 32, "std-tie")


def test_mode_switch_between_inserts_equals_oracle(pkg, po):
    d, efc = 24, 200
    X = numpy_data(np.float32, "DistL2", N, d, 5)
    levels = promoting_levels(po, N, 5)
    half = N // 2
    o = oracle(po, np.float32, "DistL2", d, efc)
    h = engine(pkg, np.float32, "DistL2", d, efc)
    o.insert_batch(X[:half], levels=levels[:half])
    h.insert_flat(X[:half], levels=levels[:half])
    h.set_link_mode(1)
    insert_link_mode1(o, X[half:], levels[half:])
    h.insert_flat(X[half:], ids=np.arange(half, N), levels=levels[half:])
    assert_same_lists(h, o)


@pytest.mark.parametrize("n,d,kind", [(20000, 25, "uniform"), (20000, 128, "clustered")])
def test_batched_mode1_build_recall_and_inlinks(pkg, po, n, d, kind):
    efc = 200
    X = pkg.datagen.make(kind, n, d, 1)
    Q = pkg.datagen.make(kind, 500, d, 2)
    ti, _ = po.bruteforce(X, Q, 10, "DistL2")
    o = po.Oracle(16, n, 16, efc, "DistL2", d, mode=po.MODE_DET, order=po.ORDER_GPU)
    levels = o.draw_levels(n)
    insert_link_mode1(o, X, levels)
    _, _, oi, _, oc = o.search_batch(Q, 10, 64)
    r_o = recall_ids(oi, oc, ti)
    rec, orphans, selfhit = {}, {}, {}
    for mode in (0, 1):
        h = pkg.Hnsw(16, n, 16, efc, "DistL2")
        h.set_link_mode(mode)
        h.insert_flat(X, levels=levels)
        _, _, gi, _, gc = h.search_flat(Q, 10, 64)
        rec[mode] = recall_ids(gi, gc, ti)
        _, _, _, entry = h.export_points()
        orphans[mode] = len(without_layer0_inlink(h.export_layer(0), levels, entry))
        _, _, si, _, _ = h.search_flat(X, 1, 64)
        selfhit[mode] = float((si[:, 0] == np.arange(n)).mean())
        h.close()
    print(f"{kind} {n}x{d}: recall@10 ef 64 oracle mode 1 {r_o:.4f}, gpu mode 0 {rec[0]:.4f}, gpu mode 1 {rec[1]:.4f}; "
          f"level >= 1 points without a layer-0 in-link {orphans[0]} -> {orphans[1]}; "
          f"self-retrieval {selfhit[0]:.4f} -> {selfhit[1]:.4f}")
    assert rec[1] >= r_o - 0.01
    assert rec[1] >= rec[0]
    assert orphans[1] <= orphans[0] / 10


def test_link_mode_settings(pkg):
    h = pkg.Hnsw(M, 100, 16, 48, "DistL2")
    assert h.get_link_mode() == 0
    for bad in (2, -1, 7):
        with pytest.raises(pkg.HnswError):
            h.set_link_mode(bad)
        assert h.get_link_mode() == 0
    h.set_link_mode(1)
    with pytest.raises(pkg.HnswError):
        h.set_link_mode(5)
    assert h.get_link_mode() == 1
    h.set_link_mode(0)
    assert h.get_link_mode() == 0


@pytest.mark.parametrize("when", ["before", "after"])
def test_partitions_build_in_mode1(pkg, po, when):
    P, n, d, efc = 2, 2000, 24, 200
    X = numpy_data(np.float32, "DistL2", n, d, 9)
    levels = po.Oracle(M, n, 16, efc, "DistL2", d).draw_levels(n)
    h = pkg.Hnsw(M, n, 16, efc, "DistL2")
    h.set_insert_batching(1 << 30, 1)
    if when == "before":
        h.set_link_mode(1)
    h.partition([0] * P)
    if when == "after":
        h.set_link_mode(1)
    assert h.get_link_mode() == 1
    h.insert_flat(X, levels=levels)
    for p in range(P):
        v = h.partition_view(p)
        assert v.get_link_mode() == 1
        with pytest.raises(pkg.HnswError):
            v.set_link_mode(0)
        o = oracle(po, np.float32, "DistL2", d, efc, n=len(X[p::P]))
        insert_link_mode1(o, X[p::P], levels[p::P], ids=np.arange(p, n, P))
        assert_same_lists(v, o)


def test_mode1_dump_reload_and_insert(tmp_path, pkg, po):
    import dumpfmt
    n, d, efc = 1200, 20, 48
    X = numpy_data(np.float32, "DistL2", n, d, 13)
    levels = promoting_levels(po, n, 13)
    h = engine(pkg, np.float32, "DistL2", d, efc)
    h.set_link_mode(1)
    h.insert_flat(X, levels=levels)
    h.file_dump(tmp_path, "lm1")
    # the independent reader finds every exported list at every layer, with its distances
    b = dumpfmt.read_dump(str(tmp_path / "lm1"), np.float32)
    lv, rk, og, entry = h.export_points()
    order = np.lexsort((rk, lv))
    inv = np.empty(n, np.int64)
    inv[order] = np.arange(n)
    assert b["entry"] == inv[entry] and np.array_equal(b["origin"], og[order])
    for layer in range(int(lv.max()) + 1):
        off, ids, ds = h.export_layer(layer)
        for p in range(n):
            want = [(int(inv[ids[j]]), float(ds[j])) for j in range(int(off[p]), int(off[p + 1]))]
            assert b["lists"][layer][int(inv[p])] == want, (layer, p)
    # reload: mode 0 (dumps store no mode), same answers
    h2 = pkg.Hnsw.load(tmp_path, "lm1", "DistL2")
    assert h2.get_link_mode() == 0
    Q = numpy_data(np.float32, "DistL2", 100, d, 14)
    a1, a2 = h.search_flat(Q, 10, 48), h2.search_flat(Q, 10, 48)
    assert np.array_equal(a1[0], a2[0]) and np.array_equal(a1[1].view(np.uint32), a2[1].view(np.uint32))
    # an insert into the reloaded handle in mode 1 equals the oracle's on the same graph
    lv2, _, og2, entry2 = h2.export_points()
    o = po.Oracle(M, n + 50, 16, efc, "DistL2", d, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.import_graph(h2.export_vectors(), og2, lv2, entry2, {l: h2.export_layer(l) for l in range(int(lv2.max()) + 1)})
    o.set_extend_candidates(True)   # a reload turns extend_candidates on (hnswio.rs:510, 599); set it on both explicitly
    extra = numpy_data(np.float32, "DistL2", 50, d, 15)
    xlev = np.minimum(po.Oracle(M, 50, 16, efc, "DistL2", d, seed=16).draw_levels(50), 2)
    insert_link_mode1(o, extra, xlev, ids=np.arange(7000, 7050))
    h2.set_extend_candidates(True)
    h2.set_insert_batching(1 << 30, 1)
    h2.set_link_mode(1)
    h2.insert_flat(extra, ids=np.arange(7000, 7050), levels=xlev)
    assert_same_lists(h2, o)

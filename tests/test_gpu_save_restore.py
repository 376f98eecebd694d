"""GPU tests of saved indexes (Hnsw.save / Hnsw.restore, include/hnsw_b200.h "Saved indexes"): a restored handle is
the same index as the saved one, bit for bit, in every search, column, export and continued build; partitioned handles
round-trip; save's pairs are file_dump's bytes and still load; refusals leave no handle and no files; and a manifest
and pair written by an independent writer (tests/savefmt.py, oracle/dumpfmt.py) restore an oracle graph with the
oracle's ranks."""
import os

import numpy as np
import pytest

import graphs
import restrict
import savefmt
from util import oracle_layers

pytestmark = pytest.mark.gpu

K, EF = 10, 48


def _data(dtype, metric, n, d, seed):
    X = graphs.data(dtype, metric, n, d, seed)
    X[1::40] = X[0::40][:len(X[1::40])]   # identical point pairs: equal distances, so ties occur
    return X


def _build(pkg, dtype, metric, n=3000, d=16, M=8, efc=40, tie=0, link=1, extend=False, P=None, seed=1):
    X = _data(dtype, metric, n, d, seed)
    h = pkg.Hnsw(M, n + 2000, 16, efc, metric, dtype=dtype)
    if P is not None:
        h.partition([0] * P)
    h.set_level_seed(987 + seed)
    h.set_link_mode(link)
    h.set_tie_mode(tie)
    h.set_keeping_pruned(True)
    h.set_extend_candidates(extend)
    h.set_insert_batching(8, 256)
    ids = 50_000 + 7 * np.arange(n, dtype=np.uint64)      # origin ids apart from the ranks
    h.insert_flat(X[:n // 2], ids=ids[:n // 2])
    h.insert_flat(X[n // 2:], ids=ids[n // 2:])
    return h, X, ids


def _columns(h, n, seed=3):
    lab, attr = restrict.point_labels(n, seed), restrict.point_attrs(n, seed)
    h.set_labels(0, lab)
    h.set_attributes(0, attr)
    dele = np.unique(np.random.default_rng(seed).choice(n, n // 15, replace=False))
    h.delete_points(dele)
    return lab, attr


def _flat(a):
    return tuple(np.ascontiguousarray(x).view(np.uint8).tobytes() if isinstance(x, np.ndarray) else x for x in a)


def _every_answer(h, Q, ids, n):
    """(name, answers, counters) of every search and count the handle serves, statistics on"""
    nq = len(Q)
    rng = np.random.default_rng(5)
    qlab = np.array([[0, 1, 7, 8, 5][i % 5] for i in range(nq)], np.uint32)
    sets = [[0, 1], [7, 8], [1], [0xFFFFFFFF], [3, 9, 0]] * (nq // 5)
    ranges = np.array([[-500, 500], [0, 10], [-1000, -900], [-(1 << 63), (1 << 63) - 1]] * (nq // 4), np.int64)
    excl = [rng.choice(n, i % 7 * 3, replace=False) for i in range(nq)]
    qids = rng.choice(n, nq, replace=False).astype(np.uint64)
    flist = np.sort(ids[rng.random(n) < 0.3])
    calls = [
        ("search_flat", lambda: h.search_flat(Q, K, EF)),
        ("parallel_search", lambda: [[(x.d_id, np.float32(x.distance).view(np.uint32)) for x in r]
                                     for r in h.parallel_search(list(Q), K, EF)]),
        ("search_exact", lambda: h.search_exact(Q, K)),
        ("filter_t", lambda: h.search_flat(Q, K, EF, filter=flist)),
        ("labeled", lambda: h.search_flat_labeled(Q, K, EF, qlab)),
        ("exact_labeled", lambda: h.search_exact_labeled(Q, K, qlab)),
        ("label_sets", lambda: h.search_flat_label_sets(Q, K, EF, sets)),
        ("ranges", lambda: h.search_flat_ranges(Q, K, EF, ranges)),
        ("ranges_in_sets", lambda: h.search_flat_ranges(Q, K, EF, ranges, sets=sets)),
        ("exact_ranges", lambda: h.search_exact_ranges(Q, K, ranges, sets=sets)),
        ("excluding", lambda: h.search_flat_excluding(Q, K, EF, excl)),
        ("exact_excluding", lambda: h.search_exact_excluding(Q, K, excl)),
        ("by_id", lambda: h.search_by_id(qids, K, EF)),
        ("by_id_self", lambda: h.search_by_id(qids, K, EF, exclude_self=True)),
        ("exact_by_id_self", lambda: h.search_exact_by_id(qids, K, sets=sets, exclude_self=True)),
        ("planned", lambda: h.search_planned(Q, K, EF, excluded=excl, sets=sets)),
        ("count_admitted", lambda: h.count_admitted(sets=sets, ranges=ranges, n=nq)),
        ("radius", lambda: h.search_exact_radius(Q, np.float32(0.5 if h.dtype == np.float32 else 40), K)),
    ]
    out = []
    h.enable_stats(True)
    for name, call in calls:
        h.get_stats(reset=True)
        out.append((name, _flat(call()) if name != "parallel_search" else call(), h.get_stats(reset=True)))
    with h.make_filter(flist) as rf:
        h.get_stats(reset=True)
        out.append(("resident", _flat(h.search_flat(Q, K, EF, filter=rf)), h.get_stats(reset=True)))
        out.append(("exact_resident", _flat(h.search_exact(Q, K, filter=rf)), h.get_stats(reset=True)))
    h.enable_stats(False)
    return out


def _same_answers(a, b):
    for (na, xa, sa), (nb, xb, sb) in zip(a, b):
        assert na == nb
        assert xa == xb, f"{na}: answers differ after restore"
        assert sa == sb, f"{na}: counters differ after restore ({sa} vs {sb})"


def _state(h):
    n = h.get_nb_point()
    lv, rk, og, e = h.export_points()
    top = int(lv.max()) + 1 if n else 0
    layers = [tuple(x.tobytes() for x in h.export_layer(l)) for l in range(top + 1)]
    return (n, lv.tobytes(), rk.tobytes(), og.tobytes(), e, layers, h.get_max_level_observed(), h.get_link_mode(),
            h.get_labels(0, n).tobytes(), h.get_attributes(0, n).tobytes(), h.deleted().tobytes(),
            h.export_vectors().tobytes())


@pytest.mark.parametrize("dtype,metric,tie", [(np.float32, "DistL2", 0), (np.float32, "DistCosine", 0),
                                              (np.uint8, "DistHamming", 1), (np.uint16, "DistL1", 0)])
def test_round_trip_is_the_same_index(tmp_path, pkg, dtype, metric, tie):
    n = 3000
    h, X, ids = _build(pkg, dtype, metric, n=n, tie=tie)
    _columns(h, n)
    lv = h.export_points()[0]
    assert lv.max() >= 1 and not np.array_equal(savefmt.file_order(lv), np.arange(n)), "file order must differ from rank order"
    assert h.save(tmp_path, "idx") == "idx"
    assert sorted(os.listdir(tmp_path)) == ["idx.hnsw.b200", "idx.hnsw.data", "idx.hnsw.graph"]
    r = pkg.Hnsw.restore(tmp_path, "idx")
    assert (r.dtype, r.dist_name, r.max_nb_connection, r.ef_construction) == (np.dtype(dtype), metric, 8, 40)
    assert _state(r) == _state(h)
    Q = _data(dtype, metric, 200, 16, 9)
    Q[:20] = X[:20]
    _same_answers(_every_answer(r, Q, ids, n), _every_answer(h, Q, ids, n))
    if not tie:   # the std tie mode, set alike on both after the restore
        for x in (h, r):
            x.set_tie_mode(1)
        assert _flat(r.search_flat(Q, K, EF)) == _flat(h.search_flat(Q, K, EF))
    # the manifest as the independent reader sees it
    m = savefmt.unpack(open(tmp_path / "idx.hnsw.b200", "rb").read())
    savefmt.check_pairs(str(tmp_path), "idx", m)
    assert m["counts"] == [n] and np.array_equal(m["pairs"][0][4], savefmt.file_order(lv))
    assert np.array_equal(m["labels"], h.get_labels(0, n)) and np.array_equal(m["attrs"], h.get_attributes(0, n))
    assert np.array_equal(m["deleted"], h.deleted()) and m["link_mode"] == 1 and m["tie_std"] == bool(tie)


@pytest.mark.parametrize("link,extend", [(0, False), (1, False), (0, True)])
def test_continued_build_equals_the_uninterrupted_one(tmp_path, pkg, link, extend):
    n1, n2, M, efc = 2000, 1500, 8, 40
    dtype, metric = np.float32, "DistL2"
    X = _data(dtype, metric, n1 + 2 * n2, 16, 4)
    ids = np.arange(n1 + 2 * n2, dtype=np.uint64) * 3 + 11

    def fresh():
        h = pkg.Hnsw(M, n1, 16, efc, metric)       # max_elements below the total: the store grows on the way
        h.set_level_seed(42)
        h.set_link_mode(link)
        h.set_extend_candidates(extend)
        h.set_insert_batching(4, 128)
        h.modify_level_scale(0.6)
        return h
    full, h = fresh(), fresh()
    for x in (full, h):
        x.insert_flat(X[:n1], ids=ids[:n1])
    h.save(tmp_path, "c")
    r = pkg.Hnsw.restore(tmp_path, "c")
    if extend:   # a plain load would switch it on whatever it was; restore keeps the saved value
        assert pkg.load_library().hnsw_b200_get_extend_candidates(r._h) == 1
    else:
        assert pkg.load_library().hnsw_b200_get_extend_candidates(r._h) == 0
        assert pkg.load_library().hnsw_b200_get_extend_candidates(pkg.Hnsw.load(tmp_path, "c", metric)._h) == 1
    for lo, hi in ((n1, n1 + n2), (n1 + n2, n1 + 2 * n2)):
        for x in (full, h, r):
            x.insert_flat(X[lo:hi], ids=ids[lo:hi])
    assert _state(r) == _state(h) == _state(full)


def _global_rows(h, Q):
    return _flat(h.search_flat(Q, K, EF)), _flat(h.search_exact(Q, K)), _flat(h.search_by_id(np.arange(40), K, EF))


@pytest.mark.parametrize("P,n", [(2, 2500), (3, 2500), (3, 2)])
def test_partitioned_round_trip(tmp_path, pkg, P, n):
    h, X, ids = _build(pkg, np.float32, "DistL2", n=n, P=P)
    if n > 100:
        _columns(h, n)
    base = h.save(tmp_path, "part", overwrite=False)
    names = sorted(os.listdir(tmp_path))
    assert "part.hnsw.b200" in names and all(f"part-p{p}.hnsw.graph" in names for p in range(min(P, n)))
    assert len(names) == 1 + 2 * min(P, n)     # a partition without a point gets no pair
    m = savefmt.unpack(open(tmp_path / "part.hnsw.b200", "rb").read())
    assert m["counts"] == [(n + P - 1 - p) // P for p in range(P)]
    r = pkg.Hnsw.restore(tmp_path, base, devices=[0] * P)
    assert r.partition_count() == P and r.get_nb_point() == n
    Q = _data(np.float32, "DistL2", 100, 16, 8)
    if n > 100:
        assert _global_rows(r, Q) == _global_rows(h, Q)
        assert r.get_labels(0, n).tobytes() == h.get_labels(0, n).tobytes()
        assert r.deleted().tobytes() == h.deleted().tobytes()
    else:
        assert _flat(r.search_flat(Q, K, EF)) == _flat(h.search_flat(Q, K, EF))
    for p in range(P):
        if (n + P - 1 - p) // P:
            assert _state(r.partition_view(p)) == _state(h.partition_view(p))
    more = _data(np.float32, "DistL2", 700, 16, 12)
    for x in (h, r):
        x.insert_flat(more, ids=np.arange(700, dtype=np.uint64) + 90_000)
    for p in range(P):
        assert _state(r.partition_view(p)) == _state(h.partition_view(p))
    assert _flat(r.search_flat(Q, K, EF)) == _flat(h.search_flat(Q, K, EF))
    with pytest.raises(pkg.HnswError):
        pkg.Hnsw.restore(tmp_path, base, devices=[0] * (P + 1))
    with pytest.raises(pkg.HnswError):
        pkg.Hnsw.restore(tmp_path, base)


def test_partitioned_restore_onto_other_devices(tmp_path, pkg):
    ndev = pkg.load_library().hnsw_b200_device_count()
    if ndev < 2:
        pytest.skip("needs two GPUs")
    h, X, ids = _build(pkg, np.float32, "DistL2", n=2000, P=2)
    h.save(tmp_path, "dev")
    r = pkg.Hnsw.restore(tmp_path, "dev", devices=[1, 0])
    Q = _data(np.float32, "DistL2", 100, 16, 8)
    assert _global_rows(r, Q) == _global_rows(h, Q)


def test_pairs_are_file_dump_bytes_and_still_load(tmp_path, pkg):
    h, X, ids = _build(pkg, np.uint16, "DistL1", n=2000)
    _columns(h, 2000)
    h.save(tmp_path, "s")
    h.file_dump(tmp_path, "d")
    for ext in ("graph", "data"):
        assert open(tmp_path / f"s.hnsw.{ext}", "rb").read() == open(tmp_path / f"d.hnsw.{ext}", "rb").read()
    a, b = pkg.Hnsw.load(tmp_path, "s", "DistL1", dtype=np.uint16), pkg.Hnsw.load(tmp_path, "d", "DistL1", dtype=np.uint16)
    assert _state(a) == _state(b)
    Q = _data(np.uint16, "DistL1", 80, 16, 8)
    assert _flat(a.search_flat(Q, K, EF)) == _flat(b.search_flat(Q, K, EF))
    # a partitioned save's pairs: partition_view(p)'s file_dump bytes, each loading as that partition searches
    hp, _, _ = _build(pkg, np.float32, "DistL2", n=1500, P=2)
    hp.save(tmp_path, "ps")
    Qf = _data(np.float32, "DistL2", 80, 16, 8)
    for p in range(2):
        v = hp.partition_view(p)
        v.file_dump(tmp_path, f"pv{p}")
        for ext in ("graph", "data"):
            assert open(tmp_path / f"ps-p{p}.hnsw.{ext}", "rb").read() == open(tmp_path / f"pv{p}.hnsw.{ext}", "rb").read()
        got = pkg.Hnsw.load(tmp_path, f"ps-p{p}", "DistL2").search_flat(Qf, K, EF)
        want = v.search_flat(Qf, K, EF)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))


def test_refusals_leave_no_handle_and_no_files(tmp_path, pkg):
    h, X, ids = _build(pkg, np.float32, "DistL2", n=1200)
    h.save(tmp_path, "r")
    raw = bytearray(open(tmp_path / "r.hnsw.data", "rb").read())
    raw[len(raw) // 2] ^= 0x10
    open(tmp_path / "r.hnsw.data", "wb").write(bytes(raw))
    with pytest.raises(pkg.HnswError, match="r.hnsw.data"):
        pkg.Hnsw.restore(tmp_path, "r")
    with pytest.raises(pkg.HnswError, match="r.hnsw.b200"):
        pkg.Hnsw.restore(tmp_path, "r", devices=[0, 0])
    os.remove(tmp_path / "r.hnsw.b200")
    with pytest.raises(pkg.HnswError, match="r.hnsw.b200"):
        pkg.Hnsw.restore(tmp_path, "r")
    out = tmp_path / "out"
    out.mkdir()
    hp, _, _ = _build(pkg, np.float32, "DistL2", n=300, P=2)
    with pytest.raises(pkg.HnswError, match="partition view"):
        hp.partition_view(0).save(out, "v")
    with pytest.raises(pkg.HnswError):
        pkg.Hnsw(8, 10, 16, 20, "DistL2").save(out, "empty")
    assert os.listdir(out) == []


def test_independent_writer_restores_the_oracle_graph(tmp_path, pkg, po):
    import dumpfmt
    n, d, M, efc = 2000, 16, 8, 60
    X = pkg.datagen.uniform(n, d, 5)
    o = po.Oracle(M, n, 16, efc, "DistL2", d, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X, ids=np.arange(100, 100 + n))
    lv, rk, og = o.export_points()
    assert not np.array_equal(savefmt.file_order(lv), np.arange(n))
    dumpfmt.write_dump(str(tmp_path / "orc"), X, og, lv, o.entry, oracle_layers(o, int(lv.max()) + 1), M, efc,
                       1 / np.log(M), "DistL2")
    g, gs = savefmt.file_sum(str(tmp_path / "orc.hnsw.graph"))
    dz, ds = savefmt.file_sum(str(tmp_path / "orc.hnsw.data"))
    lab = (np.arange(n) % 4).astype(np.uint32)
    m = {"dtype": 0, "metric": 1, "M": M, "max_layer": 16, "dim": d, "ef_c": efc, "max_elements": n, "link_mode": 0,
         "visited_stages": 0, "batch_ratio": 16, "batch_max": 16384, "extend": False, "keep_pruned": False,
         "tie_std": False, "level_scale": 1 / np.log(M), "rng": 397, "counts": [n],
         "pairs": [(g, gs, dz, ds, savefmt.file_order(lv))], "labels": lab, "attrs": None, "deleted": None}
    open(tmp_path / "orc.hnsw.b200", "wb").write(savefmt.pack(m))
    h = pkg.Hnsw.restore(tmp_path, "orc")
    Q = pkg.datagen.uniform(100, d, 6)
    oo, od, oi, _, oc = o.search_batch(Q, 10, 48)
    go, gd, gi, _, gc = h.search_flat(Q, 10, 48)
    assert np.array_equal(gc, oc) and np.array_equal(go, oo) and np.array_equal(gi, oi)   # the oracle's ranks
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32))
    assert np.array_equal(h.get_labels(0, n), lab)
    hl, hr, ho, he = h.export_points()
    assert np.array_equal(hl, lv) and np.array_equal(ho, og) and he == o.entry

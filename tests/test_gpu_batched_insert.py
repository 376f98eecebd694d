"""Batched GPU builds, bit-exact against the oracle's batch-synchronous build.

Index::insert_batch cuts every insert call into batches (tests/batched.py engine_batches restates the schedule).  Phase
A of a batch (insert_search_kernel) searches the graph as it stood when the batch began, phase B (insert_link_kernel)
files the back-links under per-point locks; DESIGN.md §4.3 argues the result is deterministic.  pyoracle's
insert_batched restates those semantics, so every batched build here must equal it exactly:
  * entry point, levels, ranks and origins equal, every materialised list equal, layer-0 link distances bit-equal
    (graphs.assert_same_graph);
  * the insert path's traversal counters `expansions` and `adj_read` equal the oracle's.  `evals` is not compared: the
    kernel does not count dist_to_entry (hnsw.rs:1110-1112) or the recompute at hnsw.rs:1146, and it evaluates every
    kept neighbour of a selection step at once, where the oracle stops at the first one that rejects the candidate.

The cases: the insert instantiation matrix of test_gpu_matrix under the default schedule, and per element type under
(ratio 1, max_batch 1 << 30), the stalest snapshot there is (every batch doubles the graph), with a lean and a generic
search on each graph; long lists (2M = 80, 258) under lock contention; extend_candidates + keep_pruned; link mode 1 and a
switch to it between calls; incremental calls into a growing index and into an imported graph; per-point layer masks;
partitions building concurrently on one device; the row-pointer upload across its 8 MB staging chunk; and bench.py's
c2 graph at full size.  test_zz_every_insert_kernel_ran_batched checks that every compiled insert_search_kernel entry
point ran in a bit-exact case of this module.
"""
import re
import subprocess
import time

import numpy as np
import pytest

from answers import same
from batched import engine_batches, promoting_levels
from graphs import (CASES, INSERT_CASES, LOG_METRICS, NTH, State, assert_same_graph, case_id, cuobjdump, data,
                    insert_both, make_engine, make_oracle)
from util import oracle_layers

pytestmark = pytest.mark.gpu

T0 = time.time()
LEDGER = set()   # insert_search_kernel instantiations that ran in a case compared bit for bit
DONE = []        # ids of the cases that ran to the end
N, M = 1000, 8
STALE = (1, 1 << 30)   # every batch as large as the graph before it


def same_with_counters(h, o, Q, k, ef, what):
    o.counters()
    want = o.search_batch(Q, k, ef, nthreads=NTH)
    co = o.counters()
    h.enable_stats(True)
    h.get_stats()
    same(h.search_flat(Q, k, ef), want, what)
    cg = h.get_stats()
    h.enable_stats(False)
    for key in ("evals", "expansions", "adj_read"):
        assert cg[key] == co[key], (what, key, cg, co)


def prob_data(n, d, seed):
    X = np.random.default_rng(seed).random((n, d), dtype=np.float32) + np.float32(1e-3)
    return X / X.sum(1, keepdims=True)


def build_and_search(pkg, po, dtype, metric, d, efc, X, levels, sched=None, n=N):
    o = make_oracle(po, dtype, metric, d, M, efc, n)
    h = make_engine(pkg, dtype, metric, M, efc, n, sched)
    insert_both(pkg, h, o, X, levels, State(), sched, ledger=LEDGER)
    assert_same_graph(h, o, n)
    Q = X[::10][:100].copy() if metric == "DistHellinger" else data(dtype, metric, 100, d, d + 100)
    Q[:10] = X[:10]
    same_with_counters(h, o, Q, 10, 64, "lean")
    same_with_counters(h, o, Q, 10, 129, "generic")
    h.close()


# ---------------------------------------------------------------- the insert instantiation matrix, batched
MATRIX = ([(c[0], c[1], c[2], c[3], 200 if np.dtype(c[0]) == np.float32 else 48) for c in CASES]
          + [(np.float32, m, d, False, efc) for m, d, efc in INSERT_CASES]
          + [(np.float32, "DistHellinger", 24, False, 200)])


def matrix_id(c):
    return case_id(c[:4]) + f"-efc{c[4]}"


@pytest.mark.parametrize("dtype,metric,d,ties,efc", MATRIX, ids=[matrix_id(c) for c in MATRIX])
def test_batched_matrix(pkg, po, dtype, metric, d, ties, efc):
    X = prob_data(N, d, d) if metric == "DistHellinger" else data(dtype, metric, N, d, d + 7, ties)
    build_and_search(pkg, po, dtype, metric, d, efc, X, promoting_levels(po, N, d))
    DONE.append(matrix_id((dtype, metric, d, ties, efc)))


STALE_CASES = [(np.float32, "DistL2", 24, 200), (np.uint8, "DistL1", 100, 48), (np.uint16, "DistJaccard", 50, 48),
               (np.uint32, "DistHamming", 24, 48), (np.int32, "DistL2", 24, 48)]


@pytest.mark.parametrize("dtype,metric,d,efc", STALE_CASES, ids=[case_id(c[:3] + (False,)) for c in STALE_CASES])
def test_batched_stalest_schedule(pkg, po, dtype, metric, d, efc):
    X = data(dtype, metric, N, d, d + 8)
    build_and_search(pkg, po, dtype, metric, d, efc, X, promoting_levels(po, N, d + 1), sched=STALE)
    DONE.append(f"stale-{case_id((dtype, metric, d, False))}")


# ---------------------------------------------------------------- long lists, options, link mode
@pytest.mark.parametrize("M2,efc", [(40, 120), (40, 300), (129, 120), (129, 300)])
def test_long_lists(pkg, po, M2, efc):
    """2M = 80 and 258 slots at layer 0: phase B's shift spans several 32-wide chunks, and with every batch doubling the
    graph many back-links of one batch meet in the same lists"""
    n, d = 1500, 24
    X = data(np.float32, "DistL2", n, d, M2 + efc)
    lv = promoting_levels(po, n, M2)
    o = make_oracle(po, np.float32, "DistL2", d, M2, efc, n)
    h = make_engine(pkg, np.float32, "DistL2", M2, efc, n, STALE)
    insert_both(pkg, h, o, X, lv, State(), STALE, ledger=LEDGER)
    assert_same_graph(h, o, n)
    assert int(np.diff(h.export_layer(0)[0].astype(np.int64)).max()) > 32
    DONE.append(f"long-{M2}-{efc}")


@pytest.mark.parametrize("sched", [None, STALE], ids=["default", "stalest"])
def test_extend_candidates_and_keep_pruned(pkg, po, sched):
    d, efc = 48, 200
    X = data(np.float32, "DistL2", N, d, 21)
    lv = promoting_levels(po, N, 21)
    o = make_oracle(po, np.float32, "DistL2", d, M, efc, N, extend=True, keep_pruned=True)
    h = make_engine(pkg, np.float32, "DistL2", M, efc, N, sched, extend=True, keep_pruned=True)
    insert_both(pkg, h, o, X, lv, State(), sched, ledger=LEDGER)
    assert_same_graph(h, o, N)
    DONE.append(f"ext-kp-{sched}")


@pytest.mark.parametrize("sched", [None, STALE], ids=["default", "stalest"])
def test_link_mode1(pkg, po, sched):
    d, efc = 24, 200
    X = data(np.float32, "DistL2", N, d, 22)
    lv = promoting_levels(po, N, 22)
    o = make_oracle(po, np.float32, "DistL2", d, M, efc, N)
    h = make_engine(pkg, np.float32, "DistL2", M, efc, N, sched, link_mode=1)
    insert_both(pkg, h, o, X, lv, State(), sched, link_mode=1, ledger=LEDGER)
    assert_same_graph(h, o, N)
    DONE.append(f"mode1-{sched}")


def test_link_mode_switch_between_calls(pkg, po):
    d, efc, half = 24, 200, N // 2
    X = data(np.float32, "DistL2", N, d, 23)
    lv = promoting_levels(po, N, 23)
    o = make_oracle(po, np.float32, "DistL2", d, M, efc, N)
    h = make_engine(pkg, np.float32, "DistL2", M, efc, N)
    st = State()
    insert_both(pkg, h, o, X[:half], lv[:half], st, ledger=LEDGER)
    h.set_link_mode(1)
    insert_both(pkg, h, o, X[half:], lv[half:], st, ids=np.arange(half, N), link_mode=1, ledger=LEDGER)
    assert_same_graph(h, o, N)
    DONE.append("mode-switch")


# ---------------------------------------------------------------- incremental calls
def test_incremental_calls_and_capacity_growth(pkg, po):
    """the batched twin of test_gpu_edge.test_incremental_inserts_and_capacity_growth: an index created for 16 points
    grows over uneven calls, and every call's schedule starts from the state the previous one left"""
    n, d, efc = 5000, 12, 40
    X = data(np.float32, "DistL2", n, d, 41)
    lv = promoting_levels(po, n, 41)
    o = make_oracle(po, np.float32, "DistL2", d, M, efc, 16)
    h = make_engine(pkg, np.float32, "DistL2", M, efc, 16)
    st, pos = State(), 0
    for sz in (1, 1, 3, 50, 700, 1, 2000, 2244):
        insert_both(pkg, h, o, X[pos:pos + sz], lv[pos:pos + sz], st, ids=np.arange(pos, pos + sz), ledger=LEDGER)
        pos += sz
    assert pos == n and h.get_nb_point() == n
    assert_same_graph(h, o, n)
    DONE.append("incremental")


def test_batched_insert_into_imported_graph(pkg, po):
    """a graph from the oracle's threaded build, imported on both sides, then one batched call"""
    n0, n1, d, efc = 3000, 2000, 24, 100
    X = data(np.float32, "DistL2", n0 + n1, d, 42)
    src = make_oracle(po, np.float32, "DistL2", d, M, efc, n0)
    src.insert_batch(X[:n0], nthreads=8)
    lv0, _, og0 = src.export_points()
    V0 = src.export_vectors()   # a threaded build stores the rows in completion order
    h = make_engine(pkg, np.float32, "DistL2", M, efc, n0 + n1)
    h.import_graph(V0, og0, lv0, src.entry, oracle_layers(src))
    o = make_oracle(po, np.float32, "DistL2", d, M, efc, n0 + n1)
    o.import_graph(V0, og0, lv0, src.entry, {l: src.export_layer(l) for l in range(16)})
    st = State()
    st.n, st.top = n0, int(lv0[src.entry])
    lv1 = np.minimum(promoting_levels(po, n1, 43), int(lv0.max()))
    lv1[700] = int(lv0.max()) + 1   # one promotion in the middle of the call
    insert_both(pkg, h, o, X[n0:], lv1, st, ids=np.arange(n0, n0 + n1), ledger=LEDGER)
    assert_same_graph(h, o, n0 + n1)
    DONE.append("imported")


# ---------------------------------------------------------------- layer masks
def test_layer_mask_per_point(pkg, po):
    """Point 0 has level 2 and every point before 320 level 0, so layer 1 is empty (the reference tests emptiness by the
    points of exactly that level, hnsw.rs:942-946).  Point 320 has level 1 and sits in the middle of the default batch
    [311, 330): points 311..319 must skip layer 1, points 320..329 search it.  The entry point's layer-1 list is empty,
    so a wrong mask changes no list the engine keeps; it shows in the counters."""
    n, d, efc = 1200, 24, 100
    X = data(np.float32, "DistL2", n, d, 44)
    lv = np.zeros(n, np.int32)
    lv[0], lv[320] = 2, 1
    lv[600:] = promoting_levels(po, n - 600, 45).clip(0, 2)
    sched = engine_batches(0, -1, lv)
    starts = np.cumsum([0] + sched)
    assert 311 in starts and 330 in starts and 320 not in starts
    o = make_oracle(po, np.float32, "DistL2", d, M, efc, n)
    h = make_engine(pkg, np.float32, "DistL2", M, efc, n)
    insert_both(pkg, h, o, X, lv, State(), ledger=LEDGER)
    assert_same_graph(h, o, n)
    DONE.append("masks")


# ---------------------------------------------------------------- partitions
@pytest.mark.parametrize("P", [2, 3])
def test_partitions_on_one_device(pkg, po, P):
    """partitions build concurrently, each on its own schedule; partition p holds the points p, p + P, ..."""
    n, d, efc = 3000, 24, 100
    X = data(np.float32, "DistL2", n, d, 46 + P)
    lv = promoting_levels(po, n, 46 + P)
    h = make_engine(pkg, np.float32, "DistL2", M, efc, n)
    h.partition([0] * P)
    h.enable_stats(True)
    h.get_stats()
    h.insert_flat(X, levels=lv)
    LEDGER.add(pkg.last_kernel())
    cg = h.get_stats()
    h.enable_stats(False)
    tot = {"expansions": 0, "adj_read": 0}
    for p in range(P):
        Xp, lp = X[p::P], lv[p::P]
        o = make_oracle(po, np.float32, "DistL2", d, M, efc, len(Xp))
        o.insert_batched(Xp, ids=np.arange(p, n, P), levels=lp, batches=engine_batches(0, -1, lp), nthreads=NTH)
        c = o.counters()
        for key in tot:
            tot[key] += c[key]
        assert_same_graph(h.partition_view(p), o, len(Xp))
    for key in tot:
        assert cg[key] == tot[key], (key, cg, tot)
    DONE.append(f"partitions-{P}")


# ---------------------------------------------------------------- row pointers
def test_row_pointer_upload_crosses_staging_chunk(pkg):
    """parallel_insert stages rows through an 8 MB pinned buffer (16 384 rows of 512 bytes); 20 000 rows cross it.  The
    graph must equal insert_flat's on an identically created handle, levels drawn by each handle's own RNG."""
    n, d = 20000, 128
    X = pkg.datagen.clustered(n, d, 7)
    a, b = pkg.Hnsw(16, n, 16, 100, "DistL2"), pkg.Hnsw(16, n, 16, 100, "DistL2")
    a.parallel_insert([(X[i], 5 * i) for i in range(n)])
    LEDGER.add(pkg.last_kernel())
    b.insert_flat(X, ids=5 * np.arange(n))
    pa, pb = a.export_points(), b.export_points()
    for x, y in zip(pa, pb):
        assert np.array_equal(x, y)
    for layer in range(int(pa[0].max()) + 1):
        for x, y in zip(a.export_layer(layer), b.export_layer(layer)):
            assert np.array_equal(x.view(np.uint32) if x.dtype == np.float32 else x,
                                  y.view(np.uint32) if y.dtype == np.float32 else y), layer
    DONE.append("rows")


# ---------------------------------------------------------------- full size
def test_c2_full_size_equals_batched_oracle(pkg, po):
    """bench.py's c2 graph (1 000 000 x 128 clustered f32 L2, M = 16, ef_construction = 200, default batching, levels
    drawn by the handle) against the oracle's batch-synchronous build from the same levels: layer 0 as whole arrays
    (offsets, ids, distance bits), the upper layers list by list."""
    n, d, M16, efc = 1000000, 128, 16, 200
    X = pkg.datagen.clustered(n, d, 1)
    h = pkg.Hnsw(M16, n, 16, efc, "DistL2")
    h.insert_flat(X)
    lv, rk, og, entry = h.export_points()
    o = make_oracle(po, np.float32, "DistL2", d, M16, efc, n)
    t = time.time()
    o.insert_batched(X, levels=lv, batches=engine_batches(0, -1, lv), nthreads=NTH)
    print(f"\nc2 batch-synchronous oracle build: {time.time() - t:.0f} s on {NTH} CPU threads")
    olv, ork, oog = o.export_points()
    assert entry == o.entry
    assert np.array_equal(lv, olv) and np.array_equal(rk, ork) and np.array_equal(og, oog)
    goff, gids, gds = h.export_layer(0)
    ooff, oids, ods = o.export_layer(0)
    assert np.array_equal(goff, ooff), "layer-0 offsets differ"
    assert np.array_equal(gids, oids), "layer-0 ids differ"
    assert np.array_equal(gds.view(np.uint32), ods.view(np.uint32)), "layer-0 link distances differ"
    for layer in range(1, int(lv.max()) + 1):
        goff, gids, _ = h.export_layer(layer)
        ooff, oids, _ = o.export_layer(layer)
        # every list the engine stores, and every list of a point of this level (assert_same_graph's rule)
        for p in np.nonzero((lv >= layer) | (np.diff(goff.astype(np.int64)) > 0))[0].tolist():
            assert gids[goff[p]:goff[p + 1]].tolist() == oids[ooff[p]:ooff[p + 1]].tolist(), (layer, p)
    DONE.append("c2")


# ---------------------------------------------------------------- the mini-ledger
# instantiations exempt from bit equality in test_gpu_matrix (device logf against std::log), by their op's mangled name
EXEMPT = {"10OpJeffreysE": "DistJeffreys", "4OpJSE": "DistJensenShannon"}


def test_zz_every_insert_kernel_ran_batched(pkg):
    expected = len(MATRIX) + len(STALE_CASES) + 4 + 2 + 2 + 1 + 1 + 1 + 1 + 2 + 1 + 1
    if len(DONE) != expected:
        pytest.fail(f"the ledger needs every case of this module to pass: {len(DONE)} of {expected} did")
    assert set(EXEMPT.values()) == set(LOG_METRICS)
    exe = cuobjdump()
    if exe is None:
        pytest.fail("cuobjdump (CUDA toolkit) not found: the compiled kernel list cannot be read")
    out = subprocess.run([exe, "-symbols", pkg.lib_path()], capture_output=True, text=True, check=True).stdout
    compiled = {s for s in re.findall(r"STO_ENTRY\s+(\S+)", out) if "insert_search_kernel" in s}
    exempt = {s for s in compiled if any(k in s for k in EXEMPT)}
    assert len(exempt) == len(EXEMPT), sorted(exempt)
    ran = {s for s in LEDGER if "insert_search_kernel" in s}
    assert ran <= compiled, sorted(ran - compiled)
    missed = sorted(compiled - ran - exempt)
    print(f"\ninsert ledger: {len(ran)} of {len(compiled)} insert_search_kernel entry points ran batched and bit-exact; "
          f"exempt ({', '.join(sorted(EXEMPT.values()))}, not bit-exact in test_gpu_matrix): {len(exempt)}; "
          f"module wall time {time.time() - T0:.0f} s")
    assert not missed, f"{len(missed)} insert kernels never ran batched:\n" + "\n".join(missed)

"""The graph search and insert kernels at every CTA shape their host side can choose, against the oracle and float64.

Four warp kernels run one query or insert per warp: search_kernel (search.cu), search_filter_kernel (filter.cu) and
search_std_kernel (search_std.cu) with up to 8 warps per CTA, insert_search_kernel (build.cu) with up to 4.  cta_shape
(kernels.h) halves the warps until one CTA's shared memory fits SMEM_BUDGET, and with fewer warps each kernel finds its
slot and its shared memory from the launch's own width while the host sizes the grid, the visited pool and the filtered
candidate buffer from it.  Those shapes arise only with wide rows or a large ef / ef_construction, so this module restates
the host's choice (stage_bytes, the per-warp layouts, the queue kinds, cta_shape) and for every launch:
  * checks that the kernel was of the expected family, with warps x 32 threads and warps x the layout's bytes;
  * compares every answer with the oracle (ids, distance bits, PointIds, counts, and the traversal counters with stats
    on), and with float64 (exactref.F64): each returned distance within its bound and, where the search is
    exhaustive (fewer points than ef), no returned point beyond the float64 k-th nearest plus both bounds;
  * compares every GPU build with the oracle's: serial with its MODE_DET build, batched with its batch-synchronous one.
It also checks the largest ef / ef_construction / dimension that one warp fits, the refusal one step past it, and
dist_batch (aux.cu), which sizes its CTAs with the same cta_shape, at its own shapes and its own limit.  Each launch adds (family, warps, staged) to a ledger;
test_zz_every_cta_shape_was_reached fails when a shape the host can choose was never launched."""
import time

import numpy as np
import pytest
import scipy.sparse
import scipy.sparse.csgraph

from answers import same
from exactref import F64, check_f64, d4_of
from graphs import State, assert_same_graph, data, insert_both, make_engine, make_oracle
from util import oracle_layers

pytestmark = pytest.mark.gpu

T0 = time.time()
LEDGER = set()   # (family, warps, staged) of every launch
LOG = []         # one line per launch
DONE = []        # cases that ran to the end
NTH = 8          # oracle threads

# ---------------------------------------------------------------- the host's shape choices, restated
SMEM_BUDGET = 220 * 1024   # kernels.h
STAGE_ROWS = 8             # common.cuh
MAX_WARPS = {"generic": 8, "filtered": 8, "std": 8, "insert": 4, "dist": 8}   # SEARCH_THREADS / 32, BUILD_THREADS / 32
KERNEL = {"generic": "search_kernel", "filtered": "search_filter_kernel", "std": "search_std_kernel",
          "insert": "insert_search_kernel", "dist": "dist_batch_kernel"}
COMMON = ("DistL1", "DistL2", "DistDot", "DistCosine")


def round128(b):
    return (b + 127) // 128 * 128


def stage_bytes(d4):
    """kernels.h stage_bytes: rows of up to 512 bytes are staged by TMA, STAGE_ROWS of them per warp"""
    return STAGE_ROWS * d4 * 16 if d4 <= 32 else 0


def query_layout(d4, q_smem):
    """kernels.h query_layout(...).bytes: [stage][query][queue keys][64 chunk ids][64 chunk distances][mbarrier]"""
    return round128(stage_bytes(d4) + d4 * 16 + q_smem * 8 + 64 * 4 + 64 * 4 + 16)


def std_layout(d4, q_smem):
    """kernels.h std_layout(...).bytes: [query][W heap][32 chunk ids][32 chunk distances]"""
    return round128(d4 * 16 + q_smem * 8 + 32 * 4 + 32 * 4)


def insert_layout(d4, ef_c, deg0, q_smem):
    """kernels.h insert_layout(...).bytes: [stage][new point][selection point][queue keys][64 chunk ids][64 chunk
    distances][mbarrier][selected ids, distances, step distances: deg0 each][discarded positions, ef_c u16]"""
    return round128(stage_bytes(d4) + 2 * d4 * 16 + q_smem * 8 + 64 * 4 * 2 + 16 + 3 * deg0 * 4 + ef_c * 2)


def queue_kind(ef, metric, dtype):
    """kernels.h queue_kind: the chunked queues of 32 / 64 / 128 / 256 slots for f32 L1 / L2 / Dot / Cosine up to
    ef = 256, else the generic one (0)"""
    if np.dtype(dtype) != np.float32 or metric not in COMMON or ef > 256:
        return 0
    return 101 if ef <= 32 else 102 if ef <= 64 else 104 if ef <= 128 else 108


def queue_slots(kind, ef):
    return 32 * (kind - 100) if kind >= 100 else ef


def cta_shape(spw, max_warps):
    """kernels.h cta_shape: (warps, smem) with warps halved from max_warps until warps x spw fits; (0, 0) refused"""
    w = max_warps
    while w > 1 and spw * w > SMEM_BUDGET:
        w >>= 1
    return (w, spw * w) if spw * w <= SMEM_BUDGET else (0, 0)


def query_spw(family, d4, ef, metric, dtype):
    """shared memory per warp of a query launch (Index::search_on_ctx, query_queue_slots, query_smem_per_warp); ef is
    the launch's max(ef, k)"""
    if family == "std":
        return std_layout(d4, ef + 2)   # the W heap holds at most ef + 1 items
    kind = queue_kind(ef, metric, dtype) if family == "generic" else 0
    return query_layout(d4, queue_slots(kind, ef))


def insert_spw(d4, ef_c, M, metric, dtype):
    """Index::insert_shape: the insert kernel has no 32 / 64-slot queue and takes the 128-slot one instead"""
    kind = queue_kind(ef_c, metric, dtype)
    if kind and kind < 104:
        kind = 104
    return insert_layout(d4, ef_c, 2 * M, queue_slots(kind, ef_c))


def spw_of(family, d4, metric, dtype, ef=0, M=0):
    if family == "insert":
        return insert_spw(d4, ef, M, metric, dtype)
    if family == "dist":
        return d4 * 16 + 256   # Index::dist_batch: [query row][32 candidate ids][32 distances]
    return query_spw(family, d4, ef, metric, dtype)


def warps_of(family, d4, metric, dtype, ef=0, M=0):
    return cta_shape(spw_of(family, d4, metric, dtype, ef, M), MAX_WARPS[family])[0]


def largest(fits, lo, hi):
    """the largest x in [lo, hi] with fits(x), fits(lo) being true and fits monotone"""
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if fits(mid) else (lo, mid - 1)
    return lo


def check_launch(pkg, family, d4, metric, dtype, ef=0, M=0, what="", warps=None):
    """the launch just made ran the family's kernel at the restated shape; into the ledger.  warps: the case's own
    expectation, which must agree with the restatement"""
    spw = spw_of(family, d4, metric, dtype, ef, M)
    w, smem = cta_shape(spw, MAX_WARPS[family])
    assert w >= 1, f"{what}: the restatement refuses this launch"
    if warps is not None:
        assert w == warps, f"{what}: the restatement gives {w} warps, the case was chosen for {warps}"
    kern = pkg.last_kernel()
    name = KERNEL[family]
    assert f"2hb{len(name)}{name}I" in kern, f"{what}: the last kernel was {kern}, not {name}"
    got, threads, bps = pkg.last_kernel_shape()
    assert (got, threads) == (smem, w * 32), \
        f"{what}: {got} bytes x {threads} threads, the restatement says {smem} x {w * 32} ({w} warps of {spw} bytes)"
    LEDGER.add((family, w, d4 <= 32))
    LOG.append(f"{what}: {family} {w} warps x {spw} B, d4 {d4}, {bps} CTA/SM")


# ---------------------------------------------------------------- helpers
def oracle_graph(po, dtype, metric, X, M=8, efc=40):
    n, d = X.shape
    o = po.Oracle(M, n, 16, efc, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X, levels=o.draw_levels(n))
    return o


def imported(pkg, o, X, metric, dtype, M=8, efc=40):
    """a handle holding the oracle's serial graph (rows in insertion order, which is its internal-id order)"""
    lv, _, og = o.export_points()
    h = pkg.Hnsw(M, len(X), 16, efc, metric, dtype=dtype)
    h.import_graph(X, og, lv, o.entry, oracle_layers(o))
    return h


def ringed_graph(pkg, po, dtype, metric, X, M=8, efc=40):
    """(oracle, handle) holding the oracle's graph of X with each layer-0 list extended by the edge to the next point,
    i -> i + 1 mod n, so that layer 0 is strongly connected.  (About 3 % of a serial build's points have no layer-0
    in-link, and no search reaches them.)  Both import it with M + 1, which leaves room for the extra edge."""
    n, d = X.shape
    src = oracle_graph(po, dtype, metric, X, M, efc)
    lv, _, og = src.export_points()
    layers = oracle_layers(src)
    off, ids, ds = layers[0]
    nids, nds = [], []
    for i in range(n):
        a, b = int(off[i]), int(off[i + 1])
        nids.append(ids[a:b])
        nds.append(ds[a:b])
        j = (i + 1) % n
        if j not in ids[a:b]:
            nids.append(np.array([j], np.uint32))
            nds.append(np.array([po.dist(X[i], X[j], metric, po.ORDER_GPU)], np.float32))
    sizes = np.diff(off.astype(np.int64)) + np.array([(i + 1) % n not in ids[int(off[i]):int(off[i + 1])] for i in range(n)])
    layers[0] = (np.concatenate([[0], np.cumsum(sizes)]).astype(np.uint64), np.concatenate(nids), np.concatenate(nds))
    o = po.Oracle(M + 1, n, 16, efc, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.import_graph(X, og, lv, src.entry, dict(enumerate(layers)))
    h = pkg.Hnsw(M + 1, n, 16, efc, metric, dtype=dtype)
    h.import_graph(X, og, lv, src.entry, layers)
    layer0_reaches_all(o, n)
    return o, h


def layer0_reaches_all(o, n):
    """a BFS over the oracle's layer 0 from its entry point reaches every point, so that a search of ef > n is exhaustive"""
    off, ids, _ = o.export_layer(0)
    g = scipy.sparse.csr_matrix((np.ones(len(ids)), ids.astype(np.int64), off.astype(np.int64)), shape=(n, n))
    seen = scipy.sparse.csgraph.breadth_first_order(g, o.entry, directed=True, return_predecessors=False)
    assert len(seen) == n, f"layer 0 reaches {len(seen)} of {n} points from the entry point"


def check_dists(F, Q, got, what):
    """every returned distance within its float64 bound (F64.exact)"""
    dist, it, cnt = got[1], got[2], got[4]
    for i in range(len(Q)):
        c = int(cnt[i])
        v, b = F.exact(it[i, :c].astype(np.int64), Q[i])
        g = dist[i, :c].astype(np.float64)
        if F.metric == "DistL2":
            g = g * g
        bad = np.flatnonzero(np.abs(g - v) > b)
        assert not len(bad), f"{what}, row {i}, slot {bad[0]}: got {g[bad[0]]!r}, float64 {v[bad[0]]!r} +- {b[bad[0]]:.3g}"


def searches(pkg, po, h, o, X, Q, metric, dtype, k, ef, F=None, exhaustive=False, allow=None, what=""):
    """generic and std-tie with stats on, and filtered (sorted ids `allow`), at (k, ef): answers equal to the oracle's,
    traversal counters too, and within float64 when F is given (exhaustive: also no point beyond the true k-th)"""
    d4, n, e = d4_of(X.shape[1], dtype), len(X), max(ef, k)

    def f64(got, adm, tag):
        if F is not None and exhaustive:
            check_f64(F, Q, got, k, [adm] * len(Q), tag)
        elif F is not None:
            check_dists(F, Q, got, tag)

    for family, mode, tie in (("generic", po.MODE_DET, 0), ("std", po.MODE_STD, 1)):
        tag = f"{what} {family} k={k} ef={ef}"
        o.set_mode(mode)
        h.set_tie_mode(tie)
        o.counters()
        want = o.search_batch(Q, k, ef, nthreads=NTH)
        co = o.counters()
        h.enable_stats(True)
        h.get_stats()
        got = h.search_flat(Q, k, ef)
        check_launch(pkg, family, d4, metric, dtype, e, what=tag)
        cg = h.get_stats()
        h.enable_stats(False)
        same(got, want, tag)
        for key in ("evals", "expansions", "adj_read"):
            assert cg[key] == co[key], (tag, key, cg, co)
        f64(got, np.arange(n), tag)
    o.set_mode(po.MODE_DET)
    h.set_tie_mode(0)
    if allow is not None:
        tag = f"{what} filtered k={k} ef={ef}"
        got = h.search_flat(Q, k, ef, filter=allow)
        check_launch(pkg, "filtered", d4, metric, dtype, e, what=tag)
        same(got, o.search_batch(Q, k, ef, filter_ids=allow, nthreads=NTH), tag)
        f64(got, allow, tag)


# ---------------------------------------------------------------- staged rows, large ef
# f32 d = 24 (128-byte rows, staged by TMA): (metric, ef, n < ef, expected warps of every query family)
STAGED = [("DistL2", 4000, 3000, 4), ("DistCosine", 8000, 6000, 2), ("DistL2", 16000, 12000, 1)]


@pytest.mark.parametrize("metric,ef,n,warps", STAGED, ids=[f"{m}-ef{ef}" for m, ef, _, _ in STAGED])
def test_staged_rows_large_ef(pkg, po, metric, ef, n, warps):
    """every query family at ef > n on an oracle graph whose layer 0 reaches every point (ringed_graph): exhaustive
    searches, equal to the oracle and within float64 of the true k nearest.  At 1 warp also k = ef (every point back)
    and a batch of per-query label sets through the filtered kernel."""
    d, dtype, nq = 24, np.float32, 6
    X = data(dtype, metric, n, d, ef)
    Q = data(dtype, metric, nq, d, ef + 1)
    Q[0] = X[n // 2]
    for family in ("generic", "filtered", "std"):
        assert warps_of(family, d4_of(d, dtype), metric, dtype, ef) == warps, family
    o, h = ringed_graph(pkg, po, dtype, metric, X)
    F = F64(X, metric)
    allow = np.arange(1, n, 3)
    for k in (1, 10, 100) + ((ef,) if warps == 1 else ()):
        searches(pkg, po, h, o, X, Q, metric, dtype, k, ef, F, exhaustive=True, allow=allow, what=f"staged ef={ef}")
    if warps == 1:
        lab = np.random.default_rng(ef).integers(1, 4, n).astype(np.uint32)
        h.set_labels(0, lab)
        sets = [[1, 3] if i % 2 == 0 else [2] for i in range(nq)]
        got = h.search_flat_label_sets(Q, 10, ef, sets)
        check_launch(pkg, "filtered", d4_of(d, dtype), metric, dtype, ef, what="label sets", warps=1)
        for par, s in ((0, [1, 3]), (1, [2])):
            rows = np.arange(par, nq, 2)
            adm = np.flatnonzero(np.isin(lab, s))
            part = tuple(x[rows] for x in got)
            same(part, o.search_batch(Q[rows], 10, ef, filter_ids=adm, nthreads=NTH), f"label set {s}")
            check_f64(F, Q[rows], part, 10, [adm] * len(rows), f"label set {s}")
    DONE.append(f"staged {metric} ef{ef}")


# ---------------------------------------------------------------- wide rows
# (dtype, metric, d, n, warps of the query families at ef 32 / k <= 32); k = 100 raises ef to 100, same warps
WIDE = [(np.float32, "DistDot", 7000, 300, 4), (np.float32, "DistCosine", 14000, 300, 2),
        (np.float32, "DistL2", 40000, 250, 1),
        (np.uint8, "DistL2", 30000, 300, 4), (np.uint8, "DistJaccard", 60000, 250, 2),
        (np.uint8, "DistHamming", 120000, 200, 1),
        (np.uint16, "DistJaccard", 15000, 300, 4), (np.uint16, "DistL2", 30000, 250, 2),
        (np.uint16, "DistL2", 60000, 200, 1)]
F64_METRICS = ("DistL2", "DistCosine", "DistHamming", "DistJaccard")


def wide_id(c):
    return f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}"


@pytest.mark.parametrize("dtype,metric,d,n,warps", WIDE, ids=[wide_id(c) for c in WIDE])
def test_wide_rows(pkg, po, dtype, metric, d, n, warps):
    """every query family at k = 1, 10, 100 (ef 32) on an oracle graph of rows too wide for 8 warps, and dist_batch at
    its own shape; at 1 warp, search_by_id equal to the search on the stored rows"""
    nq, ef = 20, 32
    d4 = d4_of(d, dtype)
    for family in ("generic", "filtered", "std"):
        for e in (32, 100):
            assert warps_of(family, d4, metric, dtype, e) == warps, (family, e)
    X = data(dtype, metric, n, d, d + n)
    Q = data(dtype, metric, nq, d, d + n + 1)
    Q[:2] = X[:2]
    o = oracle_graph(po, dtype, metric, X)
    h = imported(pkg, o, X, metric, dtype)
    F = F64(X, metric) if metric in F64_METRICS else None
    allow = np.arange(1, n, 3)
    for k in (1, 10, 100):
        searches(pkg, po, h, o, X, Q, metric, dtype, k, ef, F, allow=allow if k == 10 else None, what=wide_id((dtype, metric, d)))
    cand = np.random.default_rng(d).integers(0, n, (nq, 40)).astype(np.uint32)
    got = h.dist_batch(Q, cand)
    check_launch(pkg, "dist", d4, metric, dtype, what=f"dist_batch d={d}")
    want = np.array([[po.dist(Q[i], X[j], metric, po.ORDER_GPU) for j in cand[i]] for i in range(nq)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), "dist_batch differs from ORDER_GPU"
    if warps == 1:
        qids = np.array([3, 17, n - 1], np.uint64)
        a = h.search_by_id(qids, 10, ef)
        check_launch(pkg, "generic", d4, metric, dtype, ef, what="search_by_id", warps=1)
        same(a, h.search_flat(X[qids.astype(np.int64)], 10, ef), "search_by_id against the stored rows")
    DONE.append(wide_id((dtype, metric, d)))


# ---------------------------------------------------------------- inserts
def builds(pkg, po, dtype, metric, X, M, efc, warps, extend=False, keep_pruned=False, what=""):
    """a serial GPU build equal to the oracle's MODE_DET build, and a build on the default batched schedule equal to the
    batch-synchronous oracle (with its insert counters); searches on the serial graph equal the oracle's"""
    n, d = X.shape
    d4 = d4_of(d, dtype)
    assert warps_of("insert", d4, metric, dtype, efc, M) == warps
    o = make_oracle(po, dtype, metric, d, M, efc, n, extend, keep_pruned)
    levels = o.draw_levels(n)
    o.insert_batch(X, levels=levels)
    h = make_engine(pkg, dtype, metric, M, efc, n, (1 << 30, 1), extend, keep_pruned)
    h.insert_flat(X, levels=levels)
    check_launch(pkg, "insert", d4, metric, dtype, efc, M, what=f"{what} serial", warps=warps)
    assert_same_graph(h, o, n)
    ob = make_oracle(po, dtype, metric, d, M, efc, n, extend, keep_pruned)
    hb = make_engine(pkg, dtype, metric, M, efc, n, None, extend, keep_pruned)
    insert_both(pkg, hb, ob, X, levels, State())
    check_launch(pkg, "insert", d4, metric, dtype, efc, M, what=f"{what} batched", warps=warps)
    assert_same_graph(hb, ob, n)
    hb.close()
    return o, h


# (dtype, metric, d, n, M, ef_construction, extend + keep_pruned, expected warps)
INSERTS = [(np.float32, "DistL2", 24, 1500, 8, 8000, False, 2), (np.float32, "DistCosine", 24, 1500, 8, 12000, False, 1),
           (np.float32, "DistL2", 24, 3000, 8, 12000, True, 1), (np.float32, "DistL2", 24, 1500, 256, 6000, False, 2),
           (np.float32, "DistL2", 14000, 300, 8, 40, False, 1), (np.uint8, "DistL2", 60000, 200, 8, 40, False, 1)]


def insert_id(c):
    return f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}-M{c[4]}-efc{c[5]}" + ("-ext-kp" if c[6] else "")


@pytest.mark.parametrize("dtype,metric,d,n,M,efc,ext,warps", INSERTS, ids=[insert_id(c) for c in INSERTS])
def test_insert_shapes(pkg, po, dtype, metric, d, n, M, efc, ext, warps):
    X = data(dtype, metric, n, d, d + efc)
    o, h = builds(pkg, po, dtype, metric, X, M, efc, warps, ext, ext, insert_id((dtype, metric, d, n, M, efc, ext)))
    Q = data(dtype, metric, 20, d, d + efc + 1)
    same(h.search_flat(Q, 10, 48), o.search_batch(Q, 10, 48, nthreads=NTH), "search on the serial graph")
    DONE.append(insert_id((dtype, metric, d, n, M, efc, ext)))


def test_very_wide_rows_run_with_fewer_warps_per_block(pkg, po):
    """d = 7000 f32 (28 KB per row): 8 warps' worth of query rows no longer fit one block's shared memory; the kernels
    run fewer warps per block instead of failing (the search 4, the insert 2), and the answers still equal the oracle's"""
    n, d = 400, 7000
    X = pkg.datagen.uniform(n, d, 1)
    o, h = builds(pkg, po, np.float32, "DistL2", X, 8, 40, 2, what="d=7000")
    Q = pkg.datagen.uniform(40, d, 2)
    got = h.search_flat(Q, 5, 32)
    check_launch(pkg, "generic", d4_of(d, np.float32), "DistL2", np.float32, 32, what="d=7000 search", warps=4)
    same(got, o.search_batch(Q, 5, 32), "d=7000 search")
    assert pkg.load_library().hnsw_b200_get_extend_candidates(h._h) == 0
    DONE.append("very wide rows")


# ---------------------------------------------------------------- the single-warp limits
def test_largest_ef_and_refusal(pkg, po):
    """at d = 24 f32: the largest ef one warp fits answers as the oracle does, for the generic, filtered and std-tie
    kernels and for search_by_id with exclude_self (which searches knbn + 1); one ef more is refused before any launch,
    and the handle answers as before"""
    n, d, dtype, metric, nq = 3000, 24, np.float32, "DistL2", 3
    d4 = d4_of(d, dtype)
    X = data(dtype, metric, n, d, 71)
    Q = data(dtype, metric, nq, d, 72)
    o, h = ringed_graph(pkg, po, dtype, metric, X)
    F = F64(X, metric)
    limit = {f: largest(lambda e: warps_of(f, d4, metric, dtype, e) >= 1, 300, 1 << 20) for f in ("generic", "filtered", "std")}
    LOG.append(f"largest ef at d = 24 f32: {limit}")
    for f, e in limit.items():
        assert query_spw(f, d4, e + 1, metric, dtype) > SMEM_BUDGET >= query_spw(f, d4, e, metric, dtype)
    allow = np.arange(0, n, 2)
    for family, e in limit.items():
        tag = f"largest ef {e} {family}"
        if family == "std":
            o.set_mode(po.MODE_STD)
            h.set_tie_mode(1)
        filt = allow if family == "filtered" else None
        want = o.search_batch(Q, 10, e, filter_ids=filt, nthreads=NTH)
        got = h.search_flat(Q, 10, e, filter=filt)
        check_launch(pkg, family, d4, metric, dtype, e, what=tag, warps=1)
        same(got, want, tag)
        check_f64(F, Q, got, 10, [allow if filt is not None else np.arange(n)] * nq, tag)
        with pytest.raises(pkg.HnswError, match="ef / dimension too large"):
            h.search_flat(Q, 10, e + 1, filter=filt)
        assert "ef / dimension too large" in pkg.last_error()
        same(h.search_flat(Q, 10, e, filter=filt), got, f"{tag}, after the refused call")
        if family == "std":
            h.set_tie_mode(0)
            o.set_mode(po.MODE_DET)
    # search_by_id with exclude_self: knbn = e - 1 searches e and runs, knbn = e is refused
    e = limit["generic"]
    qids = np.array([5, 1000, n - 1], np.uint64)
    got = h.search_by_id(qids, e - 1, e, exclude_self=True)
    check_launch(pkg, "generic", d4, metric, dtype, e, what="by id, exclude_self", warps=1)
    full = h.search_flat(X[qids.astype(np.int64)], e, e)
    for i, q in enumerate(qids.tolist()):
        keep = np.flatnonzero(full[2][i, :full[4][i]] != q)[:e - 1]   # the row without the point itself, cut to knbn
        c = int(got[4][i])
        assert c == len(keep) == min(e - 1, n - 1), (i, c, len(keep))
        assert np.array_equal(got[2][i, :c], full[2][i, keep]), f"by id row {i}: ids"
        assert np.array_equal(got[1][i, :c].view(np.uint32), full[1][i, keep].view(np.uint32)), f"by id row {i}: dists"
    with pytest.raises(pkg.HnswError, match=r"exclude_self searches knbn \+ 1: ef / dimension too large"):
        h.search_by_id(qids, e, e, exclude_self=True)
    same(h.search_by_id(qids, e - 1, e, exclude_self=True), got, "by id after the refused call")
    DONE.append("largest ef")


def refused_insert(pkg, po, dtype, metric, X, M, efc, what):
    """a handle holding an imported graph refuses an insert at (X's dimension, efc) before anything changes"""
    n, d = X.shape
    o = oracle_graph(po, dtype, metric, X, M, efc)
    h = imported(pkg, o, X, metric, dtype, M, efc)
    Q = X[:4].copy()
    before = h.search_flat(Q, 5, 16)
    with pytest.raises(pkg.HnswError, match="ef_construction / dimension too large"):
        h.insert_flat(X[:3], ids=np.arange(n, n + 3))
    assert "ef_construction / dimension too large" in pkg.last_error(), what
    assert h.get_nb_point() == n, what
    same(h.search_flat(Q, 5, 16), before, f"{what}: after the refused insert")
    same(before, o.search_batch(Q, 5, 16), f"{what}: the imported graph")


def test_largest_ef_construction_and_dimension(pkg, po):
    """the largest ef_construction one insert warp fits at d = 24 f32 (M = 8), and the largest f32 dimension at
    ef_construction 40, build as the oracle does; one step past either is refused before the index changes"""
    M, metric, dtype = 8, "DistL2", np.float32
    d4 = d4_of(24, dtype)
    efc = largest(lambda e: warps_of("insert", d4, metric, dtype, e, M) >= 1, 300, 1 << 20)
    assert insert_spw(d4, efc + 1, M, metric, dtype) > SMEM_BUDGET
    X = data(dtype, metric, 1200, 24, 81)
    builds(pkg, po, dtype, metric, X, M, efc, 1, what=f"largest ef_construction {efc}")
    refused_insert(pkg, po, dtype, metric, X[:300], M, efc + 1, f"ef_construction {efc + 1}")
    dmax = largest(lambda dd: warps_of("insert", d4_of(dd, dtype), metric, dtype, 40, M) >= 1, 24, 1 << 20)
    LOG.append(f"largest insert ef_construction at d = 24 f32, M = 8: {efc}; largest f32 dimension at 40: {dmax}")
    assert warps_of("generic", d4_of(dmax + 1, dtype), metric, dtype, 16) >= 1   # search still runs past the insert limit
    Xd = data(dtype, metric, 60, dmax + 1, 82)
    builds(pkg, po, dtype, metric, Xd[:, :dmax].copy(), M, 40, 1, what=f"largest dimension {dmax}")
    refused_insert(pkg, po, dtype, metric, Xd, M, 40, f"dimension {dmax + 1}")
    DONE.append("largest ef_construction and dimension")


def test_dist_batch_widest_row_and_refusal(pkg, po):
    """the widest f32 row one dist_batch warp fits answers as ORDER_GPU does; one 128-byte line more is refused before
    any launch"""
    dtype, metric, n = np.float32, "DistL2", 4
    dmax = largest(lambda dd: warps_of("dist", d4_of(dd, dtype), metric, dtype) >= 1, 1, 1 << 20)
    cand = np.array([[0, 1, 2, 3], [3, 2, 1, 0]], np.uint32)
    for d in (dmax, dmax + 1):
        X = data(dtype, metric, n, d, d)
        h = pkg.Hnsw(8, n, 16, 40, metric)
        h.import_graph(X, np.arange(n, dtype=np.uint64), np.zeros(n, np.uint8), 0,
                       [(np.zeros(n + 1, np.uint64), np.zeros(0, np.uint32), None)])
        if d == dmax:
            got = h.dist_batch(X[:2], cand)
            check_launch(pkg, "dist", d4_of(d, dtype), metric, dtype, what=f"dist_batch d={d}", warps=1)
            want = np.array([[po.dist(X[i], X[j], metric, po.ORDER_GPU) for j in cand[i]] for i in range(2)], np.float32)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), "dist_batch differs from ORDER_GPU"
        else:
            with pytest.raises(pkg.HnswError, match="dimension too large for dist_batch"):
                h.dist_batch(X[:2], cand)
        h.close()
    DONE.append("dist_batch limit")


# ---------------------------------------------------------------- the ledger
def test_zz_every_cta_shape_was_reached():
    want = len(STAGED) + len(WIDE) + len(INSERTS) + 1 + 1 + 1 + 1
    if len(DONE) != want:
        pytest.fail(f"the shape ledger needs every case of this module to pass: {len(DONE)} of {want} did")
    print("\nCTA shapes (family, warps, staged):\n" + "\n".join(map(str, sorted(LEDGER))))
    print("\n".join(LOG))
    print(f"module wall time {time.time() - T0:.0f} s")
    need = [(f, w, s) for f in ("generic", "filtered", "std") for w in (4, 2, 1) for s in (True, False)]
    need += [("insert", w, s) for w in (2, 1) for s in (True, False)]
    need += [("dist", w, False) for w in (4, 2, 1)]
    missing = [x for x in need if x not in LEDGER]
    assert not missing, "shapes never launched: " + ", ".join(map(str, missing))

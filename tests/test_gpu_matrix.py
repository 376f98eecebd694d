"""The kernel instantiation matrix, bit-exact against the oracle, with a ledger of the kernels it reached.

Each query, insert and aux kernel is a template over (distance op, compile-time row chunks CH, queue size, stats on/off),
and the host picks one instantiation per call.  This module builds one graph per (element type, metric, dimension,
ef_construction) twice, serially on the GPU and in the oracle (MODE_DET, ORDER_GPU), asserts that the graphs are equal,
and then runs every query kernel on it at the shapes where a template goes wrong: ef at the queue-size boundaries
(1, k, 64/65, 128/129, 256/257), k beyond one warp (40, 128), rows of 128 / 256 / 512 / more bytes, stats on and off,
filtered, std-tie, dist_batch and bruteforce.  Ids, distance bits, PointIds, counts and traversal counters must equal the
oracle's.

Every call records hnsw_b200_last_kernel().  test_zz_every_compiled_kernel_was_reached compares that set with the entry
points `cuobjdump -symbols` lists for the loaded library and names every compiled kernel no case reached.

It also covers the visited tables' two rare paths (overflow then grow and re-run; epoch wrap-around with its table clear)
and checks the device's dist_batch against the float64 formulas of tests/distref.py at every row-chunk size.
"""
import os
import re
import shutil
import subprocess
import time

import numpy as np
import pytest

import distref
from util import csr_lists, oracle_layers, recall_ids

pytestmark = pytest.mark.gpu

T0 = time.time()
LEDGER = set()   # mangled names of the kernels the cases launched
DONE = []        # ids of the cases that ran to the end


def launched(pkg, result=None):
    LEDGER.add(pkg.last_kernel())
    return result


def same(got, want, what):
    go, gd, gi, gpid, gc = got
    oo, od, oi, opid, oc = want
    assert np.array_equal(gc, oc), f"{what}: counts differ"
    assert np.array_equal(gi, oi), f"{what}: internal ids differ"
    assert np.array_equal(go, oo), f"{what}: origin ids differ"
    assert np.array_equal(gd.view(np.uint32), od.view(np.uint32)), f"{what}: distances are not bit-identical"
    assert np.array_equal(gpid, opid), f"{what}: PointIds differ"


def assert_same_graph(h, o, n):
    lv, rk, og, entry = h.export_points()
    olv, ork, oog = o.export_points()
    assert entry == o.entry
    assert np.array_equal(lv, olv) and np.array_equal(rk, ork) and np.array_equal(og, oog)
    for layer in range(0, int(olv.max()) + 1):
        goff, gids, gds = h.export_layer(layer)
        ooff, oids, ods = o.export_layer(layer)
        if layer == 0:
            assert np.array_equal(goff, ooff) and np.array_equal(gids, oids), "layer 0 differs"
            assert np.array_equal(gds.view(np.uint32), ods.view(np.uint32)), "layer-0 link distances differ"
            continue
        gl, ol = csr_lists(goff, gids), csr_lists(ooff, oids)
        for p in range(n):
            if not gl[p] and olv[p] < layer:   # a list no search can reach, which the engine does not store
                continue
            assert gl[p] == ol[p], (layer, p, gl[p], ol[p])


def data(dtype, metric, n, d, seed, ties=False):
    rng = np.random.default_rng(seed)
    dt = np.dtype(dtype)
    if dt == np.float32:
        kind = "unit" if metric == "DistDot" else "uniform"
        import importlib
        dg = importlib.import_module("hnswlib-rs_b200").datagen
        if ties:   # every vector stored 4 times: the kernels must order equal distances by id
            base = dg.make(kind, (n + 3) // 4, d, seed)
            return np.repeat(base, 4, axis=0)[:n].copy()
        return dg.make(kind, n, d, seed)
    hi = {"DistHamming": 3, "DistJaccard": 16 if dt == np.uint8 else 1000}.get(metric)
    if hi is None:
        hi = {np.dtype(np.uint8): 256, np.dtype(np.uint16): 5000, np.dtype(np.uint32): 100000}.get(dt, 2000)
    lo = -hi if dt == np.int32 and metric != "DistHamming" else 0
    return rng.integers(lo, hi, (n, d)).astype(dt)


def build_both(pkg, po, dtype, metric, n, d, M, efc, seed, ties=False, max_elements=None):
    X = data(dtype, metric, n, d, seed, ties)
    o = po.Oracle(M, n, 16, efc, metric, d, dtype=dtype, mode=po.MODE_DET, order=po.ORDER_GPU)
    levels = o.draw_levels(n)
    o.insert_batch(X, levels=levels)
    h = pkg.Hnsw(M, max_elements or n, 16, efc, metric, dtype=dtype)
    h.set_insert_batching(1 << 30, 1)   # one insert in flight: a deterministic serial build
    launched(pkg, h.insert_flat(X, levels=levels))
    assert_same_graph(h, o, n)
    return X, o, h


def queries(X, dtype, metric, nq, seed):
    Q = data(dtype, metric, nq, X.shape[1], seed + 100)
    Q[: nq // 10] = X[: nq // 10]   # stored points: distance-0 answers
    return Q


# ---------------------------------------------------------------- the matrix
F32_OPS = ["DistL1", "DistL2", "DistDot", "DistCosine"]
F32_DIMS = [24, 48, 100, 150]          # rows of 128 / 256 / 512 / 640 bytes: CH = 1, 2, 4, generic
U8_DIMS = [100, 200, 400, 600]
U16_DIMS = [50, 100, 200, 300]
CASES = ([(np.float32, m, d, False) for m in F32_OPS for d in F32_DIMS]
         + [(np.float32, "DistL2", 24, True), (np.float32, "DistCosine", 100, True)]
         + [(np.uint8, m, d, False) for m in distref.INT_METRICS for d in U8_DIMS]
         + [(np.uint16, m, d, False) for m in distref.INT_METRICS for d in U16_DIMS]
         + [(np.uint32, m, 24, False) for m in distref.INT_METRICS]
         + [(np.int32, m, 24, False) for m in ("DistL1", "DistL2", "DistHamming")])
N, NQ, M = 1000, 100, 8
KS = [1, 10, 40, 128]
EFS = [1, 64, 65, 128, 129, 256, 257]


def k_ef_pairs():
    """(k, ef) with ef in EFS or k - 1 (which the search raises to k), ef >= k - 1; 25 pairs"""
    return sorted({(k, max(ef, k)) for k in KS for ef in EFS + [k - 1] if ef >= k - 1})


def case_id(c):
    return f"{np.dtype(c[0]).name}-{c[1]}-d{c[2]}" + ("-ties" if c[3] else "")


@pytest.mark.parametrize("dtype,metric,d,ties", CASES, ids=[case_id(c) for c in CASES])
def test_instantiation_matrix(pkg, po, dtype, metric, d, ties):
    X, o, h = build_both(pkg, po, dtype, metric, N, d, M, 200 if np.dtype(dtype) == np.float32 else 48, seed=d + 7, ties=ties)
    Q = queries(X, dtype, metric, NQ, d)
    # unfiltered search, stats off and on: same answers, and with stats the oracle's traversal counters
    for k, ef in k_ef_pairs():
        o.counters()
        want = o.search_batch(Q, k, ef)
        co = o.counters()
        h.enable_stats(False)
        same(launched(pkg, h.search_flat(Q, k, ef)), want, f"k={k} ef={ef}")
        h.enable_stats(True)
        h.get_stats()
        same(launched(pkg, h.search_flat(Q, k, ef)), want, f"k={k} ef={ef} stats")
        cg = h.get_stats()
        for key in ("evals", "expansions", "adj_read"):
            assert cg[key] == co[key], (k, ef, key, cg, co)
    h.enable_stats(False)
    # filtered search (sorted id list) at three ef values; at ef = k = 5 the result list is full early, so ties with its
    # farthest entry meet the accept rule
    allow = np.arange(1, N, 3)
    for k, ef in ((5, 5), (10, 24), (10, 150)):
        want = o.search_batch(Q, k, ef, filter_ids=allow)
        same(launched(pkg, h.search_flat(Q, k, ef, filter=allow)), want, f"filtered k={k} ef={ef}")
    # std-tie mode against the oracle's literal-reference heaps on the same graph
    o.set_mode(po.MODE_STD)
    h.set_tie_mode(1)
    for k, ef in ((10, 32), (40, 160)):
        o.counters()
        want = o.search_batch(Q, k, ef)
        co = o.counters()
        h.enable_stats(True)
        h.get_stats()
        same(launched(pkg, h.search_flat(Q, k, ef)), want, f"std-tie k={k} ef={ef}")
        cg = h.get_stats()
        for key in ("evals", "expansions", "adj_read"):
            assert cg[key] == co[key], ("std-tie", k, ef, key, cg, co)
    h.enable_stats(False)
    h.set_tie_mode(0)
    o.set_mode(po.MODE_DET)
    # dist_batch and bruteforce against the oracle's ORDER_GPU sums, bit for bit
    cand = np.random.default_rng(d).integers(0, N, (NQ, 40)).astype(np.uint32)
    got = launched(pkg, h.dist_batch(Q, cand))
    want = np.array([[po.dist(Q[i], X[j], metric, po.ORDER_GPU) for j in cand[i]] for i in range(NQ)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), "dist_batch differs from ORDER_GPU"
    bi, bd = launched(pkg, h.bruteforce(Q, 10))
    ti, td = po.bruteforce(X, Q, 10, metric, po.ORDER_GPU)
    assert np.array_equal(bi, ti) and np.array_equal(bd.view(np.uint32), td.view(np.uint32)), "bruteforce differs"
    DONE.append(case_id((dtype, metric, d, ties)))


INSERT_CASES = [(m, d, efc) for m in F32_OPS for d in F32_DIMS for efc in (48, 300)]


@pytest.mark.parametrize("metric,d,efc", INSERT_CASES)
def test_insert_queue_kinds(pkg, po, metric, d, efc):
    """the f32 insert kernel's other queues: 128 slots (ef_construction <= 128) and the generic one (> 256); the
    256-slot queue (129..256) builds the graphs of test_instantiation_matrix"""
    X, o, h = build_both(pkg, po, np.float32, metric, 600, d, M, efc, seed=d + efc)
    Q = queries(X, np.float32, metric, 50, d + 1)
    same(launched(pkg, h.search_flat(Q, 10, 300)), o.search_batch(Q, 10, 300), "search")
    DONE.append(f"insert-{metric}-{d}-{efc}")


PROB = ["DistHellinger", "DistJeffreys", "DistJensenShannon"]


@pytest.mark.parametrize("metric", PROB)
def test_probability_metric_kernels(pkg, po, metric):
    """Hellinger / Jeffreys / Jensen-Shannon: the device's logf and the oracle's std::log differ in the last bit, so the
    bar is 1e-5 relative on distances and >= 99 % identical ids, on a graph the oracle built; the GPU-built graph must
    reach the recall of the oracle-built one within 0.02"""
    n, d = 1500, 32
    rng = np.random.default_rng(5)
    X = rng.random((n, d), dtype=np.float32) + np.float32(1e-3)
    X /= X.sum(1, keepdims=True)
    Q = rng.random((200, d), dtype=np.float32) + np.float32(1e-3)
    Q /= Q.sum(1, keepdims=True)
    o = po.Oracle(M, n, 16, 80, metric, d, mode=po.MODE_DET, order=po.ORDER_GPU)
    levels = o.draw_levels(n)
    o.insert_batch(X, levels=levels)
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, n, 16, 80, metric)
    h.import_graph(X, og, lv, o.entry, oracle_layers(o))

    def close(got, want, what):
        same_ids = got[2] == want[2]
        assert same_ids.mean() >= 0.99, (what, same_ids.mean())
        assert np.allclose(got[1][same_ids], want[1][same_ids], rtol=1e-5, atol=1e-7), what

    close(launched(pkg, h.search_flat(Q, 10, 48)), o.search_batch(Q, 10, 48), "generic")
    close(launched(pkg, h.search_flat(Q, 10, 300)), o.search_batch(Q, 10, 300), "generic ef 300")
    allow = np.arange(0, n, 2)
    close(launched(pkg, h.search_flat(Q, 10, 48, filter=allow)), o.search_batch(Q, 10, 48, filter_ids=allow), "filtered")
    o.set_mode(po.MODE_STD)
    h.set_tie_mode(1)
    close(launched(pkg, h.search_flat(Q, 10, 48)), o.search_batch(Q, 10, 48), "std-tie")
    h.set_tie_mode(0)
    cand = rng.integers(0, n, (200, 20)).astype(np.uint32)
    got = launched(pkg, h.dist_batch(Q, cand))
    want = np.array([[po.dist(Q[i], X[j], metric, po.ORDER_GPU) for j in cand[i]] for i in range(200)], np.float32)
    assert np.allclose(got, want, rtol=1e-5, atol=1e-7)
    bi, bd = launched(pkg, h.bruteforce(Q, 10))
    ti, td = po.bruteforce(X, Q, 10, metric, po.ORDER_GPU)
    assert (bi == ti).mean() >= 0.99 and np.allclose(bd, td, rtol=1e-5, atol=1e-7)
    h2 = pkg.Hnsw(M, n, 16, 80, metric)
    launched(pkg, h2.insert_flat(X, levels=levels))
    ti, _ = po.bruteforce(X, Q, 10, metric)
    g = h2.search_flat(Q, 10, 48)
    w = o.search_batch(Q, 10, 48)
    assert recall_ids(g[2], g[4], ti) >= recall_ids(w[2], w[4], ti) - 0.02
    DONE.append(f"prob-{metric}")


# ---------------------------------------------------------------- distances against the float64 formulas
GPU_DIMS = [1, 3, 15, 17, 33, 100, 129, 257]    # f32 rows of 128 (CH 1), 256, 512 (CH 4) and more bytes
LOG_METRICS = ("DistJeffreys", "DistJensenShannon")
DIST_CASES = [(dt, m) for dt in (np.float32, np.uint8, np.uint16, np.uint32, np.int32)
              for m in distref.F32_METRICS + ["DistHamming", "DistJaccard"] if distref.supported(dt, m)]


@pytest.mark.parametrize("dtype,metric", DIST_CASES, ids=[f"{np.dtype(a).name}-{b}" for a, b in DIST_CASES])
def test_dist_batch_matches_float64_formula(pkg, po, dtype, metric):
    """the GPU twin of tests/test_distances_cpu.py: h.dist_batch on the edge inputs at every row-chunk size, within the
    stated forward-error bound of the float64 formula, exactly 0 where the formula is, and bit-equal to ORDER_GPU (within
    1e-5 relative for Jeffreys and Jensen-Shannon, whose device logf and the oracle's std::log may differ in the last bit)"""
    for d in GPU_DIMS:
        pairs = distref.edge_pairs(dtype, metric, d)
        A = np.stack([a for _, a, _ in pairs] + [b for _, _, b in pairs])
        B = np.stack([b for _, _, b in pairs] + [a for _, a, _ in pairs])
        n = len(B)
        h = pkg.Hnsw(M, n, 16, 48, metric, dtype=dtype)
        h.import_graph(B, np.arange(n, dtype=np.uint64), np.zeros(n, np.uint8), 0,
                       [(np.zeros(n + 1, np.uint64), np.zeros(0, np.uint32), None)])
        got = launched(pkg, h.dist_batch(A, np.arange(n, dtype=np.uint32)[:, None]))[:, 0]
        names = [p[0] for p in pairs] * 2
        for i in range(n):
            ok, msg = distref.within(got[i], metric, A[i], B[i])
            assert ok, f"{names[i]}: {msg}"
            if (metric, names[i]) in distref.EXACT_ZERO:
                assert got[i] == 0.0, (names[i], metric, d, got[i])
            ref = np.float32(po.dist(A[i], B[i], metric, po.ORDER_GPU))
            if metric in LOG_METRICS:
                assert abs(got[i] - ref) <= 1e-5 * abs(ref) + 1e-7, (names[i], metric, d, got[i], ref)
            else:
                assert got[i].view(np.uint32) == ref.view(np.uint32), (names[i], metric, d, got[i], ref)
        h.close()
    DONE.append(f"dist-{np.dtype(dtype).name}-{metric}")


# ---------------------------------------------------------------- visited tables
def test_visited_overflow_grows_and_reruns(pkg, po):
    """A filtered search whose filter admits almost nothing keeps expanding until its candidate queue is empty
    (hnsw.rs:992-1001), i.e. it visits the whole connected graph.  With ef = 10 and M = 8 the first table has
    next_pow2(max(1024, 2 * 26 * 16)) = 1024 slots and overflows at 768 entries, so on 20 000 points the library doubles it
    and re-runs the batch five times (1024 -> 32768 slots).  The answers must equal the oracle's, through the batched
    host path (search_flat: search_host_finish's slow path) and the single-query one (search_filter); a second call, on
    the grown tables, must too."""
    n, d = 20000, 24
    X = data(np.float32, "DistL2", n, d, 3)
    o = po.Oracle(M, n, 16, 32, "DistL2", d, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X, nthreads=8)
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, n, 16, 32, "DistL2")
    # a threaded build assigns internal ids in completion order: the rows go in by internal id, not in the order of X
    h.import_graph(o.export_vectors(), og, lv, o.entry, oracle_layers(o))
    Q = data(np.float32, "DistL2", 16, d, 4)
    allow = np.array([17, 9000, 19999])
    want = o.search_batch(Q, 10, 10, filter_ids=allow)
    assert np.all(want[4] >= 1)
    for attempt in range(2):
        same(launched(pkg, h.search_flat(Q, 10, 10, filter=allow)), want, f"search_flat, call {attempt}")
        one = h.search_filter(Q[5], 10, 10, filter=allow.tolist())
        assert [r.d_id for r in one] == want[0][5, :want[4][5]].tolist()
        assert np.array_equal(np.array([r.distance for r in one], np.float32), want[1][5, :want[4][5]])
    DONE.append("overflow")


def test_visited_epoch_wraps(pkg, po):
    """Epoch wrap-around.  A table entry is (epoch << id_bits) | id with id_bits = ceil(log2(capacity)); an index created
    with max_elements = 1 << 22 has id_bits = 22, so epoch_max = 2^10 - 1 = 1023, and a warp slot clears its table and
    restarts at epoch 1 on the begin() after its 1023rd epoch (a fresh pool starts at epoch 0xFFFFFFFF, which clears at
    once).  How many begin() calls one slot sees:
      * insert: with one insert in flight each launch runs one CTA of BUILD_THREADS / 32 = 4 warps, and the warp that takes
        the point calls begin() at least once (layer 0); 4200 points => 4199 begins over 4 slots => some slot >= 1050 >
        1023: it wraps.  The graph must still equal the oracle's.
      * queries: a single-threaded caller always leases search context 0.  The lean kernel runs one warp per CTA, so a
        1-query batch always lands on slot 0: 2100 calls = 2100 begins = two wraps.  The generic, filtered and std-tie
        kernels run one CTA of SEARCH_THREADS / 32 = 8 warps for an 8-query batch; 2100 such calls are 16 800 begins over
        8 slots, so some slot sees >= 2100 > 2 * 1023.
    Every answer is compared with the oracle."""
    n, d = 4200, 24
    X, o, h = build_both(pkg, po, np.float32, "DistL2", n, d, M, 48, seed=11, max_elements=1 << 22)
    calls = 2100
    Q = data(np.float32, "DistL2", 8 * calls, d, 12)
    allow = np.arange(0, n, 2)

    def run(q_per_call, k, ef, filt=None, what="", stats=True):
        nq = q_per_call * calls
        o.counters()
        want = o.search_batch(Q[:nq], k, ef, filter_ids=filt, nthreads=8)
        co = o.counters()
        h.enable_stats(stats)
        h.get_stats()
        parts = [h.search_flat(Q[i:i + q_per_call], k, ef, filter=filt) for i in range(0, nq, q_per_call)]
        launched(pkg)
        cg = h.get_stats()
        got = tuple(np.concatenate([p[j] for p in parts]) for j in range(5))
        same(got, want, what)
        # a visited entry lost or kept across the wrap shows in the traversal counters even where the answers survive it
        for key in ("evals", "expansions", "adj_read") if stats else ():
            assert cg[key] == co[key], (what, key, cg, co)

    run(1, 10, 10, what="lean")
    run(8, 10, 200, what="generic ef 200")
    run(8, 10, 10, allow, what="filtered", stats=False)
    o.set_mode(po.MODE_STD)
    h.set_tie_mode(1)
    run(8, 10, 10, what="std-tie")
    DONE.append("epoch")


# ---------------------------------------------------------------- the ledger
# compiled kernels no call records, with the reason
NOT_RECORDED = {
    "_ZN2hb18insert_link_kernelENS_12InsertParamsE":
        "launched directly after every insert search (run_insert_range), not through launch_kernel, so that the insert "
        "search kernel stays the recorded one",
}


def cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None:
        for root in (os.environ.get("CUDA_HOME"), os.environ.get("CUDA_PATH"), "/usr/local/cuda"):
            if root and os.path.exists(os.path.join(root, "bin", "cuobjdump")):
                return os.path.join(root, "bin", "cuobjdump")
    return exe


def test_zz_every_compiled_kernel_was_reached(pkg):
    expected = len(CASES) + len(INSERT_CASES) + len(PROB) + len(DIST_CASES) + 2
    if len(DONE) != expected:
        pytest.fail(f"the ledger needs every case of this module to pass: {len(DONE)} of {expected} did")
    exe = cuobjdump()
    if exe is None:
        pytest.fail("cuobjdump (CUDA toolkit) not found: the compiled kernel list cannot be read")
    out = subprocess.run([exe, "-symbols", pkg.lib_path()], capture_output=True, text=True, check=True).stdout
    compiled = set(re.findall(r"STO_ENTRY\s+(\S+)", out))
    assert len(compiled) > 300, f"cuobjdump listed {len(compiled)} kernels"
    assert not (set(NOT_RECORDED) - compiled), "stale NOT_RECORDED entry"
    stray = LEDGER - compiled
    assert not stray, f"recorded kernels that cuobjdump does not list: {sorted(stray)}"
    missed = sorted(compiled - LEDGER - set(NOT_RECORDED))
    print(f"\nkernel ledger: {len(LEDGER)} of {len(compiled)} compiled entry points reached, "
          f"{len(NOT_RECORDED)} not recorded by design; module wall time {time.time() - T0:.0f} s")
    assert not missed, f"{len(missed)} compiled kernels never ran:\n" + "\n".join(missed)

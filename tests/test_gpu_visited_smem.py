"""The lean kernel's visited first stage in shared memory (VisitedT<FirstStage::Shared>, csrc/common.cuh), bit-exact.

A staged lean launch keeps each warp's first stage (cap / 4 entries) in a window of its shared memory and moves a search
that fills 3/4 of it to the full stage in the slot's global table; a launch whose window would cost CTAs per SM runs
single-stage.  hnsw_b200_set_visited_stages mode 1 forces the stages on for these small graphs.  Each case checks ids,
distance bits, PointIds, counts and traversal counters against the oracle and against the same search run single-stage
(mode 2): searches that stay in the window, searches that move to the full stage, searches that overflow the full stage
(the host re-runs the batch with larger tables), an epoch wrap, and a shape whose window does not fit.
"""
import numpy as np
import pytest

from answers import same
from visited import ALWAYS, EF, K, NEVER, move_at, staged_graph

pytestmark = pytest.mark.gpu

M4 = 4  # staged_graph's M


def lean_bytes(ef):
    """shared memory of a lean CTA without a window (kernels.h lean_layout): 64 or 128 queue keys, 32 ids, 32 distances"""
    return (64 if ef <= 64 else 128) * 8 + 256


def search(pkg, h, Q, ef, mode):
    h.set_visited_stages(mode)
    h.enable_stats(True)
    h.get_stats()
    got = h.search_flat(Q, K, ef)
    st = h.get_stats()
    h.enable_stats(False)
    assert "search_lean_kernel" in pkg.last_kernel()
    return got, st, pkg.last_kernel_shape()


def check_both(pkg, h, o, Q, ef, what, window, rerun=False):
    """the window (mode 1) and single-stage (mode 2) against the oracle, answers and counters; `window`: the entries
    of the first stage in shared memory that mode 1 must have launched with (0: none, the launch ran single-stage).
    `rerun`: mode 1 overflows and the host re-runs the batch, so its counters also hold the overflowed attempts' work and
    only its answers are compared."""
    o.counters()
    want = o.search_batch(Q, K, ef, nthreads=8)
    co = o.counters()
    shapes = {}
    for mode in (ALWAYS, NEVER):
        got, cg, shapes[mode] = search(pkg, h, Q, ef, mode)
        same(got, want, f"{what}, mode {mode}")
        for key in ("evals", "expansions", "adj_read") if not (rerun and mode == ALWAYS) else ():
            assert cg[key] == co[key], (what, mode, key, cg, co)
    h.set_visited_stages(ALWAYS)
    assert shapes[ALWAYS][0] == lean_bytes(ef) + 4 * window and shapes[NEVER][0] == lean_bytes(ef), (what, shapes)
    assert shapes[ALWAYS][2] == shapes[NEVER][2], ("the window cost CTAs per SM", what, shapes)


def evals_per_query(o, Q, ef):
    ev = []
    o.counters()
    for i in range(len(Q)):
        o.search_batch(Q[i:i + 1], K, ef)
        ev.append(o.counters()["evals"])
    return np.array(ev)


@pytest.fixture(scope="module")
def graph(pkg, po):
    return staged_graph(pkg, po, 6000, 24, seed=41)


def test_stay_in_window_and_move(pkg, po, graph):
    """M = 4, ef = 16: a 256-entry window (1 KB) and a 1024-entry full stage; a search moves after 192 insertions.
    One batch of queries that all stay in the window, one of queries that all move, each checked on its own."""
    X, o, h, top = graph
    Q = pkg.datagen.make("uniform", 1200, 24, 43)
    Q[:40] = X[:40]
    ev = evals_per_query(o, Q, EF)
    at = move_at(EF)
    stay, moved = Q[ev < at], Q[ev >= at + 1 + top * M4]
    assert len(stay) >= 20 and len(moved) >= 20, (at, len(stay), len(moved), ev.min(), ev.max())
    check_both(pkg, h, o, stay, EF, "stay in the window", 256)
    check_both(pkg, h, o, moved, EF, "move to the full stage", 256)
    check_both(pkg, h, o, Q, EF, "mixed", 256)


def chain_graph(pkg, po, n, d, M):
    """points 0, 1, 2, ... on a line, layer-0 lists [i+1, i+2, i-1, i-2], one layer, entry 0: a query beyond point n-1
    walks the whole chain (n + 1 evaluations)"""
    X = np.zeros((n, d), np.float32)
    X[:, 0] = np.arange(n, dtype=np.float32)
    lists = [[j for j in (i + 1, i + 2, i - 1, i - 2) if 0 <= j < n] for i in range(n)]
    off = np.zeros(n + 1, np.uint64)
    off[1:] = np.cumsum([len(l) for l in lists])
    ids = np.array([j for l in lists for j in l], np.uint32)
    ds = np.array([abs(float(j - i)) for i, l in enumerate(lists) for j in l], np.float32)
    origin, levels = np.arange(n, dtype=np.uint64), np.zeros(n, np.uint8)
    o = po.Oracle(M, n, 16, 48, "DistL2", d, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.import_graph(X, origin, levels, 0, {0: (off, ids, ds)})
    h = pkg.Hnsw(M, n, 16, 48, "DistL2")
    h.import_graph(X, origin, levels, 0, [(off, ids, ds)])
    return o, h


def test_overflow_reruns(pkg, po):
    """M = 2, ef = 16: full stage 1024 entries, window 256.  Every search of the chain inserts 3 001 ids: it moves at
    192, overflows at 768, and the host re-runs the batch with 2048 (overflow at 1536), then 4096 entries (a 4 KB
    window), where it fits"""
    n, d = 3000, 24
    o, h = chain_graph(pkg, po, n, d, 2)
    Q = np.zeros((64, d), np.float32)
    Q[:, 0] = n + np.arange(64, dtype=np.float32)
    Q[:, 1] = 0.25 * np.arange(64, dtype=np.float32)
    ev = evals_per_query(o, Q[:2], EF)
    assert (ev > 2048 * 3 // 4).all() and (ev < 4096 * 3 // 4).all(), ev
    for call in range(2):  # the second call starts on the grown tables
        check_both(pkg, h, o, Q, EF, f"overflow, call {call}", 1024, rerun=call == 0)


def test_epoch_wrap(pkg, po):
    """max_elements = 1 << 22 gives id_bits = 22 and 1023 epochs per slot; 1-query calls all land on slot 0 of search
    context 0, so 1100 of them wrap its epoch once, with searches that stay in the window and searches that moved"""
    X, o, h, top = staged_graph(pkg, po, 6000, 24, seed=45, max_elements=1 << 22)
    calls = 1100
    Q = pkg.datagen.make("uniform", calls, 24, 46)
    Q[:100] = X[:100]
    o.counters()
    want = o.search_batch(Q, K, EF, nthreads=8)
    co = o.counters()
    h.set_visited_stages(ALWAYS)
    h.enable_stats(True)
    h.get_stats()
    parts, ev = [], []
    for i in range(calls):
        parts.append(h.search_flat(Q[i:i + 1], K, EF))
        ev.append(h.get_stats(reset=False)["evals"])
    cg = h.get_stats()
    h.enable_stats(False)
    per_q = np.diff(np.array([0] + ev))
    at = move_at(EF)
    assert (per_q >= at + 1 + top * M4).sum() > 10 and (per_q < at).sum() > 10, "too few moved or stayed"
    same(tuple(np.concatenate([p[j] for p in parts]) for j in range(5)), want, "epoch wrap")
    for key in ("evals", "expansions", "adj_read"):
        assert cg[key] == co[key], (key, cg, co)


def test_window_does_not_fit(pkg, po):
    """M = 16, ef = 128: full stage next_pow2(2 * 144 * 32) = 16 384 entries, a 16 KB window; with the 1 280-byte lean
    layout of a 128-slot queue that is 17.3 KB per CTA, and ~20 one-warp CTAs per SM would need ~360 KB of the 228 KB an
    H100 SM has.  Forced staging must fall back to one stage and still answer exactly."""
    n, d, M = 4000, 24, 16
    X = pkg.datagen.make("uniform", n, d, 47)
    o = po.Oracle(M, n, 16, 100, "DistL2", d, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X, nthreads=8)
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, n, 16, 100, "DistL2")
    h.import_graph(o.export_vectors(), og, lv, o.entry, [o.export_layer(l) for l in range(16)])
    Q = pkg.datagen.make("uniform", 300, d, 48)
    check_both(pkg, h, o, Q, 128, "ef 128, no window", 0)

"""The visited set's two stages (Visited, csrc/common.cuh), bit-exact against the oracle.

A search can start in a first stage of cap / 4 entries and move to the full stage of `cap` entries once the first one
holds 3/4 of its capacity.  By default (hnsw_b200_set_visited_stages mode 0) searches do so only when the launch's
full-size tables would not fit in L2, which these small graphs never reach, so the cases here force the stages on (mode 1).
With M = 4 (layer-0 degree 8) and ef = 16 the full stage has next_pow2(max(1024, 2 * 32 * 8)) = 1024 entries and the first
stage 256, so a search moves after 192 layer-0 insertions.  One insertion is one layer-0 evaluation (the entry point
included), so each case first counts, with the oracle, the evaluations of every query at its own ef and filter, and checks
that the batch has queries that move (and, where the ef allows it, queries that stay) before it relies on them.  Every kernel that searches a
visited set runs here: lean, generic (ef > 128, and rows over 512 bytes), filtered and std-tie.  Answers, distance bits,
PointIds, counts and traversal counters must equal the oracle's.
"""
import numpy as np
import pytest

from answers import same
from visited import ALWAYS, AUTO, EF, EFC, K, M, NEVER, move_at, staged_graph

pytestmark = pytest.mark.gpu

def assert_mix(o, Q, ef, top, what, filt=None, some_stay=True):
    """the oracle's evaluations of each query: some pass the move point even after the descent's evaluations (at most
    1 + top * M) are taken off, and (some_stay) others stay below it"""
    ev = []
    o.counters()
    for i in range(len(Q)):
        o.search_batch(Q[i:i + 1], K, ef, filter_ids=filt)
        ev.append(o.counters()["evals"])
    ev = np.array(ev)
    at = move_at(ef)
    stayed, moved = int((ev < at).sum()), int((ev >= at + 1 + top * M).sum())
    assert moved > 0 and (stayed > 0 or not some_stay), (what, at, stayed, moved, ev.min(), ev.max())


def check(h, o, Q, ef, what, filt=None, stats=True):
    o.counters()
    want = o.search_batch(Q, K, ef, filter_ids=filt, nthreads=8)
    co = o.counters()
    h.enable_stats(stats)
    h.get_stats()
    got = h.search_flat(Q, K, ef, filter=filt)
    cg = h.get_stats()
    h.enable_stats(False)
    same(got, want, what)
    for key in ("evals", "expansions", "adj_read") if stats else ():
        assert cg[key] == co[key], (what, key, cg, co)


@pytest.fixture(scope="module")
def graph(pkg, po):
    return staged_graph(pkg, po, 6000, 24, seed=21)


def test_lean_every_mode_and_back(pkg, po, graph):
    """the lean kernel staged, single-stage, auto and staged again on one handle: a change of layout must not leave
    entries that the next layout reads as visited"""
    X, o, h, top = graph
    Q = pkg.datagen.make("uniform", 500, 24, 23)
    Q[:20] = X[:20]
    assert_mix(o, Q, EF, top, "lean")
    for mode in (ALWAYS, NEVER, AUTO, ALWAYS):
        h.set_visited_stages(mode)
        check(h, o, Q, EF, f"lean, mode {mode}")
    with pytest.raises(Exception):
        h.set_visited_stages(3)


@pytest.mark.parametrize("what,ef,tie", [("generic ef 160", 160, False), ("std-tie", EF, True)])
def test_unfiltered_kernels(pkg, po, graph, what, ef, tie):
    X, o, h, top = graph
    Q = pkg.datagen.make("uniform", 500, 24, 23)
    Q[:20] = X[:20]
    if tie:
        o.set_mode(po.MODE_STD)
        h.set_tie_mode(1)
    try:
        assert_mix(o, Q, ef, top, what, some_stay=not ef > 128)   # at ef 160 every search outgrows the first stage
        check(h, o, Q, ef, what)
    finally:
        if tie:
            o.set_mode(po.MODE_DET)
            h.set_tie_mode(0)


def test_filtered_kernel(pkg, po, graph):
    X, o, h, top = graph
    Q = pkg.datagen.make("uniform", 300, 24, 24)
    allow = np.arange(0, len(X), 3)
    assert_mix(o, Q, EF, top, "filtered", filt=allow, some_stay=False)   # a filtered search expands further
    check(h, o, Q, EF, "filtered", filt=allow, stats=False)


def test_generic_wide_rows(pkg, po):
    """rows of 640 bytes: the generic kernel at ef = 16, the same 256 / 1024-entry stages"""
    X, o, h, top = staged_graph(pkg, po, 3000, 150, seed=25)
    Q = pkg.datagen.make("uniform", 300, 150, 26)
    assert_mix(o, Q, EF, top, "generic wide rows")
    check(h, o, Q, EF, "generic wide rows")


def test_moves_then_overflows_and_reruns(pkg, po):
    """a filter that admits almost nothing keeps the search expanding over the whole graph: it moves to the full stage
    at 192 insertions, overflows it at 768, and the host re-runs the batch with larger tables until it fits"""
    n, d = 12000, 24
    X = pkg.datagen.make("uniform", n, d, 27)
    o = po.Oracle(M, n, 16, EFC, "DistL2", d, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.insert_batch(X, nthreads=8)
    lv, rk, og = o.export_points()
    h = pkg.Hnsw(M, n, 16, EFC, "DistL2")
    h.import_graph(o.export_vectors(), og, lv, o.entry, [o.export_layer(l) for l in range(16)])
    h.set_visited_stages(ALWAYS)
    Q = pkg.datagen.make("uniform", 16, d, 28)
    allow = np.array([5, 6000, 11999])
    o.counters()
    want = o.search_batch(Q, K, EF, filter_ids=allow)
    assert o.counters()["evals"] >= 1024 * len(Q), "the searches do not outgrow the first full stage"
    for call in range(2):   # the second call runs on the grown tables
        same(h.search_flat(Q, K, EF, filter=allow), want, f"call {call}")


def test_epoch_wrap_with_both_stages(pkg, po):
    """max_elements = 1 << 22 gives id_bits = 22 and 1023 epochs per table; 1-query lean calls all land on slot 0 of
    search context 0, so 1100 of them wrap its epoch once, with entries of moved searches left in the full stage.  A
    full stage that the wrap did not clear would hold entries of the restarted epochs, which the counters would show."""
    X, o, h, top = staged_graph(pkg, po, 6000, 24, seed=29, max_elements=1 << 22)
    calls = 1100
    Q = pkg.datagen.make("uniform", calls, 24, 30)
    o.counters()
    want = o.search_batch(Q, K, EF, nthreads=8)
    co = o.counters()
    h.enable_stats(True)
    h.get_stats()
    parts, ev = [], []
    for i in range(calls):
        parts.append(h.search_flat(Q[i:i + 1], K, EF))
        ev.append(h.get_stats(reset=False)["evals"])
    cg = h.get_stats()
    h.enable_stats(False)
    per_q = np.diff(np.array([0] + ev))
    assert (per_q >= move_at(EF) + 1 + top * M).sum() > 10, "too few searches moved to the full stage"
    same(tuple(np.concatenate([p[j] for p in parts]) for j in range(5)), want, "epoch wrap")
    for key in ("evals", "expansions", "adj_read"):
        assert cg[key] == co[key], (key, cg, co)

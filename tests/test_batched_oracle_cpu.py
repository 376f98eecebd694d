"""The oracle's batch-synchronous insert (Oracle.insert_batched) and the engine's batch schedule (batched.engine_batches),
without a GPU.

insert_batched restates how Index::insert_batch builds: every batch searches the graph as it stood when the batch began,
then links its points.  These tests pin that restatement to the serial builds the suite already trusts (batches of one
point), pin the two freedoms DESIGN.md §4.3 claims do not matter (the order phase B links a batch in, the threads phase
A runs on), show that the default schedule builds a different graph than a serial build does (so the GPU tests of
test_gpu_batched_insert.py check something the serial tests do not), and work two small cases by hand.
"""
import numpy as np
import pytest

from batched import engine_batches, entry_level_after, promoting_levels
from linkgraph import insert_link_mode1

N, D, M, EFC = 2000, 16, 8, 48


def oracle(po, n=N, extend=False, keep_pruned=False):
    o = po.Oracle(M, n, 16, EFC, "DistL2", D, mode=po.MODE_DET, order=po.ORDER_GPU)
    o.set_extend_candidates(extend)
    o.set_keeping_pruned(keep_pruned)
    return o


def points(n=N, seed=3):
    return np.random.default_rng(seed).random((n, D), dtype=np.float32)


def graph(o):
    """everything a build decides: entry, levels, ranks, origins and every list of every layer, distances as bits"""
    lv, rk, og = o.export_points()
    out = [np.array([o.entry]), lv, rk, og]
    for layer in range(16):
        off, ids, ds = o.export_layer(layer)
        out += [off, ids, ds.view(np.uint32)]
    return out


def assert_same(a, b):
    ga, gb = graph(a), graph(b)
    for i, (x, y) in enumerate(zip(ga, gb)):
        assert np.array_equal(x, y), f"graph part {i} differs"


@pytest.mark.parametrize("options", [False, True], ids=["plain", "ext-kp"])
def test_batches_of_one_equal_the_serial_build(po, options):
    X, lv = points(), promoting_levels(po, N, 5)
    serial, batched = oracle(po, extend=options, keep_pruned=options), oracle(po, extend=options, keep_pruned=options)
    serial.insert_batch(X, levels=lv)
    cs = serial.counters()
    batched.insert_batched(X, levels=lv, batches=[1] * N)
    cb = batched.counters()
    assert_same(serial, batched)
    assert cs == cb


def test_batches_of_one_in_link_mode1_equal_linkgraph(po):
    X, lv = points(800), promoting_levels(po, 800, 6)
    ref, batched = oracle(po, 800), oracle(po, 800)
    insert_link_mode1(ref, X, lv)
    batched.insert_batched(X, levels=lv, batches=[1] * 800, link_mode=1)
    assert_same(ref, batched)


@pytest.mark.parametrize("link_mode", [0, 1])
def test_link_order_does_not_matter(po, link_mode):
    X, lv = points(), promoting_levels(po, N, 7)
    sched = engine_batches(0, -1, lv)
    builds = []
    for seed in (0, 11, 12345):
        o = oracle(po)
        o.insert_batched(X, levels=lv, batches=sched, link_mode=link_mode, order_seed=seed)
        builds.append(o)
    assert_same(builds[0], builds[1])
    assert_same(builds[0], builds[2])


def test_thread_count_does_not_matter(po):
    X, lv = points(), promoting_levels(po, N, 8)
    sched = engine_batches(0, -1, lv, ratio=4)
    builds, counters = [], []
    for nthreads in (1, 8):
        o = oracle(po, extend=True, keep_pruned=True)
        o.insert_batched(X, levels=lv, batches=sched, nthreads=nthreads)
        builds.append(o)
        counters.append(o.counters())
    assert_same(builds[0], builds[1])
    assert counters[0] == counters[1]


def test_default_schedule_builds_another_graph_than_serial(po):
    X, lv = points(), promoting_levels(po, N, 9)
    sched = engine_batches(0, -1, lv)
    assert max(sched) > 1
    serial, batched = oracle(po), oracle(po)
    serial.insert_batch(X, levels=lv)
    batched.insert_batched(X, levels=lv, batches=sched)
    s0, b0 = serial.export_layer(0), batched.export_layer(0)
    assert not (np.array_equal(s0[0], b0[0]) and np.array_equal(s0[1], b0[1]))


def test_two_equal_vectors_in_one_batch_do_not_link(po):
    """the second copy of a vector finds the first at distance 0 in a serial build; in one batch neither sees the other"""
    X = points(202, 10)
    X[201] = X[200]
    lv = np.zeros(202, np.int32)
    for batches in ([1] * 202, engine_batches(0, -1, lv[:200]) + [2]):
        o = oracle(po, 202)
        o.insert_batched(X, levels=lv, batches=batches)
        off, ids, ds = o.export_layer(0)
        l200, l201 = ids[off[200]:off[201]].tolist(), ids[off[201]:off[202]].tolist()
        if batches[-1] == 1:
            assert l201[0] == 200 and ds[off[201]] == 0.0
        else:
            assert 200 not in l201 and 201 not in l200


def test_layer_mask_is_taken_per_point(po):
    """Point 0 has level 2, every other stored point level 0, so layer 1 is empty (the reference tests emptiness by the
    points of exactly that level, hnsw.rs:942-946).  A batch holds two level-0 points x, y and then a level-1 point z:
    x and y must skip layer 1 in their descent, z searches it.  Were the masks taken after the whole batch, x and y would
    expand the entry point at layer 1 as well, which adds to the counters but to no list the engine keeps.  So the
    batch's counters must be those of [x, y] alone plus those of [z] alone, each on the same graph."""
    n0 = 300
    X = points(n0 + 3, 12)
    lv = np.zeros(n0 + 3, np.int32)
    lv[0], lv[-1] = 2, 1
    prefix = engine_batches(0, -1, lv[:n0])
    assert engine_batches(n0, 2, lv[n0:]) == [3]

    def tail(take, batch):
        o = oracle(po, n0 + 3)
        o.insert_batched(X[:n0], levels=lv[:n0], batches=prefix)
        o.counters()
        o.insert_batched(X[n0:][take], ids=np.arange(n0, n0 + 3)[take], levels=lv[n0:][take], batches=batch)
        return o.counters()

    whole = tail([0, 1, 2], [3])
    xy, z = tail([0, 1], [2]), tail([2], [1])
    for key in ("evals", "expansions", "adj_read"):
        assert whole[key] == xy[key] + z[key], (key, whole, xy, z)


def test_engine_batches_worked_examples():
    # empty index, ratio 16: the first point alone, then one at a time until 32 are linked, then 2
    assert engine_batches(0, -1, np.zeros(40, int)) == [1] * 32 + [2] * 4
    # 100 linked points at entry level 1: batches of 6; the level-2 point at 3 is cut off and goes alone
    lv = np.zeros(20, int)
    lv[3] = 2
    assert engine_batches(100, 1, lv) == [3, 1, 6, 6, 4]
    # a point at the entry level does not cut; the batch grows to 7 once 112 points are linked
    lv[3] = 1
    assert engine_batches(100, 1, lv) == [6, 6, 7, 1]
    # max_batch caps
    assert engine_batches(1000, 3, np.zeros(300, int), ratio=1, max_batch=128) == [128, 128, 44]
    # state across two calls: 40 points, then 12 more whose first is promoted
    lv = np.zeros(52, int)
    lv[40] = 1
    first = engine_batches(0, -1, lv[:40])
    top = entry_level_after(0, -1, lv[:40])
    assert top == 0
    assert engine_batches(40, top, lv[40:]) == [1, 2, 2, 2, 2, 3]
    assert entry_level_after(40, top, lv[40:]) == 1
    assert first == [1] * 32 + [2] * 4


def test_refused_batches_are_not_the_engines(po):
    """the oracle aborts on batches the engine never makes; check the schedule never contains one"""
    for seed in range(5):
        lv = promoting_levels(po, N, seed)
        sched = engine_batches(0, -1, lv)
        assert sched[0] == 1 and sum(sched) == N
        start, top = 0, -1
        for b in sched:
            if b > 1:
                assert lv[start:start + b].max() <= top
            top = max(top, int(lv[start:start + b].max()))
            start += b
